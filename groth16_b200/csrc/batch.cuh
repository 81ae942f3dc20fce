// batch.cuh -- host rules of proving: how many proofs of a batch (g16_prove_batch) share one pass of the kernels, and the
// tail every prover path shares, which turns a proof's MSM results and its five key products into its group elements.
// Pure host code over the field / curve templates, so tests/host/batch_plan_check.cu checks it without a GPU.
#pragma once
#include <algorithm>
#include <cstdint>
#include "ec.cuh"

namespace g16 {

static constexpr uint32_t BATCH_MAX_GRID_Y = 65535;            // proofs of a group index blockIdx.y
static constexpr uint64_t BATCH_MEMORY_MARGIN = 1ull << 30;   // left free for everything else on the device

// Proofs per group.  `entries_per_proof`: padded sorted entries of the largest MSM of one proof (the sorted offsets are
// 32-bit); `bytes_per_proof`: device workspace one proof of a group needs; `slots`: groups resident at once.
// group == 0: the largest G <= count with G * entries_per_proof < 2^32, G <= 65535 and slots * G * bytes_per_proof within
// free_bytes less 1 GiB.  group > 0: that many (at most count), still under the first two limits, which are correctness
// limits.  Never less than 1 (for count > 0).
inline uint32_t batch_group_size(uint32_t count, uint32_t group, uint64_t entries_per_proof, uint64_t bytes_per_proof,
                                 uint64_t free_bytes, uint32_t slots) {
  if (count == 0) return 0;
  uint64_t g = count;
  if (entries_per_proof > 0) g = std::min<uint64_t>(g, 0xffffffffull / entries_per_proof);
  g = std::min<uint64_t>(g, BATCH_MAX_GRID_Y);
  if (group > 0) {
    g = std::min<uint64_t>(g, group);
  } else {
    const uint64_t avail = free_bytes > BATCH_MEMORY_MARGIN ? free_bytes - BATCH_MEMORY_MARGIN : 0;
    const uint64_t per = std::max<uint64_t>(1, bytes_per_proof) * std::max<uint32_t>(1, slots);
    g = std::min<uint64_t>(g, avail / per);
  }
  return (uint32_t)std::max<uint64_t>(1, g);
}

// The tail of every proof (prover.rs:76-131), regrouped so that each scalar multiplication of a KEY point by r, s or r s
// is one of five key products, with P_a = a_query[0] + alpha_g1, P_b = b_g1_query[0] + beta_g1 and
// P_2 = b_g2_query[0] + beta_g2:
//   g_a  = r d1 + P_a + A
//   g2_b = s d2 + P_2 + B2
//   g_c  = (r s) d1 + s P_a + r P_b + C,      C = s A + r B1 + L + H
// prover.rs forms g_c = s g_a + r g1_b - (r s) d1 + L + H with g1_b = s d1 + P_b + B1; expanding gives the line above
// (when r == 0, prover.rs skips g1_b: r P_b and r B1 are the identity here too).  A, B2 and C are sums over the ranks
// when the key is sharded.  The affine result is unique, so the bytes equal the prover.rs order's.
template <class Fq, class Fq2>
struct KeyProducts {
  XYZZ<Fq> r_d1, rs_d1, s_pa, r_pb;
  XYZZ<Fq2> s_d2;
};
template <class Fq, class Fq2>
struct ProofPoints {
  XYZZ<Fq> g_a;
  XYZZ<Fq2> g2_b;
  XYZZ<Fq> g_c;
};
template <class Fq, class Fq2>
ProofPoints<Fq, Fq2> proof_tail(const KeyProducts<Fq, Fq2>& k, const Affine<Fq>& p_a, const Affine<Fq2>& p_2,
                                const XYZZ<Fq>& a, const XYZZ<Fq2>& b2, const XYZZ<Fq>& c) {
  ProofPoints<Fq, Fq2> p{k.r_d1, k.s_d2, k.rs_d1};
  p.g_a.madd(p_a);
  p.g_a.add(a);
  p.g2_b.madd(p_2);
  p.g2_b.add(b2);
  p.g_c.add(k.s_pa);
  p.g_c.add(k.r_pb);
  p.g_c.add(c);
  return p;
}

}  // namespace g16
