// batch.cuh -- host rules of batch proving (g16_prove_batch): how many proofs share one pass of the kernels, and the
// per-proof tail that turns the five MSM results and the five fixed-base products of one proof into its group elements.
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

// The (r, s)-only terms of a proof, regrouped so that every scalar multiplication by r or s of a KEY point is one
// fixed-base product computed on the GPU for the whole batch (prover.rs:76-131, with P_a = a_query[0] + alpha_g1,
// P_b = b_g1_query[0] + beta_g1, P_2 = b_g2_query[0] + beta_g2):
//   g_a  = r d1 + P_a + A
//   g2_b = s d2 + P_2 + B2
//   g_c  = (r s) d1 + s P_a + r P_b + s A + r B1 + L + H
// prover.rs forms g_c = s g_a + r g1_b - (r s) d1 + L + H with g1_b = s d1 + P_b + B1; expanding gives the line above
// (when r == 0, prover.rs skips g1_b: every r term is the identity here too).  The affine result is unique, so the bytes
// equal g16_prove's.
template <class Fq, class Fq2>
struct BatchTailIn {
  Affine<Fq> r_d1, rs_d1, s_pa, r_pb;   // fixed-base products of this proof
  Affine<Fq2> s_d2;
  XYZZ<Fq> a, b1, l, h;                 // MSM results of this proof
  XYZZ<Fq2> b2;
};
// r, s: canonical (not Montgomery) 32-bit limbs
template <class Fq, class Fq2>
void batch_tail(const BatchTailIn<Fq, Fq2>& x, const Affine<Fq>& p_a, const Affine<Fq2>& p_2, const uint32_t r[8],
                const uint32_t s[8], bool r_zero, XYZZ<Fq>& g_a, XYZZ<Fq2>& g2_b, XYZZ<Fq>& g_c) {
  g_a = XYZZ<Fq>::from_affine(x.r_d1);
  g_a.madd(p_a);
  g_a.add(x.a);
  g2_b = XYZZ<Fq2>::from_affine(x.s_d2);
  g2_b.madd(p_2);
  g2_b.add(x.b2);
  g_c = x.a.mul_u32(s, 8);
  g_c.madd(x.rs_d1);
  g_c.madd(x.s_pa);
  if (!r_zero) {
    g_c.madd(x.r_pb);
    g_c.add(x.b1.mul_u32(r, 8));
  }
  g_c.add(x.l);
  g_c.add(x.h);
}

}  // namespace g16
