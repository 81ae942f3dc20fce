// Host-only check (built by nvcc, runs without a GPU) of the batch-proving rules and the proof tail of groth16_b200/csrc:
//   1. the bucket-reduction layout of a batched MSM pass (msm.cuh): K proofs x ne bucket sets, msm_sum_strided replaced by
//      literal host sums as in msm_plan_check.cu; msm_finish(ws, g, k) must equal the Horner definition for proof k alone;
//   2. a zero-initialised MsmGeom (batch 0) and batch 1 give the same layout and result;
//   3. batch_group_size (batch.cuh): each of its three caps binds, the result stays in [1, count], an explicit group is kept;
//   4. proof_tail (batch.cuh), which every prover path uses, against a tail in prover.rs's own order kept here as the
//      reference, with the key products in projective and in affine form, on the host EC back-end, for BN254 and BLS12-381;
//   5. the batch prover's per-proof workspace bound (msm_batch_bytes_per_proof, which Engine::batch_bytes_per_proof sums):
//      G times it covers what MsmWorkspace::prepare reserves (msm_ws_bytes) for a group of G = 1, 2, 64 at every acc_k0
//      (4 .. 7 included), 0 .. 6 rounds, uneven rounds on a shared B sorted list, msm_ne 0 / 1 / 8, msm_c 12 .. 16.
// stdin: the G1 and G2 generators of BN254 then BLS12-381 as Montgomery u64 limbs in hex (affine x || y).
#include <cstdio>
#include <cstring>
#include <utility>
#include <vector>
#include "../../groth16_b200/csrc/batch.cuh"
#include "../../groth16_b200/csrc/msm.cuh"
using namespace g16;

static int bad = 0, cases = 0;
#define CHECK(cond, ...)                   \
  do {                                     \
    cases++;                               \
    if (!(cond)) {                         \
      bad++;                               \
      fprintf(stderr, __VA_ARGS__);        \
      fprintf(stderr, "\n");               \
    }                                      \
  } while (0)

static uint64_t seed = 0x5eed;
static uint32_t rnd() { seed = seed * 6364136223846793005ull + 1442695040888963407ull; return (uint32_t)(seed >> 32); }

template <class PT>
static bool same(const PT& a, const PT& b) {
  auto x = a.to_affine(), y = b.to_affine();
  return x.x == y.x && x.y == y.y;
}

// ---- 1 / 2: reduction layout of a batched pass ------------------------------------------------------------------------
using F1 = Fp<BN254_FqP>;
using Pt = XYZZ<F1>;
static F1 fp_small(uint32_t x) {
  F1 r = F1::zero();
  r.v[0] = x;
  return F1::to_mont(r);
}
// buckets[set][b] = s * G with random s; returns the per-proof Horner results computed by msm_finish for geometry g and
// checks them against the definition
static std::vector<Pt> layout_case(int m, int ne, uint32_t K, uint32_t batch_field) {
  const Affine<F1> G{fp_small(1), fp_small(2)};   // BN254 G1 generator
  Pt mult[8];
  mult[0] = Pt::inf();
  for (int i = 1; i < 8; i++) { mult[i] = mult[i - 1]; mult[i].madd(G); }
  const int c = m + 1;
  MsmGeom g{};
  g.n = 1; g.c = c; g.ne = ne; g.W = ne; g.copies = 1; g.B = 1u << m; g.k0 = 64;
  g.batch = batch_field;
  g.nkeys = g.sets() * g.B;
  g.max_entries = 1;
  const uint32_t sets = g.sets();
  CHECK(sets == (uint32_t)ne * K, "m=%d ne=%d K=%u: sets() = %u", m, ne, K, sets);
  MsmWorkspace<F1> ws;
  ws.plan.make(m);
  const MsmRedPlan& pl = ws.plan;
  const size_t B = g.B;
  std::vector<Pt> buckets(B * sets), inner(pl.inner_pts * sets + 1), leaf(pl.leaf_pts * sets + 1);
  std::vector<uint64_t> weight(sets, 0);
  for (uint32_t w = 0; w < sets; w++)
    for (size_t b = 0; b < B; b++) {
      const uint32_t s = (rnd() % 3 == 0) ? 0 : rnd() % 8;
      buckets[w * B + b] = mult[s];
      weight[w] += (uint64_t)(b + 1) * s;
    }
  auto arr = [&](int id) -> Pt* {
    if (id == 0) return buckets.data();
    const MsmRedNode& nd = pl.nodes[id];
    return (nd.leaf ? leaf.data() : inner.data()) + nd.off * sets;   // msm_enqueue's arr(): offsets scale with sets()
  };
  for (int id = 0; id < pl.n_nodes; id++) {   // the msm_sum_strided jobs: n_out = per_win_out * sets()
    const MsmRedNode& nd = pl.nodes[id];
    if (nd.leaf) continue;
    const size_t len = (size_t)1 << nd.log_len, a0 = (size_t)1 << nd.a0, a1 = (size_t)1 << nd.a1;
    for (uint32_t w = 0; w < sets; w++) {
      for (size_t hi = 0; hi < a1; hi++) {
        Pt s = Pt::inf();
        for (size_t lo = 0; lo < a0; lo++) s.add(arr(id)[w * len + hi * a0 + lo]);
        arr(nd.child_r)[w * a1 + hi] = s;
      }
      for (size_t lo = 0; lo < a0; lo++) {
        Pt s = Pt::inf();
        for (size_t hi = 0; hi < a1; hi++) s.add(arr(id)[w * len + hi * a0 + lo]);
        arr(nd.child_c)[w * a0 + lo] = s;
      }
    }
  }
  ws.h_leaf = pl.nodes[0].leaf ? buckets.data() : leaf.data();
  std::vector<Pt> got(K);
  for (uint32_t k = 0; k < K; k++) {
    got[k] = msm_finish<F1>(ws, g, k);
    Pt want = Pt::inf();   // sum_e 2^(c e) sum_b (b + 1) bucket[k ne + e][b], proof k's sets only
    for (int e = ne - 1; e >= 0; e--) {
      for (int i = 0; i < c; i++) want.dbl_inplace();
      const uint64_t wt = weight[k * ne + e];
      uint32_t kk[2] = {(uint32_t)wt, (uint32_t)(wt >> 32)};
      want.add(Pt::from_affine(G).mul_u32(kk, 2));
    }
    CHECK(same(got[k], want), "m=%d ne=%d K=%u: msm_finish of proof %u differs from its Horner sum", m, ne, K, k);
  }
  ws.h_leaf = nullptr;
  return got;
}

// ---- 4: the regrouped tail against the prover.rs order -----------------------------------------------------------------
template <class FrP, class FqP, int NR>
struct TailCheck {
  using Fr = Fp<FrP>;
  using Fq = Fp<FqP>;
  using Fq2 = Fp2<FqP, NR>;
  using A1 = Affine<Fq>;
  using A2 = Affine<Fq2>;
  using P1 = XYZZ<Fq>;
  using P2 = XYZZ<Fq2>;
  A1 g1;
  A2 g2;
  static void canon(const Fr& x, uint32_t out[8]) { Fr c = Fr::from_mont(x); memcpy(out, c.v, 32); }
  Fr rand_fr() {
    Fr x;
    for (int i = 0; i < 8; i++) x.v[i] = rnd();
    x.v[7] &= 0x0fffffffu;   // < 2^252 < r
    return Fr::to_mont(x);
  }
  // a random multiple of the generator, or the identity one time in `inf_every`
  template <class PT, class AT>
  AT rand_point(const AT& gen, int inf_every) {
    if (inf_every && rnd() % inf_every == 0) return AT::inf();
    uint32_t k[8];
    canon(rand_fr(), k);
    return PT::from_affine(gen).mul_u32(k, 8).to_affine();
  }
  int run(const char* name) {
    const Fr zero = Fr::zero(), one = Fr::one(), minus_one = Fr::sub(Fr::zero(), Fr::one());
    const Fr special[4] = {zero, one, minus_one, zero};
    int n = 0;
    for (int it = 0; it < 48; it++) {
      // scalars: random, 0, 1, r - 1 in every combination for r and s, then random pairs
      const Fr r = it < 16 ? (it % 4 == 3 ? rand_fr() : special[it % 4]) : rand_fr();
      const Fr s = it < 16 ? ((it / 4) % 4 == 3 ? rand_fr() : special[(it / 4) % 4]) : rand_fr();
      const int inf_every = it < 24 ? 3 : 0;   // key points and MSM results include the identity
      const A1 d1 = rand_point<P1>(g1, 0), a0 = rand_point<P1>(g1, inf_every), alpha = rand_point<P1>(g1, 0);
      const A1 b1_0 = rand_point<P1>(g1, inf_every), beta = rand_point<P1>(g1, 0);
      const A2 d2 = rand_point<P2>(g2, 0), b2_0 = rand_point<P2>(g2, inf_every), beta2 = rand_point<P2>(g2, 0);
      const P1 A = P1::from_affine(rand_point<P1>(g1, inf_every)), B1 = P1::from_affine(rand_point<P1>(g1, inf_every));
      const P1 L = P1::from_affine(rand_point<P1>(g1, inf_every)), H = P1::from_affine(rand_point<P1>(g1, inf_every));
      const P2 B2 = P2::from_affine(rand_point<P2>(g2, inf_every));
      uint32_t rk[8], sk[8], rsk[8];
      canon(r, rk);
      canon(s, sk);
      canon(Fr::mul(r, s), rsk);
      // the reference: prover.rs's own order, g_c = s g_a + r g1_b - (r s) d1 + L + H
      P1 neg_rs_d1 = P1::from_affine(d1).mul_u32(rsk, 8);
      neg_rs_d1.negate();
      P1 ga0 = P1::from_affine(d1).mul_u32(rk, 8);
      ga0.madd(a0);
      ga0.madd(alpha);
      const P1 s_ga0 = ga0.mul_u32(sk, 8);
      P1 r_gb0 = P1::inf();
      if (!r.is_zero()) {
        P1 gb0 = P1::from_affine(d1).mul_u32(sk, 8);
        gb0.madd(b1_0);
        gb0.madd(beta);
        r_gb0 = gb0.mul_u32(rk, 8);
      }
      P2 gb2_0 = P2::from_affine(d2).mul_u32(sk, 8);
      gb2_0.madd(b2_0);
      gb2_0.madd(beta2);
      P1 c = A.mul_u32(sk, 8);
      if (!r.is_zero()) c.add(B1.mul_u32(rk, 8));
      c.add(L);
      c.add(H);
      P1 want_a = ga0;
      want_a.add(A);
      P2 want_b = gb2_0;
      want_b.add(B2);
      P1 want_c = s_ga0;
      want_c.add(r_gb0);
      want_c.add(neg_rs_d1);
      want_c.add(c);
      // proof_tail: the five key products as the host helpers compute them (projective) and as the GPU returns them
      // (affine), with C = s A + r B1 + L + H from above
      P1 pa = P1::from_affine(a0), pb = P1::from_affine(b1_0);
      pa.madd(alpha);
      pb.madd(beta);
      P2 p2 = P2::from_affine(b2_0);
      p2.madd(beta2);
      const A1 p_a = pa.to_affine(), p_b = pb.to_affine();
      const KeyProducts<Fq, Fq2> host{P1::from_affine(d1).mul_u32(rk, 8), P1::from_affine(d1).mul_u32(rsk, 8),
                                      P1::from_affine(p_a).mul_u32(sk, 8), P1::from_affine(p_b).mul_u32(rk, 8),
                                      P2::from_affine(d2).mul_u32(sk, 8)};
      const KeyProducts<Fq, Fq2> gpu{P1::from_affine(host.r_d1.to_affine()), P1::from_affine(host.rs_d1.to_affine()),
                                     P1::from_affine(host.s_pa.to_affine()), P1::from_affine(host.r_pb.to_affine()),
                                     P2::from_affine(host.s_d2.to_affine())};
      for (const KeyProducts<Fq, Fq2>* k : {&host, &gpu}) {
        const ProofPoints<Fq, Fq2> got = proof_tail(*k, p_a, p2.to_affine(), A, B2, c);
        CHECK(same(got.g_a, want_a) && same(got.g2_b, want_b) && same(got.g_c, want_c),
              "%s tail case %d (%s products): regrouped proof differs", name, it, k == &host ? "projective" : "affine");
      }
      n++;
    }
    return n;
  }
};

// ---- 5: the batch prover's workspace bound against what the workspaces of a group reserve ---------------------------------
// Engine::with_k0 at the geometry of a group: the automatic k0 on 132 SMs, or the explicit acc_k0
static int group_k0(const MsmGeom& g, bool g2, long long knob) {
  int k0 = msm_pick_k0(g.max_entries, 132ull * 128 * (g2 ? 2 : 3), g2 ? MSM_K0_AUTO_MIN_G2 : MSM_K0_AUTO_MIN_G1);
  if (g2 && k0 > 32) k0 = 32;
  return (knob >= 4 && knob <= 1024) ? (int)knob : k0;
}
// Engine::pick_geom
static MsmGeom resident_geom(uint64_t n, int bits, int c_knob, int ne_knob) {
  if (ne_knob <= 0) return msm_geom(n, bits, c_knob, 0);
  const int c = c_knob > 0 ? c_knob : (n >= (1u << 16) ? 16 : 0);
  int ne = ne_knob;
  MsmGeom g = msm_geom(n, bits, c, ne);
  while (g.copies > MSM_MAX_COPIES) g = msm_geom(n, bits, c, ++ne);
  return g;
}
// For a group of G proofs at every acc_k0, round count and (for a shared sorted list) every uneven pairing of round counts,
// msm_ws_bytes of the group's pass must stay within G times msm_batch_bytes_per_proof of the resident geometry.
template <class F>
static int bound_cases(const char* name, bool g2) {
  std::vector<long long> knobs = {0};
  for (long long k = 4; k <= 64; k++) knobs.push_back(k);
  for (long long k : {96, 100, 127, 128, 255, 256, 511, 512, 1000, 1023, 1024}) knobs.push_back(k);
  int n_bad = 0;
  for (uint64_t n : {(1ull << 12) - 1, (1ull << 17) - 1})
    for (int c_knob : {0, 12, 13, 14, 15, 16})
      for (int ne_knob : {0, 1, 8})
        for (int ba_m : {1, 32}) {
          MsmGeom g1 = resident_geom(n, 255, c_knob, ne_knob);
          g1.ba_m = ba_m;
          MsmRedPlan plan;
          plan.make(g1.c - 1);
          for (long long knob : knobs)
            for (bool shared : {false, true}) {
              const uint64_t per = msm_batch_bytes_per_proof<F>(g1, msm_k0_floor(g2, knob), shared);
              for (uint32_t G : {1u, 2u, 64u}) {
                MsmGeom gG = msm_geom_batch(g1, G);
                gG.k0 = group_k0(gG, g2, knob);
                for (int R = 0; R <= MSM_BA_MAX_ROUNDS; R++)
                  for (int other = 0; other <= (shared ? MSM_BA_MAX_ROUNDS : 0); other++) {
                    gG.ba = R;
                    gG.ba_pad = std::max(R, other);   // Engine::batch_geoms: one padding for the shared list
                    MsmBaPlan bap;
                    bap.make(gG);
                    const uint64_t need = msm_ws_bytes<F>(gG, bap, plan).total();
                    const bool ok = need <= per * G;
                    if (!ok && n_bad++ < 8)
                      fprintf(stderr, "%s n=%llu c=%d ne=%d ba_m=%d acc_k0=%lld shared=%d G=%u rounds=%d pad=%d: workspace %llu B > "
                              "%u x %llu B\n", name, (unsigned long long)n, g1.c, g1.ne, ba_m, knob, (int)shared, G, R, gG.ba_pad,
                              (unsigned long long)need, G, (unsigned long long)per);
                  }
              }
            }
        }
  cases++;
  if (n_bad) bad++;
  return n_bad;
}

static uint64_t read_hex() {
  unsigned long long x = 0;
  if (scanf("%llx", &x) != 1) { fprintf(stderr, "missing generator limbs on stdin\n"); exit(2); }
  return x;
}
template <class T>
static void read_point(T& p) {
  uint64_t limbs[sizeof(T) / 8];
  for (auto& l : limbs) l = read_hex();
  memcpy(&p, limbs, sizeof(T));
}

int main() {
  // 1: K proofs x ne sets, small and production-sized bucket counts
  for (int m : {5, 10, 15})
    for (int ne : {1, 2})
      for (uint32_t K : {1u, 3u, 8u}) layout_case(m, ne, K, K);
  // 2: batch 0 (MsmGeom{}) and batch 1 are the same layout and result
  for (int ne : {1, 2}) {
    const uint64_t s0 = seed;
    const std::vector<Pt> r0 = layout_case(7, ne, 1, 0);
    seed = s0;
    const std::vector<Pt> r1 = layout_case(7, ne, 1, 1);
    CHECK(same(r0[0], r1[0]), "ne=%d: batch 0 and batch 1 differ", ne);
  }
  {
    const MsmGeom a = msm_geom(4096, 255, 0, 2), b = msm_geom_batch(a, 1), z{};
    MsmGeom z3{};
    z3.ne = 3;
    CHECK(a.batch == 1 && a.sets() == (uint32_t)a.ne && b.nkeys == a.nkeys && b.max_entries == a.max_entries, "msm_geom_batch(g, 1) changed g");
    CHECK(z.sets() == 0 && z3.sets() == 3, "zero-initialised MsmGeom is not one MSM");
    const MsmGeom c = msm_geom_batch(a, 8);
    CHECK(c.sets() == 8u * a.ne && c.nkeys == 8 * a.nkeys && c.max_entries == 8 * a.max_entries && c.n == a.n,
          "msm_geom_batch(g, 8) geometry");
  }
  // 3: group size
  const uint64_t huge = 1ull << 50, GiB = 1ull << 30;
  CHECK(batch_group_size(0, 0, 1, 1, huge, 2) == 0, "count 0");
  CHECK(batch_group_size(1000, 0, 1ull << 24, 1, huge, 2) == 255, "entries cap: %u", batch_group_size(1000, 0, 1ull << 24, 1, huge, 2));
  CHECK(batch_group_size(256, 0, (1ull << 24) + 1, 1, huge, 2) == 255, "entries cap is strict (G * E < 2^32)");
  CHECK(batch_group_size(1u << 20, 0, 1, 1, huge, 2) == 65535, "grid cap");
  CHECK(batch_group_size(1000, 0, 1024, GiB, 11 * GiB, 2) == 5, "memory cap: %u", batch_group_size(1000, 0, 1024, GiB, 11 * GiB, 2));
  CHECK(batch_group_size(1000, 0, 1024, GiB, 11 * GiB, 1) == 10, "memory cap, one slot");
  CHECK(batch_group_size(1000, 0, 1024, GiB, GiB / 2, 2) == 1, "at least 1 when nothing fits");
  CHECK(batch_group_size(1000, 0, 1ull << 33, 1, huge, 2) == 1, "at least 1 past the entries cap");
  CHECK(batch_group_size(3, 0, 1024, 1, huge, 2) == 3, "at most count");
  CHECK(batch_group_size(100, 7, 1024, GiB, 11 * GiB, 2) == 7, "explicit group above the memory cap is kept");
  CHECK(batch_group_size(100, 4, 1024, 1, huge, 2) == 4, "explicit group below the automatic size is kept");
  CHECK(batch_group_size(100, 500, 1024, 1, huge, 2) == 100, "explicit group capped by count");
  CHECK(batch_group_size(1000, 900, 1ull << 24, 1, huge, 2) == 255, "explicit group capped by the 32-bit offsets");
  // 5: workspace bound, G1 and G2 points of both curves
  const int nb = bound_cases<F1>("bn254 g1", false) + bound_cases<Fp<BLS381_FqP>>("bls12_381 g1", false) +
                 bound_cases<Fp2<BN254_FqP, BN254_Params::FQ2_NONRESIDUE_NEG>>("bn254 g2", true) +
                 bound_cases<Fp2<BLS381_FqP, BLS381_Params::FQ2_NONRESIDUE_NEG>>("bls12_381 g2", true);
  // 4: tail formula
  TailCheck<BN254_FrP, BN254_FqP, BN254_Params::FQ2_NONRESIDUE_NEG> bn;
  TailCheck<BLS381_FrP, BLS381_FqP, BLS381_Params::FQ2_NONRESIDUE_NEG> bls;
  read_point(bn.g1); read_point(bn.g2); read_point(bls.g1); read_point(bls.g2);
  const int nt = bn.run("bn254") + bls.run("bls12_381");
  printf("%d checks (%d tail cases), %d mismatches\n", cases, nt, bad);
  printf("workspace bound: %d group passes over it\n", nb);
  return bad ? 1 : 0;
}
