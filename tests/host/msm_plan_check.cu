// Host-only check (built by nvcc, runs without a GPU) of the bucket-reduction plan of groth16_b200/csrc/msm.cuh:
// MsmRedPlan (tree of row / column sums), the array layout msm_enqueue uses, and the host recombination
// MsmHostRed::T / msm_finish, against the definition  sum_e 2^(c e) * sum_b (b + 1) * bucket[e][b].
// The device kernel msm_sum_strided is replaced here by a literal host evaluation of the same sums.
#include <cstdio>
#include <utility>
#include <vector>
#include "../../groth16_b200/csrc/msm.cuh"
using namespace g16;
using F = Fp<BN254_FqP>;
using Pt = XYZZ<F>;

static F fp_small(uint32_t x) {
  F r = F::zero();
  r.v[0] = x;
  return F::to_mont(r);
}
static bool same(const Pt& a, const Pt& b) {
  Affine<F> x = a.to_affine(), y = b.to_affine();
  return x.x == y.x && x.y == y.y;
}

int main() {
  const Affine<F> G{fp_small(1), fp_small(2)};   // BN254 G1 generator
  Pt mult[8];
  mult[0] = Pt::inf();
  for (int i = 1; i < 8; i++) { mult[i] = mult[i - 1]; mult[i].madd(G); }
  uint64_t seed = 12345;
  auto rnd = [&]() { seed = seed * 6364136223846793005ull + 1442695040888963407ull; return (uint32_t)(seed >> 40); };
  int bad = 0, cases = 0;
  // up to the production shape: 2^15 buckets per window, 1 .. 16 effective windows (the bucket sets of bench.py's plans)
  const std::vector<std::pair<int, std::vector<int>>> shapes = {{2, {1, 3}}, {3, {1, 3}}, {5, {1, 3}}, {6, {1, 3}}, {7, {1, 3}},
                                                                {8, {1, 3}}, {10, {1, 3}}, {11, {1, 3}}, {13, {1, 3}},
                                                                {14, {1, 2, 8, 16}}, {15, {1, 2, 8, 16}}};
  for (const auto& shape : shapes) {
    const int m = shape.first;
    for (int ne : shape.second) {
      cases++;
      const int c = m + 1;
      MsmGeom g{};
      g.n = 1; g.c = c; g.ne = ne; g.W = ne; g.copies = 1; g.B = 1u << m; g.nkeys = g.B * ne; g.max_entries = 1; g.k0 = 64;
      MsmWorkspace<F> ws;
      ws.plan.make(m);
      const MsmRedPlan& pl = ws.plan;
      const size_t B = g.B;
      std::vector<Pt> buckets(B * ne), inner(pl.inner_pts * ne + 1), leaf(pl.leaf_pts * ne + 1);
      std::vector<uint64_t> weight(ne, 0);   // sum (b+1) s_b per window (fits: B <= 2^15, s <= 7: < 7 * 2^29)
      for (int w = 0; w < ne; w++)
        for (size_t b = 0; b < B; b++) {
          const uint32_t s = (rnd() % 3 == 0) ? 0 : rnd() % 8;
          buckets[w * B + b] = mult[s];
          weight[w] += (uint64_t)(b + 1) * s;
        }
      auto arr = [&](int id) -> Pt* {
        if (id == 0) return buckets.data();
        const MsmRedNode& nd = pl.nodes[id];
        return (nd.leaf ? leaf.data() : inner.data()) + nd.off * ne;
      };
      for (int id = 0; id < pl.n_nodes; id++) {   // what the msm_sum_strided jobs compute
        const MsmRedNode& nd = pl.nodes[id];
        if (nd.leaf) continue;
        const size_t len = (size_t)1 << nd.log_len, a0 = (size_t)1 << nd.a0, a1 = (size_t)1 << nd.a1;
        for (int w = 0; w < ne; w++) {
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
      // per window
      for (int w = 0; w < ne; w++) {
        MsmHostRed<F> hr{ws, g, w};
        Pt tot;
        Pt got = hr.T(0, tot);
        uint32_t k[2] = {(uint32_t)weight[w], (uint32_t)(weight[w] >> 32)};
        Pt want = Pt::from_affine(G).mul_u32(k, 2);
        if (!same(got, want)) { bad++; fprintf(stderr, "m=%d ne=%d window %d: weighted sum mismatch\n", m, ne, w); }
      }
      // Horner over the effective windows
      Pt fin = msm_finish<F>(ws, g);
      Pt want = Pt::inf();
      for (int w = ne - 1; w >= 0; w--) {
        for (int i = 0; i < c; i++) want.dbl_inplace();
        uint32_t k[2] = {(uint32_t)weight[w], (uint32_t)(weight[w] >> 32)};
        want.add(Pt::from_affine(G).mul_u32(k, 2));
      }
      if (!same(fin, want)) { bad++; fprintf(stderr, "m=%d ne=%d: msm_finish mismatch\n", m, ne); }
      ws.h_leaf = nullptr;
    }
  }
  // geometry helpers
  // c = 16 at 2^20 pairs for every bucket-set count of bench.py's residency plans (and a ragged one), all three scalar widths
  for (int bits : {255, 254, 253})
    for (int ne : {1, 2, 3, 4, 8, 16}) {
      const MsmGeom g = msm_geom(1u << 20, bits, 16, ne);
      if (!(g.c == 16 && g.W == 16 && g.ne == ne && g.copies == (16 + ne - 1) / ne && g.B == 32768 && g.nkeys == 32768u * ne &&
            g.max_entries == (16ull << 20))) {
        bad++;
        fprintf(stderr, "geom c=16 bits=%d ne=%d mismatch\n", bits, ne);
      }
    }
  MsmGeom g3 = msm_geom(17, 254, 0, 0);
  if (!(g3.c == 3 && g3.ne == g3.W && g3.copies == 1 && g3.W == 85)) { bad++; fprintf(stderr, "geom small mismatch\n"); }
  if (msm_pick_k0(16u << 20, 56832, 8) != 64 || msm_pick_k0(2u << 20, 56832, 8) != 16 || msm_level_threads(2048, 4) != 512) { bad++; fprintf(stderr, "k0 / level mismatch\n"); }
  printf("%d cases, %d mismatches\n", cases, bad);
  return bad ? 1 : 0;
}
