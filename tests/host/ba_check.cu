// Host-only check (built by nvcc, runs without a GPU) of the batched-affine rounds of groth16_b200/csrc/msm_ba.cuh:
// ba_forward / ba_combine / ba_backward are executed "thread by thread" on the CPU over random bucketed entry lists in
// the padded regular layout (signs, repeated bases -> tangent case, P and -P -> identity, identities among the bases,
// empty and one-entry buckets, padding slots), round after round, and every bucket of the final list must sum to the
// plain XYZZ sum of its entries.
// Also: the MsmBaPlan bounds hold for the lengths seen.  The curve only enters through a = 0, so for Fq2 an arbitrary
// (x, y) serves as generator of "its" curve y^2 = x^3 + b.
#include <cstdio>
#include <vector>
#include "../../groth16_b200/csrc/msm.cuh"
using namespace g16;

static uint64_t seed = 777;
static uint32_t rnd() { seed = seed * 6364136223846793005ull + 1442695040888963407ull; return (uint32_t)(seed >> 33); }

template <class F>
static bool same_pt(const XYZZ<F>& a, const XYZZ<F>& b) {
  if (a.is_inf() || b.is_inf()) return a.is_inf() && b.is_inf();
  Affine<F> x = a.to_affine(), y = b.to_affine();
  return x.x == y.x && x.y == y.y;
}

template <class F>
static int run_case(const Affine<F>& G, uint32_t nkeys, uint32_t nbase, uint32_t avg, int R, uint32_t m, uint32_t Gc, const char* name, uint32_t gcd = 0) {
  int bad = 0;
  // base table: k * G, a few identities
  std::vector<Affine<F>> bases(nbase);
  XYZZ<F> acc = XYZZ<F>::inf();
  for (uint32_t i = 0; i < nbase; i++) {
    acc.madd(G);
    bases[i] = (i % 11 == 7) ? Affine<F>::inf() : acc.to_affine();
  }
  // sorted slots, every bucket padded to a multiple of 2^R (what msm_scan_blocks + msm_pad_fill produce on the device)
  const uint32_t pad = (1u << R) - 1;
  std::vector<uint32_t> off(nkeys + 1, 0), cnt(nkeys, 0), sidx, skey;
  uint64_t real_entries = 0;
  for (uint32_t b = 0; b < nkeys; b++) {
    uint32_t c = rnd() % (2 * avg + 1);
    if (b % 7 == 3) c = 0;
    if (b % 7 == 5) c = 1;
    cnt[b] = c;
    real_entries += c;
    off[b] = (uint32_t)sidx.size();
    for (uint32_t e = 0; e < c; e++) {
      uint32_t ix = rnd() % nbase;
      uint32_t sg = rnd() & 1;
      if (e > 0 && rnd() % 5 == 0) {           // repeat the previous entry: same point or its negative
        ix = sidx.back() & 0x7fffffffu;
        sg = (rnd() & 1) ? (sidx.back() >> 31) : 1 - (sidx.back() >> 31);
      }
      sidx.push_back(ix | (sg << 31));
      skey.push_back(b);
    }
    for (uint32_t e = c; e < ((c + pad) & ~pad); e++) { sidx.push_back(BA_EMPTY); skey.push_back(b); }
  }
  off[nkeys] = (uint32_t)sidx.size();
  uint32_t total0 = (uint32_t)sidx.size();
  // reference bucket sums
  std::vector<XYZZ<F>> want(nkeys, XYZZ<F>::inf());
  for (uint32_t b = 0; b < nkeys; b++)
    for (uint32_t e = off[b]; e < off[b] + cnt[b]; e++) want[b].madd(bases[sidx[e] & 0x7fffffffu], (sidx[e] >> 31) != 0);
  // plan bounds
  MsmGeom g{};
  g.nkeys = nkeys; g.max_entries = real_entries; g.k0 = 64; g.ba = R; g.ba_m = (int)m; g.ba_G = (int)Gc; g.ba_gcd = (int)gcd;
  MsmBaPlan bp;
  bp.make(g);
  if (total0 > bp.len[0] || (total0 & pad)) { bad++; fprintf(stderr, "%s: padded length %u violates the plan bound %llu\n", name, total0, (unsigned long long)bp.len[0]); }
  const uint64_t len1 = bp.len[1] + 1;
  std::vector<F> pre(len1), prod(len1), pre2(len1);
  std::vector<Affine<F>> lists[2] = {std::vector<Affine<F>>(len1), std::vector<Affine<F>>(len1)};
  for (int r = 0; r < R; r++) {
    BaRound<F> a;
    a.in = r == 0 ? bases.data() : lists[(r - 1) & 1].data();
    a.sidx = r == 0 ? sidx.data() : nullptr;
    a.total0 = &total0;
    a.shift = (uint32_t)(r + 1);
    a.m = m; a.G = Gc; a.inv_gcd = gcd;   // (the plan may pick a smaller m for short lists; any m must work)
    a.pre = pre.data(); a.prod = prod.data(); a.pre2 = pre2.data();
    a.out = lists[r & 1].data();
    const uint64_t Tmax = ba_threads(bp.len[r + 1], m) + 3;   // over-launch like the kernels do
    for (uint64_t t = 0; t < Tmax; t++) ba_forward<F>(a, t);
    for (uint64_t l = 0; l < (Tmax + Gc - 1) / Gc + 2; l++) ba_combine<F>(a, l);
    for (uint64_t t = 0; t < Tmax; t++) ba_backward<F>(a, t);
  }
  // last list: slot j belongs to the bucket of sorted slot j << R (the key msm_accum_l0 reads)
  const std::vector<Affine<F>>& fin = lists[(R - 1) & 1];
  std::vector<XYZZ<F>> got(nkeys, XYZZ<F>::inf());
  for (uint32_t j = 0; j < (total0 >> R); j++) got[skey[(size_t)j << R]].madd(fin[j]);
  for (uint32_t b = 0; b < nkeys; b++)
    if (!same_pt(got[b], want[b])) { bad++; fprintf(stderr, "%s: bucket %u mismatch (count %u)\n", name, b, cnt[b]); }
  return bad;
}

static Fp<BN254_FqP> fq_small(uint32_t x) {
  Fp<BN254_FqP> r = Fp<BN254_FqP>::zero();
  r.v[0] = x;
  return Fp<BN254_FqP>::to_mont(r);
}

int main() {
  int bad = 0, cases = 0;
  {
    using F = Fp<BN254_FqP>;
    const Affine<F> G{fq_small(1), fq_small(2)};
    for (int R : {1, 2, 3, 5}) {
      bad += run_case<F>(G, 37, 50, 12, R, 4, 3, "bn254-g1"); cases++;
      bad += run_case<F>(G, 5, 3, 40, R, 8, 64, "bn254-g1-dense"); cases++;
    }
    bad += run_case<F>(G, 1, 9, 100, 6, 32, 64, "bn254-g1-onebucket"); cases++;
    bad += run_case<F>(G, 37, 50, 12, 3, 4, 3, "bn254-g1-safegcd", 1); cases++;
    bad += run_case<F>(G, 5, 3, 40, 5, 8, 64, "bn254-g1-dense-safegcd", 1); cases++;
    bad += run_case<F>(G, 64, 200, 3, 4, 16, 64, "bn254-g1-sparse-R4", 1); cases++;
  }
  {
    using B = Fp<BLS381_FqP>;
    using F = Fp2<BLS381_FqP, 1>;
    auto small = [](uint32_t x) { B r = B::zero(); r.v[0] = x; return B::to_mont(r); };
    const Affine<F> G{{small(3), small(5)}, {small(7), small(11)}};
    bad += run_case<F>(G, 19, 20, 6, 2, 4, 5, "bls381-g2"); cases++;
    bad += run_case<F>(G, 3, 4, 20, 3, 16, 64, "bls381-g2-dense"); cases++;
    bad += run_case<F>(G, 19, 20, 6, 2, 4, 5, "bls381-g2-safegcd", 1); cases++;
    bad += run_case<F>(G, 19, 20, 6, 4, 4, 5, "bls381-g2-R4", 1); cases++;
  }
  {
    using B = Fp<BLS377_FqP>;
    using F = Fp2<BLS377_FqP, 5>;
    auto small = [](uint32_t x) { B r = B::zero(); r.v[0] = x; return B::to_mont(r); };
    const Affine<F> G{{small(2), small(9)}, {small(4), small(1)}};
    bad += run_case<F>(G, 7, 6, 10, 2, 4, 2, "bls377-g2"); cases++;
    bad += run_case<F>(G, 7, 6, 10, 3, 2, 2, "bls377-g2-R3", 1); cases++;
  }
  printf("%d cases, %d mismatches\n", cases, bad);
  return bad ? 1 : 0;
}
