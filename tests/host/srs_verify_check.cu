// Host-only check (built by nvcc, runs without a GPU) of the transcript check's host arithmetic in
// groth16_b200/csrc/srs.cuh:
//  * the chunk cap (srs_verify_chunk_cap): a chunk's points, scalars, mask bytes and MSM workspace fit in the free memory
//    after the margin, and the cap is close to the largest that does; it honours chunk_points, the longest member and the
//    largest stand-alone MSM (2^27 - 1, so a 2^28 transcript streams through), and is never 0.  The workspace is that of
//    the MSM geometries the engine runs (msm_ws_bytes), with and without batched-affine rounds;
//  * the chunk split (srs_chunk_len) with caps up to that MSM limit, for members up to 2^32 - 1 points;
//  * the scalars (srs_power): rho^i0 on the host, then rho^(i0 + j) per point as srs_powers_kernel forms it, against powers
//    formed one product at a time, across chunk boundaries from 0 to just below 2^32, on the four scalar fields.  Powers
//    near 2^32 are walked down from rho^(2^32) (32 squarings) by rho^-1, so they share no step with srs_power.
#include <cstdio>
#include <vector>
#include "../../groth16_b200/csrc/msm.cuh"
#include "../../groth16_b200/csrc/srs.cuh"
using namespace g16;

static int bad = 0, cases = 0;
#define CHECK(cond, ...)            \
  do {                              \
    cases++;                        \
    if (!(cond)) {                  \
      bad++;                        \
      fprintf(stderr, __VA_ARGS__); \
      fprintf(stderr, "\n");        \
    }                               \
  } while (0)

static const uint64_t MiB = 1ull << 20, GiB = 1ull << 30, MARGIN = 512 * MiB;

// the workspace of the stand-alone MSM geometry of a cnt-point chunk: window from the size, `ba` batched-affine rounds
template <class F>
static uint64_t ws_of(uint64_t cnt, int scalar_bits, int ba) {
  MsmGeom g = msm_geom(cnt, scalar_bits, 0, 0);
  g.k0 = 8;
  g.ba = g.ba_pad = ba;
  MsmBaPlan bap;
  bap.make(g);
  MsmRedPlan plan;
  plan.make(g.c - 1);
  return msm_ws_bytes<F>(g, bap, plan).total();
}

template <class WS>
static void check_cap_fits(const char* what, uint64_t chunk_points, uint64_t longest, uint64_t free_b, uint64_t per_point,
                           WS ws) {
  const uint64_t cap = srs_verify_chunk_cap(chunk_points, longest, free_b, per_point, ws);
  const uint64_t avail = free_b > MARGIN ? free_b - MARGIN : 0;
  auto need = [&](uint64_t c) { return c * per_point + (uint64_t)ws(c); };
  uint64_t limit = std::min(longest, SRS_VERIFY_MSM_MAX);
  if (chunk_points) limit = std::min(limit, chunk_points);
  limit = std::max<uint64_t>(limit, 1);
  CHECK(cap >= 1 && cap <= limit, "%s: cap %llu outside [1, %llu]", what, (unsigned long long)cap, (unsigned long long)limit);
  CHECK(cap == 1 || need(cap) <= avail, "%s: cap %llu needs %llu bytes, %llu available", what, (unsigned long long)cap,
        (unsigned long long)need(cap), (unsigned long long)avail);
  // close to the largest chunk that fits: 1 % more points would not fit (or the cap is at its limit)
  const uint64_t more = cap + cap / 100 + 1;
  CHECK(cap == limit || need(more) > avail, "%s: cap %llu, but %llu points fit too", what, (unsigned long long)cap,
        (unsigned long long)more);
}

static void check_cap() {
  // a linear workspace with a fixed part: exact values
  auto lin = [](uint64_t c) { return 100 * c + 64 * MiB; };
  const uint64_t t[][5] = {
      // chunk_points, longest, free bytes, per point -> cap
      {0, 1ull << 20, 80 * GiB, 100, 1ull << 20},                           // everything fits: one chunk
      {7, 1ull << 20, 80 * GiB, 100, 7},                                    // explicit cap
      {1ull << 22, 1000, 80 * GiB, 100, 1000},                              // never above the longest member
      {0, 1ull << 28, 1ull << 50, 100, SRS_VERIFY_MSM_MAX},                 // never above the largest MSM
      {1ull << 40, 1ull << 31, 1ull << 50, 100, SRS_VERIFY_MSM_MAX},        // an explicit cap above it
      {0, 5, 100 * MiB, 100, 1},                                            // below the margin: still one point
      {0, 0, 80 * GiB, 100, 1},                                             // nothing to do: at least 1
  };
  for (const auto& c : t) {
    const uint64_t got = srs_verify_chunk_cap(c[0], c[1], c[2], c[3], lin);
    CHECK(got == c[4], "srs_verify_chunk_cap(%llu, %llu, %llu, %llu) = %llu, want %llu", (unsigned long long)c[0],
          (unsigned long long)c[1], (unsigned long long)c[2], (unsigned long long)c[3], (unsigned long long)got,
          (unsigned long long)c[4]);
  }
  // memory-bound with the linear workspace: exactly the largest count that fits, (2 GiB - 64 MiB) / 200 points
  {
    const uint64_t got = srs_verify_chunk_cap(0, 1ull << 30, 2 * GiB + MARGIN, 100, lin);
    const uint64_t want = (2 * GiB - 64 * MiB) / 200;
    CHECK(got == want, "linear workspace: cap %llu, want %llu", (unsigned long long)got, (unsigned long long)want);
  }
}

// the engine's workspaces on one curve: the larger of the G1 and G2 geometries, rounds off and on
template <class CP>
static void check_cap_curve(const char* name) {
  using Fq = Fp<typename CP::FqP>;
  using G2F = typename CP::G2F;
  const uint64_t per_point = std::max(sizeof(Affine<Fq>), sizeof(Affine<G2F>)) + sizeof(Fp<typename CP::FrP>) + 1;
  const int bits = CP::FrP::BITS;
  for (int ba : {0, 4})
    for (uint64_t free_b : {1 * GiB, 3 * GiB, 20 * GiB, 80 * GiB})
      for (uint64_t longest : {1000ull, 1ull << 20, (1ull << 28) + 3})
        for (uint64_t chunk_points : {0ull, 1ull << 18}) {
          char what[128];
          snprintf(what, sizeof what, "%s ba %d free %llu GiB longest %llu chunk %llu", name, ba,
                   (unsigned long long)(free_b / GiB), (unsigned long long)longest, (unsigned long long)chunk_points);
          auto ws = [&](uint64_t c) { return std::max(ws_of<Fq>(c, bits, ba), ws_of<G2F>(c, bits, ba)); };
          check_cap_fits(what, chunk_points, longest, free_b, per_point, ws);
        }
}

static void check_split(uint64_t len, uint64_t cap) {
  uint64_t i0 = 0, chunks = 0;
  bool ok = true;
  while (i0 < len) {
    const uint32_t cnt = srs_chunk_len(len, i0, cap);
    if (cnt == 0 || cnt > cap || i0 + cnt > len) { ok = false; break; }
    i0 += cnt;
    chunks++;
  }
  CHECK(ok && i0 == len && chunks == (len + cap - 1) / cap, "len %llu cap %llu: chunks do not cover [0, len) exactly",
        (unsigned long long)len, (unsigned long long)cap);
}

template <class FrP>
static void check_powers(const char* name, uint64_t seed) {
  using Fr = Fp<FrP>;
  auto elem = [&]() {
    Fr a = Fr::zero();
    for (int i = 0; i + 1 < Fr::N; i++) {
      seed = seed * 6364136223846793005ull + 1442695040888963407ull;
      a.v[i] = (uint32_t)(seed >> 32);
    }
    return a;
  };
  const Fr rho = elem(), one = Fr::one();
  Fr tab[32];
  tab[0] = rho;
  for (int k = 1; k < 32; k++) tab[k] = Fr::sqr(tab[k - 1]);
  // from 0, chunks of 1, 7, 128 and 1000 points: point i0 + j of a chunk gets rho^(i0 + j)
  const uint64_t n = 4096;
  std::vector<Fr> seq(n);
  seq[0] = one;
  for (uint64_t i = 1; i < n; i++) seq[i] = Fr::mul(seq[i - 1], rho);
  for (uint64_t cap : {1ull, 7ull, 128ull, 1000ull}) {
    int wrong = 0;
    for (uint64_t i0 = 0; i0 < n; i0 += srs_chunk_len(n, i0, cap)) {
      const Fr c = srs_power(one, tab, i0);
      for (uint64_t j = 0; j < srs_chunk_len(n, i0, cap); j++) wrong += srs_power(c, tab, j) != seq[i0 + j];
    }
    CHECK(wrong == 0, "%s: %d of the first %llu scalars wrong with chunks of %llu", name, wrong, (unsigned long long)n,
          (unsigned long long)cap);
  }
  // near 2^32: rho^(2^32 - m + k), walked down from rho^(2^32); chunk starts on both sides of every boundary there
  Fr top = rho;
  for (int k = 0; k < 32; k++) top = Fr::sqr(top);
  const Fr rinv = Fr::inv(rho);
  const uint64_t m = 3000, base = (1ull << 32) - m, len = 0xffffffffull;
  std::vector<Fr> hi(m);
  Fr cur = top;
  for (uint64_t k = m; k-- > 0;) { cur = Fr::mul(cur, rinv); hi[k] = cur; }
  for (uint64_t cap : {7ull, 1000ull, 1ull << 18, (unsigned long long)SRS_VERIFY_MSM_MAX}) {
    int wrong = 0;
    for (uint64_t i0 = base / cap * cap; i0 < len; i0 += srs_chunk_len(len, i0, cap)) {
      const Fr c = srs_power(one, tab, i0);
      const uint64_t cnt = srs_chunk_len(len, i0, cap);
      for (uint64_t j = (i0 >= base ? 0 : base - i0); j < cnt; j++) wrong += srs_power(c, tab, j) != hi[i0 + j - base];
    }
    CHECK(wrong == 0, "%s: %d scalars near 2^32 wrong with chunks of %llu", name, wrong, (unsigned long long)cap);
  }
  // the host's rho^(N - 1) of the last point (lo) and rho^-1 (hi) for the longest member
  CHECK(srs_power(one, tab, len - 1) == hi[m - 2], "%s: rho^(2^32 - 2) wrong", name);
  CHECK(Fr::mul(srs_power(one, tab, len - 1), rho) == Fr::mul(top, rinv), "%s: rho^(2^32 - 1) wrong", name);
}

int main() {
  check_cap();
  check_cap_curve<BN254_Params>("bn254");
  check_cap_curve<BLS381_Params>("bls12_381");
  check_cap_curve<BW6_Params>("bw6_761");
  for (uint64_t len : {1ull, 2ull, 7ull, 1000ull, 65536ull, (1ull << 28), (1ull << 28) + 1, 0xffffffffull})
    for (uint64_t cap : {1000ull, 1ull << 18, (unsigned long long)SRS_VERIFY_MSM_MAX}) check_split(len, cap);
  check_powers<BLS381_FrP>("bls12_381", 11);
  check_powers<BN254_FrP>("bn254", 12);
  check_powers<BLS377_FrP>("bls12_377", 13);
  check_powers<BW6_FrP>("bw6_761", 14);
  printf("srs verify: %d checks, %d mismatches\n", cases, bad);
  return bad ? 1 : 0;
}
