// Host-only check (built by nvcc, runs without a GPU) of the phase-1 contribution's host arithmetic in
// groth16_b200/csrc/srs.cuh:
//  * the chunk split (srs_chunk_len, srs_chunk_cap): chunks cover every index of a member once and in order, none is empty
//    or longer than the cap, for lengths up to 2^32 - 1; the cap honours chunk_points, the free memory, the longest member
//    and 2^32 - 1, and is never 0;
//  * the power scheme (srs_power): c = x tau^i0 on the host, then c tau^j per point as the kernel forms it, against powers
//    formed one product at a time, on the four scalar fields, for chunk starts from 0 to just below 2^32.  Powers near 2^32
//    are walked from tau^(2^32) (32 squarings) down by tau^-1, so they share no step with srs_power.
#include <cstdio>
#include <vector>
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

static void check_split(uint64_t len, uint64_t cap) {
  uint64_t i0 = 0, chunks = 0;
  bool ok = true;
  while (i0 < len) {
    const uint32_t cnt = srs_chunk_len(len, i0, cap);
    if (cnt == 0 || cnt > cap || i0 + cnt > len) { ok = false; break; }
    i0 += cnt;   // the next chunk starts right after this one: every index once, in order
    chunks++;
  }
  CHECK(ok && i0 == len, "len %llu cap %llu: chunks do not cover [0, len) exactly", (unsigned long long)len,
        (unsigned long long)cap);
  CHECK(chunks == (len + cap - 1) / cap, "len %llu cap %llu: %llu chunks", (unsigned long long)len, (unsigned long long)cap,
        (unsigned long long)chunks);
}

static void check_cap() {
  const uint64_t MiB = 1ull << 20, GiB = 1ull << 30, M32 = 0xffffffffull;
  // (chunk_points, longest, free bytes, point bytes) -> cap
  const uint64_t t[][5] = {
      {0, 1ull << 21, 80 * GiB, 64, 1ull << 21},            // everything fits: one chunk
      {7, 1ull << 21, 80 * GiB, 64, 7},                      // explicit cap
      {1ull << 22, 1000, 80 * GiB, 64, 1000},                // never above the longest member
      {0, 1ull << 31, 8 * GiB + 512 * MiB, 128, (8 * GiB) / 128},   // free memory after the margin
      {1ull << 40, 1ull << 31, 8 * GiB + 512 * MiB, 128, (8 * GiB) / 128},   // an explicit cap above the memory
      {0, M32, 1ull << 45, 64, M32},                         // at most 2^32 - 1
      {0, 5, 100 * MiB, 64, 1},                              // below the margin: still one point per chunk
      {0, 0, 80 * GiB, 64, 1},                               // nothing to do: at least 1
  };
  for (const auto& c : t) {
    const uint64_t got = srs_chunk_cap(c[0], c[1], c[2], c[3]);
    CHECK(got == c[4], "srs_chunk_cap(%llu, %llu, %llu, %llu) = %llu, want %llu", (unsigned long long)c[0],
          (unsigned long long)c[1], (unsigned long long)c[2], (unsigned long long)c[3], (unsigned long long)got,
          (unsigned long long)c[4]);
  }
}

template <class FrP>
static void check_powers(const char* name, uint64_t seed) {
  using Fr = Fp<FrP>;
  auto elem = [&]() {   // a Montgomery element below r: random low limbs, top limb 0
    Fr a = Fr::zero();
    for (int i = 0; i + 1 < Fr::N; i++) {
      seed = seed * 6364136223846793005ull + 1442695040888963407ull;
      a.v[i] = (uint32_t)(seed >> 32);
    }
    return a;
  };
  const Fr tau = elem(), x = elem();
  Fr tab[32];
  tab[0] = tau;
  for (int k = 1; k < 32; k++) tab[k] = Fr::sqr(tab[k - 1]);
  // starts from 0, with chunks of 1, 7 and 128 points: point i0 + j of a chunk is x tau^(i0 + j)
  const uint64_t n = 4096;
  std::vector<Fr> seq(n);
  seq[0] = x;
  for (uint64_t i = 1; i < n; i++) seq[i] = Fr::mul(seq[i - 1], tau);
  for (uint64_t cap : {1ull, 7ull, 128ull}) {
    int wrong = 0;
    for (uint64_t i0 = 0; i0 < n; i0 += srs_chunk_len(n, i0, cap)) {
      const Fr c = srs_power(x, tab, i0);
      for (uint64_t j = 0; j < srs_chunk_len(n, i0, cap); j++) wrong += srs_power(c, tab, j) != seq[i0 + j];
    }
    CHECK(wrong == 0, "%s: %d of the first %llu powers wrong with chunks of %llu", name, wrong, (unsigned long long)n,
          (unsigned long long)cap);
  }
  // starts near 2^32: x tau^(2^32 - 1 - k), k < m, walked down from x tau^(2^32)
  Fr top = tau;
  for (int k = 0; k < 32; k++) top = Fr::sqr(top);
  const Fr tinv = Fr::inv(tau);
  const uint64_t m = 3000;
  std::vector<Fr> hi(m);   // hi[k] = x tau^(2^32 - m + k)
  Fr cur = Fr::mul(x, top);
  for (uint64_t k = m; k-- > 0;) { cur = Fr::mul(cur, tinv); hi[k] = cur; }
  const uint64_t base = (1ull << 32) - m;
  for (uint64_t cap : {1ull, 7ull, 128ull, 1000ull}) {
    int wrong = 0;
    // a member of length 2^32 - 1 split from 0 with this cap: check the chunks whose points lie in [base, 2^32 - 1)
    const uint64_t len = 0xffffffffull;
    for (uint64_t i0 = base / cap * cap; i0 < len; i0 += srs_chunk_len(len, i0, cap)) {
      const Fr c = srs_power(x, tab, i0);
      for (uint64_t j = 0; j < srs_chunk_len(len, i0, cap); j++)
        if (i0 + j >= base) wrong += srs_power(c, tab, j) != hi[i0 + j - base];
    }
    CHECK(wrong == 0, "%s: %d powers near 2^32 wrong with chunks of %llu", name, wrong, (unsigned long long)cap);
  }
  // one chunk of 2^32 - 1 points: j itself runs to 2^32 - 2
  int wrong = 0;
  for (uint64_t k = 0; k + 1 < m; k++) wrong += srs_power(x, tab, base + k) != hi[k];
  CHECK(wrong == 0, "%s: %d in-chunk powers near 2^32 wrong", name, wrong);
}

int main() {
  const unsigned long long M32 = 0xffffffffull;
  for (uint64_t len : {0ull, 1ull, 2ull, 3ull, 7ull, 1000ull, 4097ull, 65536ull})
    for (uint64_t cap : {1ull, 2ull, 7ull, 128ull, 1000ull, 4096ull, M32}) check_split(len, cap);
  for (uint64_t len : {(1ull << 24) + 5, (1ull << 31) + 1, M32 - 1, M32})
    for (uint64_t cap : {1000ull, 1ull << 22, (1ull << 31) - 1, 1ull << 31, M32}) check_split(len, cap);
  check_cap();
  check_powers<BLS381_FrP>("bls12_381", 1);
  check_powers<BN254_FrP>("bn254", 2);
  check_powers<BLS377_FrP>("bls12_377", 3);
  check_powers<BW6_FrP>("bw6_761", 4);
  printf("srs contribute: %d checks, %d mismatches\n", cases, bad);
  return bad ? 1 : 0;
}
