// Host-only check (built by nvcc, runs without a GPU) of the host arithmetic g16_pk_contribute relies on in
// groth16_b200/csrc/srs.cuh:
//  * the chunk split of h_query and l_query under one cap (srs_chunk_len, srs_chunk_cap with the G1 affine point size of
//    each curve): the chunks of both members cover every index once and in order, none is empty or longer than the cap,
//    for lengths up to 2^32 - 1 and caps up to 2^32 - 1; the byte offset of every chunk start fits in 64 bits;
//  * the range rule (srs_overlap): ranges that share a byte overlap, touching or empty ranges do not, near the top of the
//    address space too.
#include <cstdio>
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

// both members with one cap, as the call walks them: h_query then l_query
static void check_members(uint64_t h_len, uint64_t l_len, uint64_t cap, uint64_t esz) {
  for (uint64_t len : {h_len, l_len}) {
    uint64_t i0 = 0, chunks = 0, last_off = 0;
    bool ok = true;
    while (i0 < len) {
      const uint32_t cnt = srs_chunk_len(len, i0, cap);
      if (cnt == 0 || cnt > cap || i0 + cnt > len) { ok = false; break; }
      last_off = i0 * esz;   // byte offset of the chunk in the host array
      if (last_off / esz != i0) { ok = false; break; }
      i0 += cnt;
      chunks++;
    }
    CHECK(ok && i0 == len, "len %llu cap %llu: chunks do not cover [0, len)", (unsigned long long)len, (unsigned long long)cap);
    CHECK(chunks == (len + cap - 1) / cap, "len %llu cap %llu: %llu chunks", (unsigned long long)len, (unsigned long long)cap,
          (unsigned long long)chunks);
  }
}

static void check_caps() {
  const unsigned long long GiB = 1ull << 30, M32 = 0xffffffffull;
  const uint64_t esz[] = {64, 96, 96, 192};   // G1 affine bytes: BN254, BLS12-381, BLS12-377, BW6-761
  for (uint64_t e : esz) {
    // (chunk_points, longest of h_query / l_query, free bytes) -> cap
    const uint64_t want_mem = (40 * GiB) / e;
    const uint64_t t[][4] = {
        {0, (1ull << 20) - 1, 80 * GiB, (1ull << 20) - 1},
        {7, (1ull << 20) - 1, 80 * GiB, 7},
        {0, M32, 40 * GiB + (512ull << 20), std::min<uint64_t>(want_mem, M32)},
        {1ull << 22, M32, 80 * GiB, 1ull << 22},
        {0, M32, 1ull << 50, M32},
        {0, 0, 80 * GiB, 1},
    };
    for (const auto& c : t) {
      const uint64_t got = srs_chunk_cap(c[0], c[1], c[2], e);
      CHECK(got == c[3], "esz %llu: srs_chunk_cap(%llu, %llu, %llu) = %llu, want %llu", (unsigned long long)e,
            (unsigned long long)c[0], (unsigned long long)c[1], (unsigned long long)c[2], (unsigned long long)got,
            (unsigned long long)c[3]);
    }
    for (uint64_t h : {0ull, 1ull, 1000ull, (1ull << 31) + 1, M32 - 1, M32})
      for (uint64_t l : {0ull, 7ull, M32})
        for (uint64_t cap : {1ull << 22, (1ull << 31) - 1, 1ull << 31, M32}) check_members(h, l, cap, e);
  }
  for (uint64_t cap : {1ull, 7ull, 128ull}) check_members(1000, 4097, cap, 64);
}

static void check_overlap() {
  const uintptr_t top = ~(uintptr_t)0 - 4095;
  struct { uintptr_t a; uint64_t na; uintptr_t b; uint64_t nb; bool want; } t[] = {
      {4096, 64, 4096, 64, true},          // the same range
      {4096, 64, 4160, 64, false},         // touching
      {4096, 65, 4160, 64, true},          // one byte shared
      {4160, 64, 4096, 65, true},
      {4096, 0, 4096, 64, false},          // an empty range shares nothing
      {4096, 64, 4100, 0, false},
      {4096, 1 << 20, 8192, 64, true},     // contained
      {top, 4095, top + 4000, 64, true},   // near the top of the address space
      {top, 4000, top + 4000, 64, false},
  };
  for (const auto& c : t)
    CHECK(srs_overlap(c.a, c.na, c.b, c.nb) == c.want, "srs_overlap(%#zx, %llu, %#zx, %llu) != %d", (size_t)c.a,
          (unsigned long long)c.na, (size_t)c.b, (unsigned long long)c.nb, (int)c.want);
}

int main() {
  check_caps();
  check_overlap();
  printf("pk contribute: %d checks, %d mismatches\n", cases, bad);
  return bad ? 1 : 0;
}
