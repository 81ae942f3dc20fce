// fp.cuh -- prime-field arithmetic in Montgomery form, 32-bit limbs, for sm_90a.
//
// Replaces ark-ff 0.5.0 `Fp<MontBackend<_,N>,N>` (un-vendored dependency of /root/reference; used at
// prover.rs:64,71,82 `into_bigint`, r1cs_to_qap.rs:28-67,201-232 and inside every curve operation).  The memory
// image is identical to ark's: little-endian limbs of a*R mod p with R = 2^(64*N64).
//
// Three back-ends behind one interface:
//   * __CUDA_ARCH__       : straight-line PTX carry chains (mad.lo.cc / madc.hi.cc), even/odd-column
//                           Montgomery multiplication so that ptxas can pair lo/hi into IMAD.WIDE.
//   * G16_EMULATE_PTX     : the very same algorithm with the PTX carry primitives emulated in C
//                           (host unit test of the carry-chain logic without a GPU).
//   * plain host          : 64-bit-limb CIOS with unsigned __int128 (host-side final assembly, prover.rs:76-131).
#pragma once
#include <cstdint>
#include <cstring>
#include "g16_constants.h"

namespace g16 {

// ------------------------------------------------------------------------------------------------
// carry-chain primitives
// ------------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
#define G16_PTX_PATH 1
namespace ptx {
__device__ __forceinline__ void add_cc(uint32_t& r, uint32_t a, uint32_t b) { asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); }
__device__ __forceinline__ void addc_cc(uint32_t& r, uint32_t a, uint32_t b) { asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); }
__device__ __forceinline__ void addc(uint32_t& r, uint32_t a, uint32_t b) { asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); }
__device__ __forceinline__ void sub_cc(uint32_t& r, uint32_t a, uint32_t b) { asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); }
__device__ __forceinline__ void subc_cc(uint32_t& r, uint32_t a, uint32_t b) { asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); }
__device__ __forceinline__ void subc(uint32_t& r, uint32_t a, uint32_t b) { asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); }
__device__ __forceinline__ void mul_lo(uint32_t& r, uint32_t a, uint32_t b) { asm volatile("mul.lo.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); }
__device__ __forceinline__ void mul_hi(uint32_t& r, uint32_t a, uint32_t b) { asm volatile("mul.hi.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); }
__device__ __forceinline__ void mad_lo_cc(uint32_t& r, uint32_t a, uint32_t b, uint32_t c) { asm volatile("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); }
__device__ __forceinline__ void madc_lo_cc(uint32_t& r, uint32_t a, uint32_t b, uint32_t c) { asm volatile("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); }
__device__ __forceinline__ void madc_hi_cc(uint32_t& r, uint32_t a, uint32_t b, uint32_t c) { asm volatile("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); }
__device__ __forceinline__ void madc_hi(uint32_t& r, uint32_t a, uint32_t b, uint32_t c) { asm volatile("madc.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); }
}  // namespace ptx
#elif defined(G16_EMULATE_PTX)
#define G16_PTX_PATH 1
namespace ptx {
static thread_local uint32_t CF = 0;
inline void add_cc(uint32_t& r, uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b; r = (uint32_t)t; CF = (uint32_t)(t >> 32); }
inline void addc_cc(uint32_t& r, uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b + CF; r = (uint32_t)t; CF = (uint32_t)(t >> 32); }
inline void addc(uint32_t& r, uint32_t a, uint32_t b) { r = a + b + CF; }
inline void sub_cc(uint32_t& r, uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b; r = (uint32_t)t; CF = (uint32_t)(t >> 63); }
inline void subc_cc(uint32_t& r, uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b - CF; r = (uint32_t)t; CF = (uint32_t)(t >> 63); }
inline void subc(uint32_t& r, uint32_t a, uint32_t b) { r = a - b - CF; }
inline void mul_lo(uint32_t& r, uint32_t a, uint32_t b) { r = a * b; }
inline void mul_hi(uint32_t& r, uint32_t a, uint32_t b) { r = (uint32_t)(((uint64_t)a * b) >> 32); }
inline void mad_lo_cc(uint32_t& r, uint32_t a, uint32_t b, uint32_t c) { uint64_t t = (uint64_t)(uint32_t)(a * b) + c; r = (uint32_t)t; CF = (uint32_t)(t >> 32); }
inline void madc_lo_cc(uint32_t& r, uint32_t a, uint32_t b, uint32_t c) { uint64_t t = (uint64_t)(uint32_t)(a * b) + c + CF; r = (uint32_t)t; CF = (uint32_t)(t >> 32); }
inline void madc_hi_cc(uint32_t& r, uint32_t a, uint32_t b, uint32_t c) { uint64_t t = (((uint64_t)a * b) >> 32) + c + CF; r = (uint32_t)t; CF = (uint32_t)(t >> 32); }
inline void madc_hi(uint32_t& r, uint32_t a, uint32_t b, uint32_t c) { r = (uint32_t)(((uint64_t)a * b) >> 32) + c + CF; }
}  // namespace ptx
#endif

// ------------------------------------------------------------------------------------------------
// Fp<P>: P supplies N, INV32, mod(i), one(i), r2(i)
// ------------------------------------------------------------------------------------------------
template <class P>
struct alignas(16) Fp {
  static constexpr int N = P::N;
  using Params = P;
  uint32_t v[N];

  G16_HD static Fp zero() {
    Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.v[i] = 0;
    return r;
  }
  G16_HD static Fp one() {
    Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.v[i] = P::one(i);
    return r;
  }
  G16_HD static Fp r2() {
    Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.v[i] = P::r2(i);
    return r;
  }
  G16_HD static Fp modulus() {
    Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.v[i] = P::mod(i);
    return r;
  }
  G16_HD bool is_zero() const {
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < N; i++) acc |= v[i];
    return acc == 0;
  }
  G16_HD bool operator==(const Fp& o) const {
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < N; i++) acc |= v[i] ^ o.v[i];
    return acc == 0;
  }
  G16_HD bool operator!=(const Fp& o) const { return !(*this == o); }

  // ---------------- add / sub / neg ----------------
  G16_HD static Fp add(const Fp& a, const Fp& b) {
    Fp t, u;
#ifdef G16_PTX_PATH
    ptx::add_cc(t.v[0], a.v[0], b.v[0]);
#pragma unroll
    for (int i = 1; i < N - 1; i++) ptx::addc_cc(t.v[i], a.v[i], b.v[i]);
    ptx::addc(t.v[N - 1], a.v[N - 1], b.v[N - 1]);  // 2p < 2^(32N): no carry out
    ptx::sub_cc(u.v[0], t.v[0], P::mod(0));
#pragma unroll
    for (int i = 1; i < N; i++) ptx::subc_cc(u.v[i], t.v[i], P::mod(i));
    uint32_t br;
    ptx::subc(br, 0, 0);  // 0xffffffff iff t < p
#pragma unroll
    for (int i = 0; i < N; i++) t.v[i] = br ? t.v[i] : u.v[i];
    return t;
#else
    uint64_t c = 0;
    for (int i = 0; i < N; i++) { c += (uint64_t)a.v[i] + b.v[i]; t.v[i] = (uint32_t)c; c >>= 32; }
    int64_t bw = 0;
    for (int i = 0; i < N; i++) { bw += (int64_t)t.v[i] - (int64_t)P::mod(i); u.v[i] = (uint32_t)bw; bw >>= 32; }
    return bw ? t : u;
#endif
  }
  G16_HD static Fp sub(const Fp& a, const Fp& b) {
    Fp t;
#ifdef G16_PTX_PATH
    ptx::sub_cc(t.v[0], a.v[0], b.v[0]);
#pragma unroll
    for (int i = 1; i < N; i++) ptx::subc_cc(t.v[i], a.v[i], b.v[i]);
    uint32_t br;
    ptx::subc(br, 0, 0);  // mask: all ones iff a < b
    ptx::add_cc(t.v[0], t.v[0], P::mod(0) & br);
#pragma unroll
    for (int i = 1; i < N - 1; i++) ptx::addc_cc(t.v[i], t.v[i], P::mod(i) & br);
    ptx::addc(t.v[N - 1], t.v[N - 1], P::mod(N - 1) & br);
    return t;
#else
    int64_t bw = 0;
    for (int i = 0; i < N; i++) { bw += (int64_t)a.v[i] - (int64_t)b.v[i]; t.v[i] = (uint32_t)bw; bw >>= 32; }
    if (bw) {
      uint64_t c = 0;
      for (int i = 0; i < N; i++) { c += (uint64_t)t.v[i] + P::mod(i); t.v[i] = (uint32_t)c; c >>= 32; }
    }
    return t;
#endif
  }
  G16_HD static Fp neg(const Fp& a) { return a.is_zero() ? a : sub(modulus(), a); }  // p - a never borrows for 0 < a < p
  G16_HD static Fp dbl(const Fp& a) { return add(a, a); }

  // ---------------- Montgomery multiplication ----------------
#ifdef G16_PTX_PATH
  // acc[j], acc[j+1] += x[j] * y for even j in one carry chain; leaves CF = carry out of acc[N-1]
  G16_HD static void cmad_row(uint32_t* acc, const uint32_t* x, uint32_t y) {
    ptx::mad_lo_cc(acc[0], x[0], y, acc[0]);
    ptx::madc_hi_cc(acc[1], x[0], y, acc[1]);
#pragma unroll
    for (int j = 2; j < N; j += 2) {
      ptx::madc_lo_cc(acc[j], x[j], y, acc[j]);
      ptx::madc_hi_cc(acc[j + 1], x[j], y, acc[j + 1]);
    }
  }
  // same with x = limbs (off, off+2, ...) of the modulus (compile-time constants)
  template <int OFF>
  G16_HD static void cmad_row_mod(uint32_t* acc, uint32_t y) {
    ptx::mad_lo_cc(acc[0], P::mod(OFF), y, acc[0]);
    ptx::madc_hi_cc(acc[1], P::mod(OFF), y, acc[1]);
#pragma unroll
    for (int j = 2; j < N; j += 2) {
      ptx::madc_lo_cc(acc[j], P::mod(OFF + j), y, acc[j]);
      ptx::madc_hi_cc(acc[j + 1], P::mod(OFF + j), y, acc[j + 1]);
    }
  }
  // One Montgomery step.  The running value is V = E + (O << 32) with limb 0 of E already cleared by the
  // previous step and its >>32 still pending: the caller swaps the roles of the two arrays every step, so here
  // E is last step's odd array (already aligned) and O is last step's even array (to be moved down two limbs,
  // its limb 1 landing on E[0]).  Then V += a*bi, m = V[0]*(-p^-1), V += m*p.
  template <bool FIRST>
  G16_HD static void mont_step(uint32_t* E, uint32_t* O, const uint32_t* a, uint32_t bi) {
    if (FIRST) {
#pragma unroll
      for (int j = 0; j < N; j += 2) {
        ptx::mul_lo(E[j], a[j], bi);
        ptx::mul_hi(E[j + 1], a[j], bi);
        ptx::mul_lo(O[j], a[j + 1], bi);
        ptx::mul_hi(O[j + 1], a[j + 1], bi);
      }
    } else {
      ptx::add_cc(E[0], E[0], O[1]);
#pragma unroll
      for (int j = 0; j < N - 2; j += 2) {
        ptx::madc_lo_cc(O[j], a[j + 1], bi, O[j + 2]);
        ptx::madc_hi_cc(O[j + 1], a[j + 1], bi, O[j + 3]);
      }
      ptx::madc_lo_cc(O[N - 2], a[N - 1], bi, 0);
      ptx::madc_hi(O[N - 1], a[N - 1], bi, 0);
      cmad_row(E, a, bi);
      ptx::addc(O[N - 1], O[N - 1], 0);
    }
    uint32_t m = E[0] * P::INV32;
    cmad_row_mod<1>(O, m);  // odd limbs of p; by the V < 2^(32(N+1)) bound this chain cannot carry out
    cmad_row_mod<0>(E, m);
    ptx::addc(O[N - 1], O[N - 1], 0);
  }
  G16_HD static Fp mul(const Fp& a, const Fp& b) {
    static_assert(N % 2 == 0, "even limb count required");
    uint32_t ev[N], od[N];
    mont_step<true>(ev, od, a.v, b.v[0]);
    mont_step<false>(od, ev, a.v, b.v[1]);
#pragma unroll
    for (int i = 2; i < N; i += 2) {
      mont_step<false>(ev, od, a.v, b.v[i]);
      mont_step<false>(od, ev, a.v, b.v[i + 1]);
    }
    // last step had E = od, O = ev and its >>32 is pending: result[k] = od[k+1] + ev[k]
    Fp r;
    ptx::add_cc(r.v[0], od[1], ev[0]);
#pragma unroll
    for (int k = 1; k < N - 1; k++) ptx::addc_cc(r.v[k], od[k + 1], ev[k]);
    ptx::addc(r.v[N - 1], ev[N - 1], 0);
    return reduce_once(r);
  }
#else
  G16_HD static Fp mul(const Fp& a, const Fp& b) {
    constexpr int W = N / 2;
    uint64_t x[W], y[W], p[W], t[W + 2];
    memcpy(x, a.v, sizeof(x));
    memcpy(y, b.v, sizeof(y));
    for (int i = 0; i < W; i++) p[i] = (uint64_t)P::mod(2 * i) | ((uint64_t)P::mod(2 * i + 1) << 32);
    // -p^-1 mod 2^64 from the 32-bit inverse by one Newton step
    uint64_t inv = P::INV32;  // == -p^-1 mod 2^32
    inv = inv * (2 + p[0] * inv);  // Newton on x -> x(2 + p x) for x ~ -p^-1
    for (int i = 0; i < W + 2; i++) t[i] = 0;
    for (int i = 0; i < W; i++) {
      unsigned __int128 c = 0;
      for (int j = 0; j < W; j++) { c += (unsigned __int128)x[j] * y[i] + t[j]; t[j] = (uint64_t)c; c >>= 64; }
      c += t[W]; t[W] = (uint64_t)c; t[W + 1] = (uint64_t)(c >> 64);
      uint64_t m = t[0] * inv;
      c = (unsigned __int128)m * p[0] + t[0]; c >>= 64;
      for (int j = 1; j < W; j++) { c += (unsigned __int128)m * p[j] + t[j]; t[j - 1] = (uint64_t)c; c >>= 64; }
      c += t[W]; t[W - 1] = (uint64_t)c; t[W] = t[W + 1] + (uint64_t)(c >> 64);
    }
    Fp r;
    memcpy(r.v, t, sizeof(x));
    return reduce_once(r);
  }
#endif
  G16_HD static Fp sqr(const Fp& a) { return mul(a, a); }

  // r in [0, 2p) -> [0, p)
  G16_HD static Fp reduce_once(const Fp& t) {
    Fp u;
#ifdef G16_PTX_PATH
    ptx::sub_cc(u.v[0], t.v[0], P::mod(0));
#pragma unroll
    for (int i = 1; i < N; i++) ptx::subc_cc(u.v[i], t.v[i], P::mod(i));
    uint32_t br;
    ptx::subc(br, 0, 0);
#pragma unroll
    for (int i = 0; i < N; i++) u.v[i] = br ? t.v[i] : u.v[i];
    return u;
#else
    int64_t bw = 0;
    for (int i = 0; i < N; i++) { bw += (int64_t)t.v[i] - (int64_t)P::mod(i); u.v[i] = (uint32_t)bw; bw >>= 32; }
    return bw ? t : u;
#endif
  }

  // Montgomery <-> canonical (ark `into_bigint` / `from_bigint`, prover.rs:64,71,82)
  G16_HD static Fp from_mont(const Fp& a) {
    Fp o = zero();
    o.v[0] = 1;
    return mul(a, o);
  }
  G16_HD static Fp to_mont(const Fp& a) { return mul(a, r2()); }

  // small-constant multiples
  G16_HD static Fp mul_small(const Fp& a, int k) {
    Fp r = zero();
    Fp base = a;
    while (k) {
      if (k & 1) r = add(r, base);
      k >>= 1;
      if (k) base = dbl(base);
    }
    return r;
  }

  // a^e for a little-endian u32 exponent of `nl` limbs
  G16_HD static Fp pow(const Fp& a, const uint32_t* e, int nl) {
    Fp r = one();
    bool started = false;
    for (int i = nl * 32 - 1; i >= 0; i--) {
      if (started) r = sqr(r);
      if ((e[i >> 5] >> (i & 31)) & 1) {
        r = started ? mul(r, a) : a;
        started = true;
      }
    }
    return r;
  }
  G16_HD static Fp pow_u64(const Fp& a, uint64_t e) {
    uint32_t w[2] = {(uint32_t)e, (uint32_t)(e >> 32)};
    return pow(a, w, 2);
  }
  // Fermat inverse a^(p-2); inverse of zero is zero
  G16_HD static Fp inv(const Fp& a) {
    uint32_t e[N];
    // p - 2 (p is odd and > 2, so limb 0 does not borrow beyond itself unless it is < 2)
    uint64_t bw = 2;
    for (int i = 0; i < N; i++) {
      uint64_t m = P::mod(i);
      uint64_t d = m - bw;
      e[i] = (uint32_t)d;
      bw = (m < bw) ? 1 : 0;
    }
    return pow(a, e, N);
  }

  G16_HD friend Fp operator+(const Fp& a, const Fp& b) { return add(a, b); }
  G16_HD friend Fp operator-(const Fp& a, const Fp& b) { return sub(a, b); }
  G16_HD friend Fp operator*(const Fp& a, const Fp& b) { return mul(a, b); }
};

}  // namespace g16
