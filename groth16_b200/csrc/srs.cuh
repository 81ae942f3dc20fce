// srs.cuh -- proving keys from a powers-of-tau transcript (g16_setup_from_srs) and phase-2 delta contributions
// (g16_setup_contribute): the group-valued inverse FFT (also every Lagrange level of g16_ptau_prepare), sparse sums of
// points, one scalar times many points, and the transcript point checks; phase-1 contributions to a transcript (g16_srs_contribute): every point times its own power
// of the secret; the scalars of the transcript check (g16_srs_verify_pairs): one power of the challenge per point; the
// H-query weights of the key check (g16_pk_verify_pairs); and delta contributions to a key in host memory
// (g16_pk_contribute): every point times the one scalar delta^-1.
//
// Every kernel works on XYZZ points in global memory, one point (or one butterfly, or one chunk of a sum) per thread.  The
// scalar multiplications are left-to-right double-and-add over the canonical scalar (XYZZ::mul_u32), except the transform's
// twiddle products on the groups srs_windowed names: a signed 4-bit window over a per-thread table (srs_mul_w4).
#pragma once
#include <cstdint>
#include <vector>
#include "ser.cuh"

namespace g16 {

// ---- host planning of the sparse sums -----------------------------------------------------------------------------------
// A sum runs in levels.  Level 0 forms one product (coefficient x point) per entry; every later level adds the items of
// each segment (one column of the CSC, or what is left of it) in chunks of at most SRS_CHUNK consecutive items, one thread
// per chunk, until no segment holds more than one item.  A column of every row (the One variable: one entry per constraint)
// therefore costs log_CHUNK(rows) levels, and no thread ever adds more than SRS_CHUNK items.
static constexpr uint32_t SRS_CHUNK = 16;
// seg: segment s holds items seg[s] .. seg[s + 1] - 1.  Appends to `chunk` the first item of every chunk (chunks cover the
// items in order, none spans two segments; chunk.back() = total items as the end sentinel) and sets next[s] = index of the
// first chunk of segment s (the segments of the next level).  Returns the largest segment length of the next level.
inline uint64_t srs_split(const std::vector<uint64_t>& seg, uint32_t k, std::vector<uint64_t>& chunk, std::vector<uint64_t>& next) {
  const size_t ns = seg.size() - 1;
  chunk.clear();
  next.assign(ns + 1, 0);
  uint64_t longest = 0;
  for (size_t s = 0; s < ns; s++) {
    next[s] = chunk.size();
    for (uint64_t b = seg[s]; b < seg[s + 1]; b += k) chunk.push_back(b);
    longest = std::max<uint64_t>(longest, chunk.size() - next[s]);
  }
  next[ns] = chunk.size();
  chunk.push_back(seg[ns]);
  return longest;
}
// The levels of one sum over columns with pointers `cp` (CSC): the chunk starts of every level, and the final segment
// pointers (each column holds 0 or 1 item of the last level's output).
struct SrsSumPlan {
  std::vector<std::vector<uint64_t>> levels;
  std::vector<uint64_t> last;
  void make(const std::vector<uint64_t>& cp, uint32_t k = SRS_CHUNK) {
    levels.clear();
    std::vector<uint64_t> seg = cp, next, chunk;
    uint64_t longest = 0;
    for (size_t s = 0; s + 1 < seg.size(); s++) longest = std::max<uint64_t>(longest, seg[s + 1] - seg[s]);
    while (longest > 1) {
      longest = srs_split(seg, k, chunk, next);
      levels.push_back(chunk);
      seg.swap(next);
    }
    last = seg;
  }
};

// ---- phase-1 contributions (g16_srs_contribute) -------------------------------------------------------------------------
// A member of `len` points runs in chunks of at most `cap` points; the chunk starting at point i0 holds
// srs_chunk_len(len, i0, cap) of them.  len < 2^32 and 1 <= cap < 2^32, so a chunk's count and every index fit in 32 bits.
inline uint32_t srs_chunk_len(uint64_t len, uint64_t i0, uint64_t cap) { return (uint32_t)std::min<uint64_t>(cap, len - i0); }
// Whether the byte ranges [a, a + na) and [b, b + nb) share a byte; an empty range shares none.  The contribution calls
// refuse an output range that overlaps any input or output range other than its own input (in place).
inline bool srs_overlap(uintptr_t a, uint64_t na, uintptr_t b, uint64_t nb) { return na && nb && a < b + nb && b < a + na; }
// Points per chunk: as many points of `esz` bytes as `free_bytes` of device memory hold after a 512 MiB margin, and no more
// than `chunk_points` (0: no cap of its own), `longest` (the longest member) or 2^32 - 1; at least 1.
inline uint64_t srs_chunk_cap(uint64_t chunk_points, uint64_t longest, uint64_t free_bytes, uint64_t esz) {
  const uint64_t margin = 512ull << 20;
  uint64_t cap = free_bytes > margin ? (free_bytes - margin) / esz : 0;
  if (chunk_points) cap = std::min(cap, chunk_points);
  cap = std::min(cap, std::min<uint64_t>(longest, 0xffffffffull));
  return std::max<uint64_t>(cap, 1);
}
// c tau^j from tab[k] = tau^(2^k): one Fr product per set bit of j (at most 32).  The kernel forms its point's scalar this
// way with c = x tau^i0 and j = the point's index in its chunk; the host forms c itself the same way with j = i0.
template <class FrF>
G16_HD FrF srs_power(FrF c, const FrF* tab, uint64_t j) {
  for (int k = 0; j; k++, j >>= 1)
    if (j & 1) c = FrF::mul(c, tab[k]);
  return c;
}

// ---- transcript checks (g16_srs_verify_pairs) ---------------------------------------------------------------------------
// The largest chunk one MSM of caller-supplied bases takes (the stand-alone MSM refuses n >= 2^27).
static constexpr uint64_t SRS_VERIFY_MSM_MAX = (1ull << 27) - 1;
// Points per chunk of the transcript check: the most that `free_bytes` of device memory hold after the 512 MiB margin, a
// chunk of cnt points needing cnt * per_point bytes (the point, its Fr scalar, its byte of the identity mask) and
// ws_bytes(cnt) for the MSM workspace of its geometry; and no more than `chunk_points` (0: no cap of its own), `longest`
// or SRS_VERIFY_MSM_MAX; at least 1.  The workspace is not linear in cnt (the window grows with it), so the largest chunk
// that fits is found by bisection.
template <class WsBytes>
uint64_t srs_verify_chunk_cap(uint64_t chunk_points, uint64_t longest, uint64_t free_bytes, uint64_t per_point, WsBytes ws_bytes) {
  const uint64_t margin = 512ull << 20;
  const uint64_t avail = free_bytes > margin ? free_bytes - margin : 0;
  auto fits = [&](uint64_t cnt) { return cnt * per_point + (uint64_t)ws_bytes(cnt) <= avail; };
  uint64_t cap = std::min(longest, SRS_VERIFY_MSM_MAX);
  if (chunk_points) cap = std::min(cap, chunk_points);
  if (cap <= 1 || fits(cap)) return std::max<uint64_t>(cap, 1);
  uint64_t lo = 1, hi = cap;   // hi does not fit; lo fits, or is the floor of 1
  while (hi - lo > 1) {
    const uint64_t mid = lo + (hi - lo) / 2;
    (fits(mid) ? lo : hi) = mid;
  }
  return lo;
}

// ---- device functions -----------------------------------------------------------------------------------------------
template <class P>
G16_HD bool srs_canonical(const Fp<P>& a) { return ser_lt_mod(a); }
template <class P, int NR>
G16_HD bool srs_canonical(const Fp2<P, NR>& a) { return ser_lt_mod(a.c0) && ser_lt_mod(a.c1); }
// Check flag of the transcript check alone (beside SER_VALIDATE): the identity is refused, with its own result code.
enum : uint32_t { SRS_REFUSE_IDENTITY = 1u << 8 };
enum : uint32_t { SRS_ERR_IDENTITY = 9 };   // after the SER_ERR_* codes of ser.cuh
inline const char* srs_reason(uint32_t code) { return code == SRS_ERR_IDENTITY ? "point is the identity" : ser_reason(code); }
// A transcript point: Montgomery limbs below q, on the curve, and with G16_SER_VALIDATE in the prime-order subgroup (the
// check ser.cuh runs on decoded keys; skipped for BN254 G1, whose cofactor is 1).  All-zero limbs are the identity, accepted
// unless SRS_REFUSE_IDENTITY is set.
template <class CP, bool G2>
G16_HD uint32_t srs_check_point(const Affine<SerField<CP, G2>>& p, uint32_t flags) {
  using F = SerField<CP, G2>;
  if (p.is_inf()) return (flags & SRS_REFUSE_IDENTITY) ? (uint32_t)SRS_ERR_IDENTITY : (uint32_t)SER_OK;
  if (!srs_canonical(p.x) || !srs_canonical(p.y)) return SER_ERR_NONCANONICAL;
  if (F::sqr(p.y) != F::add(F::mul(F::sqr(p.x), p.x), ser_b<CP, G2>())) return SER_ERR_OFF_CURVE;
  if ((flags & SER_VALIDATE) && !(!G2 && SerFormat<CP>::G1_COFACTOR_ONE) && !ser_in_subgroup<typename CP::FrP>(p))
    return SER_ERR_SUBGROUP;
  return SER_OK;
}
// ---- the group inverse transform: which butterfly each thread runs, and its twiddle -------------------------------------
// i < 2^log_n reversed over log_n bits (log_n < 32)
G16_HD uint32_t srs_bitrev(uint32_t i, int log_n) {
  uint32_t r = 0;
  for (int b = 0; b < log_n; b++, i >>= 1) r = (r << 1) | (i & 1u);
  return r;
}
// Stage of span h = 2^log_h over n = 2^log_n points: n / 2 butterflies in G = n / 2h groups of h, group g joining points
// 2hg + k and 2hg + k + h with twiddle k < h.  Thread t runs k = t / G, g = t mod G, so the G threads of one twiddle are
// consecutive: a warp shares one twiddle wherever G >= 32, which is every stage but the last five (h >= n / 32).  There a
// warp holds 32 / G twiddles, each shared by G lanes.
G16_HD void srs_butterfly_at(uint32_t t, int log_n, int log_h, uint32_t& k, uint32_t& i0) {
  const int log_g = log_n - 1 - log_h;
  k = t >> log_g;
  i0 = ((t & ((1u << log_g) - 1)) << (log_h + 1)) + k;
}
// The exponent e of twiddle k at span 2^log_h, omega_n^-(k n / 2h) = omega_N^-e with N = 2^tab_log >= n: e = k N / 2h.
G16_HD uint64_t srs_twiddle_exp(uint32_t k, int log_h, int tab_log) { return (uint64_t)k << (tab_log - 1 - log_h); }

// omega_N^-e in canonical form from tab[b] = omega_N^-(2^b) (Montgomery); out of line, so that its products are done
// before the butterfly's points are live
template <class FrF>
G16_HD_NOINLINE FrF srs_twiddle(const FrF* tab, uint64_t e) { return FrF::from_mont(srs_power(FrF::one(), tab, e)); }
// Signed fixed-window recoding of a canonical scalar k of nl 32-bit limbs: digits d_i in [-7, 8] with
// k = sum_i d_i 16^i, i < 8 nl + 1.  Returns the digit count.
G16_HD int srs_recode_w4(const uint32_t* k, int nl, int8_t* d) {
  int carry = 0;
  for (int i = 0; i < 8 * nl; i++) {
    const int v = (int)((k[i >> 3] >> (4 * (i & 7))) & 15u) + carry;
    carry = v > 8;
    d[i] = (int8_t)(v - 16 * carry);
  }
  d[8 * nl] = (int8_t)carry;
  return 8 * nl + 1;
}
// p times the canonical scalar k (nl limbs) by the signed 4-bit window: a table of 1P .. 8P per thread (local memory), then
// per digit from the top four doublings and one addition of +-table[|d| - 1] (skipped for d = 0).  The operation sequence is
// the same for every scalar but for zero digits and leading zero windows, about 64 additions against the ~128 of
// XYZZ::mul_u32's double-and-add.
template <class F>
G16_HD_NOINLINE XYZZ<F> srs_mul_w4(const XYZZ<F>& p, const uint32_t* k, int nl) {
  constexpr int MAXD = 8 * 12 + 1;   // up to 12 limbs (BW6-761's 377-bit scalars)
  int8_t d[MAXD];
  const int nd = srs_recode_w4(k, nl, d);
  XYZZ<F> tab[8];
  tab[0] = p;
  for (int j = 1; j < 8; j++) { tab[j] = tab[j - 1]; tab[j].add(p); }
  XYZZ<F> r = XYZZ<F>::inf();
  int top = nd - 1;
  while (top > 0 && d[top] == 0) top--;
  for (int i = top; i >= 0; i--) {
    if (i != top)
      for (int b = 0; b < 4; b++) r.dbl_inplace();
    const int a = d[i] < 0 ? -d[i] : d[i];
    if (a) {
      XYZZ<F> t = tab[a - 1];
      if (d[i] < 0) t.negate();
      r.add(t);
    }
  }
  return r;
}

template <class F, class FrF>
G16_HD XYZZ<F> srs_mul(const XYZZ<F>& p, const FrF& s_mont) {
  const FrF s = FrF::from_mont(s_mont);
  return p.mul_u32(s.v, FrF::N);
}
// *out = affine form of *p.  Base fields: the out-of-line XYZZ::to_affine.  Fq2: inlined, reading each coordinate only
// where it is used -- XYZZ::to_affine holds the whole point across the inversion, which spills for BN254's Fq2, while
// inlining the base-field form spills for BLS12-377 and BLS12-381 G1.
template <class F>
G16_HD void srs_store_affine(const XYZZ<F>* p, Affine<F>* out) { *out = p->to_affine(); }
template <class P, int NR>
G16_HD void srs_store_affine(const XYZZ<Fp2<P, NR>>* p, Affine<Fp2<P, NR>>* out) {
  using F = Fp2<P, NR>;
  const F zzz = p->ZZZ;
  if (p->ZZ.is_zero()) { *out = Affine<F>::inf(); return; }
  const F zi = F::inv(zzz);             // 1/Z^3
  const F z = F::mul(zi, p->ZZ);        // 1/Z
  out->y = F::mul(p->Y, zi);
  out->x = F::mul(p->X, F::sqr(z));
}

#ifdef __CUDACC__
// err: min over bad points of (member << 48 | index << 8 | code), so the first bad point by member, then index
template <class CP, bool G2>
__global__ void __launch_bounds__(128) srs_check_kernel(const Affine<SerField<CP, G2>>* p, uint32_t cnt, uint32_t flags,
                                                        uint32_t member, unsigned long long* err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cnt) return;
  const uint32_t code = srs_check_point<CP, G2>(p[i], flags);
  if (code) atomicMin(err, ((unsigned long long)member << 48) | ((unsigned long long)i << 8) | code);
}
// out[i] = P(a + i) - P(b + i), P(k) = pts[k] for k < len and the identity beyond: the H query's differences
template <class F>
__global__ void __launch_bounds__(128) srs_diff_kernel(const Affine<F>* pts, uint32_t len, uint32_t a, uint32_t b, uint32_t cnt,
                                                       XYZZ<F>* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cnt) return;
  XYZZ<F> r = a + i < len ? XYZZ<F>::from_affine(pts[a + i]) : XYZZ<F>::inf();
  if (b + i < len) r.madd(pts[b + i], true);
  out[i] = r;
}
template <class F>
__global__ void __launch_bounds__(128) srs_load_kernel(const Affine<F>* in, uint32_t cnt, XYZZ<F>* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cnt) out[i] = XYZZ<F>::from_affine(in[i]);
}
template <class F>
__global__ void __launch_bounds__(128) srs_affine_kernel(const XYZZ<F>* in, uint32_t cnt, Affine<F>* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cnt) srs_store_affine(in + i, out + i);
}
// p[i] *= s[i * stride]: stride 0 is one scalar for every point (uniform control flow across the warp)
template <class F, class FrF>
__global__ void __launch_bounds__(128) srs_scale_kernel(XYZZ<F>* p, uint32_t cnt, const FrF* s, uint32_t stride) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cnt) p[i] = srs_mul(p[i], s[(uint64_t)i * stride]);
}
// One chunk of a phase-1 contribution, in place: p[j] *= c tau^j (tab[k] = tau^(2^k)), affine in and out; the identity
// stays the identity.  j in 64 bits: a chunk may hold up to 2^32 - 1 points.
template <class F, class FrF>
__global__ void __launch_bounds__(128) srs_contribute_kernel(Affine<F>* p, uint32_t cnt, const FrF* tab, FrF c) {
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= cnt) return;
  const XYZZ<F> r = srs_mul(XYZZ<F>::from_affine(p[j]), srs_power(c, tab, j));
  srs_store_affine(&r, p + j);
}
// One chunk of a delta contribution to a key in host memory (g16_pk_contribute), in place: p[j] *= s for the one scalar
// s = delta^-1, affine in and out; the identity stays the identity.  Every thread has the same scalar, so each of its bits
// costs the warp the same branch.
template <class F, class FrF>
__global__ void __launch_bounds__(128) srs_scale_affine_kernel(Affine<F>* p, uint32_t cnt, FrF s) {
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= cnt) return;
  const XYZZ<F> r = srs_mul(XYZZ<F>::from_affine(p[j]), s);
  srs_store_affine(&r, p + j);
}
// The scalars of one chunk of a transcript check: out[j] = c rho^j (tab[k] = rho^(2^k), c = rho^i0), Montgomery form.
template <class FrF>
__global__ void __launch_bounds__(128) srs_powers_kernel(const FrF* tab, FrF c, uint32_t cnt, FrF* out) {
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < cnt) out[j] = srs_power(c, tab, j);
}
// The weights on tau_g1[0 .. 2n - 1) of the H-query check (g16_pk_verify_pairs), Montgomery form, k < cnt:
//   f == nullptr (LibsnarkReduction, tab = rho^(2^b), c = 1): out[k] = -rho^k (k < n - 1), 0 (k = n - 1), rho^(k-n) (k >= n)
//   otherwise    (CircomReduction, tab = w^(2^b) with w = omega_2n^-1, c = (2n)^-1): out[k] = c w^k f[k mod n]
template <class FrF>
__global__ void __launch_bounds__(128) srs_h_weights_kernel(const FrF* tab, FrF c, const FrF* f, uint32_t n, uint32_t cnt,
                                                            FrF* out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= cnt) return;
  if (f) {
    out[k] = FrF::mul(srs_power(c, tab, k), f[k & (n - 1)]);
  } else if (k + 1 < n) {
    out[k] = FrF::neg(srs_power(c, tab, k));
  } else {
    out[k] = k + 1 == n ? FrF::zero() : srs_power(c, tab, k - n);
  }
}
// The group inverse transform: load (bit reversal and scaling folded in), then one kernel per radix-2 stage.
// work[i] = s_j X_j with j = rev(i), X_j = P(j) - P(j + d) (d = 0: X_j = P(j)), P(k) = in[k] for k < len and the identity
// beyond, s_j = s[j * stride] (stride 0: one scalar for every point, uniform control flow; s == nullptr: no product).  The
// transform is linear, so a scaling of its input is the scaling of its output.
template <class F, class FrF>
__global__ void __launch_bounds__(128) srs_ifft_load_kernel(const Affine<F>* in, uint64_t len, uint64_t d, int log_n,
                                                            const FrF* s, uint32_t stride, XYZZ<F>* work) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (1u << log_n)) return;
  const uint32_t j = srs_bitrev(i, log_n);
  XYZZ<F> x = j < len ? XYZZ<F>::from_affine(in[j]) : XYZZ<F>::inf();
  if (d && j + d < len) x.madd(in[j + d], true);
  if (s) x = srs_mul(x, s[(uint64_t)j * stride]);
  work[i] = x;
}
// One radix-2 decimation-in-time stage of span h = 2^log_h over bit-reversed points: butterfly t (srs_butterfly_at) maps
// (P, Q) -> (P + w^-k Q, P - w^-k Q) with w^-k = tab-power srs_twiddle_exp(k, log_h, tab_log) (tab[b] = omega_N^-(2^b),
// N = 2^tab_log, any N >= n); k = 0 skips the product.  AFF (the last stage): both results go to out in canonical affine
// form instead of back to p.  WIN: the twiddle product by the signed window (srs_mul_w4) instead of double-and-add.
template <class F, class FrF, bool AFF, bool WIN>
__global__ void __launch_bounds__(128) srs_ifft_stage_kernel(XYZZ<F>* p, int log_n, int log_h, const FrF* tab, int tab_log,
                                                             Affine<F>* out) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (1u << (log_n - 1))) return;
  uint32_t k, i0;
  srs_butterfly_at(t, log_n, log_h, k, i0);
  const uint32_t i1 = i0 + (1u << log_h);
  XYZZ<F> q = p[i1];
  if (k) {
    const FrF w = srs_twiddle(tab, srs_twiddle_exp(k, log_h, tab_log));
    q = WIN ? srs_mul_w4(q, w.v, FrF::N) : q.mul_u32(w.v, FrF::N);
  }
  if (AFF) {   // p is not written: P is read again for the second result rather than held across the first's inversion
    XYZZ<F> r = p[i0];
    r.add(q);
    srs_store_affine(&r, out + i0);
    r = p[i0];
    q.negate();
    r.add(q);
    srs_store_affine(&r, out + i1);
  } else {
    XYZZ<F> lo = p[i0];
    XYZZ<F> hi = lo;
    lo.add(q);
    q.negate();
    hi.add(q);
    p[i0] = lo;
    p[i1] = hi;
  }
}
// level 0 of a sparse sum: out[e] = coeff[e] * src[idx[e]], the product skipped when the coefficient is One
template <class F, class FrF>
__global__ void __launch_bounds__(128) srs_terms_kernel(const XYZZ<F>* src, const uint32_t* idx, const FrF* coeff, uint32_t cnt,
                                                        XYZZ<F>* out) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= cnt) return;
  const uint32_t j = idx[e];
  FrF c = coeff[e];
  if (c == FrF::one()) { out[e] = src[j]; return; }
  c = FrF::from_mont(c);
  out[e] = src[j].mul_u32(c.v, FrF::N);
}
// a later level: out[k] = sum of in[chunk[k] .. chunk[k + 1] - 1] (at most SRS_CHUNK items)
template <class F>
__global__ void __launch_bounds__(128) srs_reduce_kernel(const XYZZ<F>* in, const uint64_t* chunk, uint32_t cnt, XYZZ<F>* out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= cnt) return;
  XYZZ<F> acc = XYZZ<F>::inf();
  for (uint64_t j = chunk[k]; j < chunk[k + 1]; j++) acc.add(in[j]);
  out[k] = acc;
}
// the column results: the single item of every segment, the identity (all-zero limbs) for an empty column
template <class F>
__global__ void __launch_bounds__(128) srs_gather_kernel(const XYZZ<F>* in, const uint64_t* seg, uint32_t cols, Affine<F>* out) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= cols) return;
  if (seg[j + 1] > seg[j]) srs_store_affine(in + seg[j], out + j);
  else out[j] = Affine<F>::inf();
}

static inline unsigned srs_blocks(uint64_t cnt) { return (unsigned)((cnt + 127) / 128); }

template <class CP, bool G2>
cudaError_t srs_check(cudaStream_t st, const void* pts, uint32_t cnt, uint32_t flags, uint32_t member, unsigned long long* err) {
  if (cnt) srs_check_kernel<CP, G2><<<srs_blocks(cnt), 128, 0, st>>>(static_cast<const Affine<SerField<CP, G2>>*>(pts), cnt,
                                                                       flags, member, err);
  return cudaGetLastError();
}
template <class F>
cudaError_t srs_diff(cudaStream_t st, const Affine<F>* pts, uint32_t len, uint32_t a, uint32_t b, uint32_t cnt, XYZZ<F>* out) {
  if (cnt) srs_diff_kernel<F><<<srs_blocks(cnt), 128, 0, st>>>(pts, len, a, b, cnt, out);
  return cudaGetLastError();
}
template <class F>
cudaError_t srs_load(cudaStream_t st, const Affine<F>* in, uint32_t cnt, XYZZ<F>* out) {
  if (cnt) srs_load_kernel<F><<<srs_blocks(cnt), 128, 0, st>>>(in, cnt, out);
  return cudaGetLastError();
}
template <class F>
cudaError_t srs_affine(cudaStream_t st, const XYZZ<F>* in, uint32_t cnt, Affine<F>* out) {
  if (cnt) srs_affine_kernel<F><<<srs_blocks(cnt), 128, 0, st>>>(in, cnt, out);
  return cudaGetLastError();
}
template <class F, class FrF>
cudaError_t srs_scale(cudaStream_t st, XYZZ<F>* p, uint32_t cnt, const FrF* s, uint32_t stride) {
  if (cnt) srs_scale_kernel<F, FrF><<<srs_blocks(cnt), 128, 0, st>>>(p, cnt, s, stride);
  return cudaGetLastError();
}
template <class F, class FrF>
cudaError_t srs_contribute(cudaStream_t st, Affine<F>* p, uint32_t cnt, const FrF* tab, FrF c) {
  if (cnt) srs_contribute_kernel<F, FrF><<<srs_blocks(cnt), 128, 0, st>>>(p, cnt, tab, c);
  return cudaGetLastError();
}
template <class F, class FrF>
cudaError_t srs_scale_affine(cudaStream_t st, Affine<F>* p, uint32_t cnt, FrF s) {
  if (cnt) srs_scale_affine_kernel<F, FrF><<<srs_blocks(cnt), 128, 0, st>>>(p, cnt, s);
  return cudaGetLastError();
}
template <class FrF>
cudaError_t srs_powers(cudaStream_t st, const FrF* tab, FrF c, uint32_t cnt, FrF* out) {
  if (cnt) srs_powers_kernel<FrF><<<srs_blocks(cnt), 128, 0, st>>>(tab, c, cnt, out);
  return cudaGetLastError();
}
template <class FrF>
cudaError_t srs_h_weights(cudaStream_t st, const FrF* tab, FrF c, const FrF* f, uint32_t n, uint32_t cnt, FrF* out) {
  if (cnt) srs_h_weights_kernel<FrF><<<srs_blocks(cnt), 128, 0, st>>>(tab, c, f, n, cnt, out);
  return cudaGetLastError();
}
// Whether the stages multiply by the twiddle with the signed window (srs_mul_w4) rather than double-and-add: in every stage,
// for the groups whose window kernels compile without spills (coordinates of at most 64 bytes: BN254 G1 and G2, BLS12-381
// and BLS12-377 G1).  Measured faster in both groups of BN254 and BLS12-381 (DESIGN.md section 21); the Fq2 points of the
// BLS curves and BW6-761's points spill their 8-point table, so they keep double-and-add.
template <class F>
constexpr bool srs_windowed() { return sizeof(F) <= 64; }
// The inverse transform of size n = 2^log_n (log_n < 32): Y_i = sum_{j<n} omega_n^(-ij) s_j X_j with X_j, s_j as
// srs_ifft_load_kernel forms them from (in, len, d, s, stride).  tab (device): omega_N^-(2^b) for b < tab_log, N >= n.
// Y goes to work (n XYZZ); with aff, the last stage writes Y in canonical affine form to aff instead (work then holds
// the stage before it).  1 + log_n launches (2 for log_n = 0 with aff).
template <class F, class FrF>
cudaError_t srs_ifft(cudaStream_t st, const Affine<F>* in, uint64_t len, uint64_t d, int log_n, const FrF* s, uint32_t stride,
                     const FrF* tab, int tab_log, XYZZ<F>* work, Affine<F>* aff, unsigned long long* launches) {
  const uint64_t n = 1ull << log_n;
  srs_ifft_load_kernel<F, FrF><<<srs_blocks(n), 128, 0, st>>>(in, len, d, log_n, s, stride, work);
  for (int lh = 0; lh < log_n; lh++) {
    const bool last = aff && lh == log_n - 1;
    const unsigned b = srs_blocks(n / 2);
    if constexpr (srs_windowed<F>()) {
      if (last) srs_ifft_stage_kernel<F, FrF, true, true><<<b, 128, 0, st>>>(work, log_n, lh, tab, tab_log, aff);
      else srs_ifft_stage_kernel<F, FrF, false, true><<<b, 128, 0, st>>>(work, log_n, lh, tab, tab_log, nullptr);
    } else {
      if (last) srs_ifft_stage_kernel<F, FrF, true, false><<<b, 128, 0, st>>>(work, log_n, lh, tab, tab_log, aff);
      else srs_ifft_stage_kernel<F, FrF, false, false><<<b, 128, 0, st>>>(work, log_n, lh, tab, tab_log, nullptr);
    }
  }
  if (aff && log_n == 0) srs_affine_kernel<F><<<1, 128, 0, st>>>(work, 1, aff);
  if (launches) *launches += 1 + log_n + (aff && log_n == 0);
  return cudaGetLastError();
}
// One sparse sum.  src: the points, d_idx / d_coeff: the entries in column order, terms: cnt XYZZ of scratch, tmp: as many
// (the reduction levels ping-pong between the two), d_chunk: room for the largest level of the plan, d_last: the plan's
// final segment pointers (cols + 1).  out: one affine point per column.
template <class F, class FrF>
cudaError_t srs_sum(cudaStream_t st, const XYZZ<F>* src, const uint32_t* d_idx, const FrF* d_coeff, uint32_t cnt,
                    const SrsSumPlan& plan, XYZZ<F>* terms, XYZZ<F>* tmp, uint64_t* d_chunk, uint64_t* d_last, uint32_t cols,
                    Affine<F>* out) {
  cudaError_t e;
  if (cnt) srs_terms_kernel<F, FrF><<<srs_blocks(cnt), 128, 0, st>>>(src, d_idx, d_coeff, cnt, terms);
  XYZZ<F>* in = terms;
  XYZZ<F>* o = tmp;
  for (const std::vector<uint64_t>& lv : plan.levels) {
    const uint32_t chunks = (uint32_t)(lv.size() - 1);
    if ((e = cudaMemcpyAsync(d_chunk, lv.data(), lv.size() * 8, cudaMemcpyHostToDevice, st)) != cudaSuccess) return e;
    if (chunks) srs_reduce_kernel<F><<<srs_blocks(chunks), 128, 0, st>>>(in, d_chunk, chunks, o);
    std::swap(in, o);
    // the next level's copy into d_chunk must wait until this level has read it: same stream, so it does
  }
  if ((e = cudaMemcpyAsync(d_last, plan.last.data(), plan.last.size() * 8, cudaMemcpyHostToDevice, st)) != cudaSuccess) return e;
  if (cols) srs_gather_kernel<F><<<srs_blocks(cols), 128, 0, st>>>(in, d_last, cols, out);
  return cudaGetLastError();
}

#define G16_SRS_POINT_TEMPLATES(X, F, FrF)                                                                          \
  X cudaError_t srs_diff<F>(cudaStream_t, const Affine<F>*, uint32_t, uint32_t, uint32_t, uint32_t, XYZZ<F>*);        \
  X cudaError_t srs_load<F>(cudaStream_t, const Affine<F>*, uint32_t, XYZZ<F>*);                                      \
  X cudaError_t srs_affine<F>(cudaStream_t, const XYZZ<F>*, uint32_t, Affine<F>*);                                    \
  X cudaError_t srs_scale<F, FrF>(cudaStream_t, XYZZ<F>*, uint32_t, const FrF*, uint32_t);                            \
  X cudaError_t srs_contribute<F, FrF>(cudaStream_t, Affine<F>*, uint32_t, const FrF*, FrF);                          \
  X cudaError_t srs_ifft<F, FrF>(cudaStream_t, const Affine<F>*, uint64_t, uint64_t, int, const FrF*, uint32_t,        \
                                 const FrF*, int, XYZZ<F>*, Affine<F>*, unsigned long long*);                         \
  X cudaError_t srs_sum<F, FrF>(cudaStream_t, const XYZZ<F>*, const uint32_t*, const FrF*, uint32_t, const SrsSumPlan&, \
                                XYZZ<F>*, XYZZ<F>*, uint64_t*, uint64_t*, uint32_t, Affine<F>*);
#define G16_SRS_TEMPLATES(X, CP)                                                                                     \
  X cudaError_t srs_check<CP, false>(cudaStream_t, const void*, uint32_t, uint32_t, uint32_t, unsigned long long*);  \
  X cudaError_t srs_check<CP, true>(cudaStream_t, const void*, uint32_t, uint32_t, uint32_t, unsigned long long*);   \
  X cudaError_t srs_powers<Fp<CP::FrP>>(cudaStream_t, const Fp<CP::FrP>*, Fp<CP::FrP>, uint32_t, Fp<CP::FrP>*);     \
  X cudaError_t srs_h_weights<Fp<CP::FrP>>(cudaStream_t, const Fp<CP::FrP>*, Fp<CP::FrP>, const Fp<CP::FrP>*,       \
                                           uint32_t, uint32_t, Fp<CP::FrP>*);                                       \
  X cudaError_t srs_scale_affine<Fp<CP::FqP>, Fp<CP::FrP>>(cudaStream_t, Affine<Fp<CP::FqP>>*, uint32_t, Fp<CP::FrP>); \
  G16_SRS_POINT_TEMPLATES(X, Fp<CP::FqP>, Fp<CP::FrP>)
#endif

}  // namespace g16
