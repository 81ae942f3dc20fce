// srs.cuh -- proving keys from a powers-of-tau transcript (g16_setup_from_srs) and phase-2 delta contributions
// (g16_setup_contribute): the group-valued inverse FFT, sparse sums of points, one scalar times many points, and the
// transcript point checks; phase-1 contributions to a transcript (g16_srs_contribute): every point times its own power
// of the secret; the scalars of the transcript check (g16_srs_verify_pairs): one power of the challenge per point; the
// H-query weights of the key check (g16_pk_verify_pairs); and delta contributions to a key in host memory
// (g16_pk_contribute): every point times the one scalar delta^-1.
//
// Every kernel works on XYZZ points in global memory, one point (or one butterfly, or one chunk of a sum) per thread.  The
// scalar multiplications are left-to-right double-and-add over the canonical scalar (XYZZ::mul_u32); a windowed form would
// need a per-thread table of points in local or shared memory (DESIGN.md section 13).
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
// in-place bit-reversal permutation of 2^log_n points
template <class F>
__global__ void __launch_bounds__(128) srs_bitrev_kernel(XYZZ<F>* p, uint32_t n, int log_n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || log_n == 0) return;
  const uint32_t r = __brev(i) >> (32 - log_n);
  if (i < r) { const XYZZ<F> t = p[i]; p[i] = p[r]; p[r] = t; }
}
// One radix-2 decimation-in-time stage of the unscaled inverse transform over bit-reversed points: butterflies of span h,
// (P, Q) -> (P + w^-k Q, P - w^-k Q) with w^-k = tw_inv[k n / 2h] (the circuit domain's omega^-i, i < n / 2); k = 0 skips
// the multiplication.
template <class F, class FrF>
__global__ void __launch_bounds__(128) srs_butterfly_kernel(XYZZ<F>* p, uint32_t n, uint32_t h, const FrF* tw_inv) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n / 2) return;
  const uint32_t k = t & (h - 1);
  const uint32_t i0 = (t - k) * 2 + k, i1 = i0 + h;
  XYZZ<F> q = p[i1];
  if (k) q = srs_mul(q, tw_inv[(uint64_t)k * (n / (2 * h))]);
  XYZZ<F> lo = p[i0];
  XYZZ<F> hi = lo;
  lo.add(q);
  q.negate();
  hi.add(q);
  p[i0] = lo;
  p[i1] = hi;
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
// the unscaled inverse transform of 2^log_n points in place: out[j] = sum_i omega^(-ij) in[i]
template <class F, class FrF>
cudaError_t srs_ifft(cudaStream_t st, XYZZ<F>* p, int log_n, const FrF* tw_inv, unsigned long long* launches) {
  const uint32_t n = 1u << log_n;
  srs_bitrev_kernel<F><<<srs_blocks(n), 128, 0, st>>>(p, n, log_n);
  for (uint32_t h = 1; h < n; h *= 2) srs_butterfly_kernel<F, FrF><<<srs_blocks(n / 2), 128, 0, st>>>(p, n, h, tw_inv);
  if (launches) *launches += 1 + log_n;
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
  X cudaError_t srs_ifft<F, FrF>(cudaStream_t, XYZZ<F>*, int, const FrF*, unsigned long long*);                       \
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
