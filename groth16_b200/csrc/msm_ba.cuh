// msm_ba.cuh -- batched-affine pre-reduction of the sorted bucket entries (default for large MSMs since round 2).
//
// The bucket accumulation of msm.cuh spends 10 field multiplications per entry (XYZZ mixed addition).  An affine
// addition costs 3 once the inverse of (x2 - x1) is known, and Montgomery's trick shares one inversion between any
// number of independent additions at 3 more multiplications each.  Inside one bucket the entries can be summed as a
// binary tree, and every level of that tree is a set of independent additions.
//
// Layout (round 2: REGULAR, no per-round offset tables and no bucket search): the counting sort pads every bucket to a
// multiple of 2^R slots (msm_scan_blocks pads the histogram, msm_pad_fill marks the unused slots empty), so that
//
//   round r:  list_r (length M >> r, M = padded number of sorted slots)  ->  list_{r+1},  out[j] = in[2j] + in[2j+1]
//
// never pairs entries of different buckets, slot j of list_r belongs to the bucket of sorted slot j << r, and every
// list of rounds >= 1 is read and written with unit stride.  Empty slots are the point at infinity: (0,0) in a list,
// MSM_INVALID in the sorted index array of round 0.  The padding costs < 2^R / 2 slots per bucket (1.5 % of the entries
// for R = 4 at 2^20 pairs).  After R rounds 1 - 2^-R of all additions are done and the last list goes through
// msm_accum_l0 (key of slot j = skey[j << R]).  One round is three launches:
//   forward : thread t owns outputs j = k*T + t (k < m): d_j = x2 - x1, exclusive running product -> pre[j],
//             thread product -> prod[t]
//   combine : lane g owns G thread products: Montgomery's trick over them, ONE inversion per lane (safegcd, fp_inv.cuh),
//             prod[t] <- prod[t]^-1
//   backward: thread t walks its outputs in reverse, recovers 1/d_j, finishes the additions, writes list_{r+1}
// = 6 multiplications per addition + (3 + inv/G)/m for the combine.
//
// Every per-thread body below is __host__ __device__ and free of warp intrinsics, so tests/host/ba_check.cu runs
// the same code on the CPU against plain XYZZ sums (exceptional cases included: equal points, opposite points,
// identities in the lists, empty slots).
#pragma once
#include "ec.cuh"
#include "fp_inv.cuh"

namespace g16 {

static constexpr uint32_t BA_EMPTY = 0xffffffffu;   // == MSM_INVALID: sorted slot without an entry (bucket padding)

template <class F>
struct BaRound {
  const Affine<F>* in;       // round 0: base table (gathered through sidx); later: the previous list
  const uint32_t* sidx;      // round 0 only: (base index | sign << 31) per sorted slot, BA_EMPTY = no entry; nullptr afterwards
  const uint32_t* total0;    // device: padded number of sorted slots M (a multiple of 2^R)
  uint32_t shift;            // this round's OUTPUT list has M >> shift slots (round r: shift = r + 1)
  uint32_t m;                // outputs per thread
  uint32_t G;                // thread products per combine lane
  uint32_t inv_gcd;          // combine: 1 = safegcd inversion (fp_inv.cuh), 0 = Fermat
  F* pre;                    // [outputs]  running product of the thread before output j
  F* prod;                   // [threads]  thread product, then its inverse
  F* pre2;                   // [threads]  running product of the lane before thread t
  Affine<F>* out;            // [outputs]
};

G16_HD uint64_t ba_threads(uint64_t outputs, uint32_t m) { return (outputs + m - 1) / m; }

template <class F>
G16_HD F ba_ld(const F* p) {
#ifdef __CUDA_ARCH__
  F v;
  const uint4* s = reinterpret_cast<const uint4*>(p);
  uint4* d = reinterpret_cast<uint4*>(&v);
#pragma unroll
  for (int j = 0; j < (int)(sizeof(F) / 16); j++) d[j] = __ldg(s + j);
  return v;
#else
  return *p;
#endif
}

// where input i of the round lives, and whether its y is to be negated; p == nullptr: empty slot (identity)
template <class F>
struct BaSrc {
  const Affine<F>* p;
  bool neg;
};
template <class F>
G16_HD BaSrc<F> ba_src(const BaRound<F>& a, uint64_t i) {
  if (a.sidx) {
    const uint32_t ix = a.sidx[i];
    if (ix == BA_EMPTY) return {nullptr, false};
    return {a.in + (ix & 0x7fffffffu), (ix >> 31) != 0};
  }
  return {a.in + i, false};
}
template <class F>
G16_HD F ba_x(const BaSrc<F>& s) { return s.p ? ba_ld(&s.p->x) : F::zero(); }
template <class F>
G16_HD F ba_y(const BaSrc<F>& s) {
  if (!s.p) return F::zero();
  F y = ba_ld(&s.p->y);
  return s.neg ? F::neg(y) : y;
}

// kind of a pair: 0 chord (d = x2 - x1), 1 tangent (d = 2 y1), 2 result = P1, 3 result = P2, 4 result = identity
enum { BA_CHORD = 0, BA_TANGENT = 1, BA_FIRST = 2, BA_SECOND = 3, BA_INF = 4 };
template <class F>
G16_HD int ba_classify(const F& x1, const F& y1, const F& x2, const F& y2, F& d) {
  const bool inf1 = x1.is_zero() && y1.is_zero(), inf2 = x2.is_zero() && y2.is_zero();
  if (inf1) return inf2 ? BA_INF : BA_SECOND;
  if (inf2) return BA_FIRST;
  if (x1 == x2) {
    if (y1 == y2 && !y1.is_zero()) { d = F::dbl(y1); return BA_TANGENT; }
    return BA_INF;
  }
  d = F::sub(x2, x1);
  return BA_CHORD;
}
// common case decided from the x coordinates alone (both finite, different abscissae); everything else looks at y too
template <class F>
G16_HD int ba_kind(const BaSrc<F>& s1, const BaSrc<F>& s2, const F& x1, const F& x2, F& d) {
  if (x1.is_zero() || x2.is_zero() || x1 == x2) return ba_classify(x1, ba_y(s1), x2, ba_y(s2), d);
  d = F::sub(x2, x1);
  return BA_CHORD;
}

template <class F>
G16_HD void ba_forward(const BaRound<F>& a, uint64_t t) {
  const uint64_t M = (uint64_t)(*a.total0) >> a.shift;
  const uint64_t T = ba_threads(M, a.m);
  if (t >= T) return;
  F run = F::one();
  uint64_t j = t;
  if (j < M) {
    BaSrc<F> s1 = ba_src(a, 2 * j), s2 = ba_src(a, 2 * j + 1);
    F x1 = ba_x(s1), x2 = ba_x(s2);
    for (uint32_t k = 0; k < a.m; k++) {
      // operands of the next output are requested before this output's product is formed
      const uint64_t jn = j + T;
      const bool more = k + 1 < a.m && jn < M;
      BaSrc<F> n1{nullptr, false}, n2{nullptr, false};
      F nx1 = F::zero(), nx2 = F::zero();
      if (more) { n1 = ba_src(a, 2 * jn); n2 = ba_src(a, 2 * jn + 1); nx1 = ba_x(n1); nx2 = ba_x(n2); }
      F d;
      const int kind = ba_kind(s1, s2, x1, x2, d);
      a.pre[j] = run;
      if (kind <= BA_TANGENT) run = F::mul(run, d);
      if (!more) break;
      j = jn; s1 = n1; s2 = n2; x1 = nx1; x2 = nx2;
    }
  }
  a.prod[t] = run;
}

// the one inversion of a combine lane
template <class P>
G16_HD Fp<P> ba_inv(const Fp<P>& a, bool gcd) { return gcd ? fp_inv_safegcd<P>(a) : Fp<P>::inv(a); }
template <class P, int NR>
G16_HD Fp2<P, NR> ba_inv(const Fp2<P, NR>& a, bool gcd) {
  using B = Fp<P>;
  const B n = B::add(B::sqr(a.c0), Fp2<P, NR>::mul_nr(B::sqr(a.c1)));
  const B ni = ba_inv(n, gcd);
  return {B::mul(a.c0, ni), B::neg(B::mul(a.c1, ni))};
}

template <class F>
G16_HD void ba_combine(const BaRound<F>& a, uint64_t g) {
  const uint64_t M = (uint64_t)(*a.total0) >> a.shift;
  const uint64_t T = ba_threads(M, a.m);
  const uint64_t lo = g * a.G;
  if (lo >= T) return;
  const uint64_t hi = (lo + a.G < T) ? lo + a.G : T;
  F acc = F::one();
  for (uint64_t k = lo; k < hi; k++) {
    a.pre2[k] = acc;
    acc = F::mul(acc, a.prod[k]);
  }
  F inv = ba_inv(acc, a.inv_gcd != 0);   // never zero: every factor is x2 - x1 != 0, 2 y1 != 0 or one
  for (uint64_t k = hi; k-- > lo;) {
    const F pk = a.prod[k];
    a.prod[k] = F::mul(inv, a.pre2[k]);
    inv = F::mul(inv, pk);
  }
}

// Operands are consumed as early as possible (x2 and y2 are folded into x1 + x2, x2 - x1 and y2 - y1 and dropped
// before the multiplications start): the Fq2 instantiation then fits in 254 registers without spilling.
template <class F>
G16_HD void ba_backward(const BaRound<F>& a, uint64_t t) {
  const uint64_t M = (uint64_t)(*a.total0) >> a.shift;
  const uint64_t T = ba_threads(M, a.m);
  if (t >= T) return;
  F run_inv = a.prod[t];
  uint32_t kn = 0;   // outputs of this thread
  while (kn < a.m && (uint64_t)kn * T + t < M) kn++;
  for (uint32_t k = kn; k-- > 0;) {
    const uint64_t j = (uint64_t)k * T + t;
    const BaSrc<F> s1 = ba_src(a, 2 * j), s2 = ba_src(a, 2 * j + 1);
    Affine<F> r;
    r.x = ba_x(s1);
    F sx, d;                        // x1 + x2 and the denominator
    int kind;
    {
      const F x2 = ba_x(s2);
      kind = ba_kind(s1, s2, r.x, x2, d);
      sx = F::add(r.x, x2);
    }
    if (kind <= BA_TANGENT) {
      F lam = F::mul(run_inv, a.pre[j]);           // 1 / d
      run_inv = F::mul(run_inv, d);
      r.y = ba_y(s1);
      if (kind == BA_CHORD) {
        lam = F::mul(F::sub(ba_y(s2), r.y), lam);
      } else {
        const F xx = F::sqr(r.x);
        lam = F::mul(F::add(F::dbl(xx), xx), lam);
      }
      const F x3 = F::sub(F::sqr(lam), sx);        // tangent: sx = 2 x1
      r.y = F::sub(F::mul(lam, F::sub(r.x, x3)), r.y);
      r.x = x3;
    } else if (kind == BA_FIRST) {
      r.y = ba_y(s1);
    } else if (kind == BA_SECOND) {
      r.x = ba_x(s2);
      r.y = ba_y(s2);
    } else {
      r = Affine<F>::inf();
    }
    a.out[j] = r;
  }
}

#ifdef __CUDACC__
// Resident blocks per SM the register allocation aims at: narrow points ask for 3 and get 4 (~125 registers); wide points
// (MsmWide: Fq2, BW6-761's Fq) 2 = the whole backward body in 254 registers (8 warps per SM).
template <class F>
struct BaCfg { static constexpr int MIN_BLOCKS = MsmWide<F>::value ? 2 : 3; };
template <class F>
__global__ void __launch_bounds__(128, BaCfg<F>::MIN_BLOCKS) ba_forward_kernel(BaRound<F> a) {
  ba_forward<F>(a, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
template <class F>
__global__ void __launch_bounds__(32) ba_combine_kernel(BaRound<F> a) {
  ba_combine<F>(a, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
template <class F>
__global__ void __launch_bounds__(128, BaCfg<F>::MIN_BLOCKS) ba_backward_kernel(BaRound<F> a) {
  ba_backward<F>(a, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
#endif  // __CUDACC__

}  // namespace g16
