// ec.cuh -- Fq2 tower and short-Weierstrass (a = 0) group arithmetic for the MSM kernels and host assembly.
//
// Replaces the ark-ec 0.5.0 arithmetic that /root/reference reaches through `E::G1::msm_bigint` /
// `E::G2::msm_bigint` (prover.rs:66,74,262) and the projective sums at prover.rs:76-131.
// Accumulators use XYZZ coordinates (x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2, identity <=> ZZ == 0):
// mixed addition 8M+2S, full addition 12M+2S, doubling 6M+3S -- fewer multiplications than Jacobian, and the
// group element (hence the affine proof, prover.rs:127-131) is representation-independent.
// Affine points are packed x||y in Montgomery form; the point at infinity is encoded x = y = 0 (never on any
// of the three curves since b != 0), SURVEY.md section 8b.
#pragma once
#include "fp.cuh"

// Point operations are compiled as real (non-inlined) device functions: one body per field instead of one per call
// site keeps ptxas time and code size sane (an Fq2 point addition is ~17k SASS instructions); the call overhead is
// a few percent of a 10..14-multiplication operation.  The bucket-accumulation kernel alone inlines its mixed add.
#ifdef __CUDACC__
#define G16_HD_NOINLINE __host__ __device__ __noinline__
#else
#define G16_HD_NOINLINE
#endif

namespace g16 {

// ------------------------------------------------------------------------------------------------
// Fq2 = Fq[u]/(u^2 + NR), NR = 1 (BLS12-381, BN254) or 5 (BLS12-377)
// ------------------------------------------------------------------------------------------------
template <class P, int NR>
struct alignas(16) Fp2 {
  using B = Fp<P>;
  B c0, c1;
  G16_HD static Fp2 zero() { return {B::zero(), B::zero()}; }
  G16_HD static Fp2 one() { return {B::one(), B::zero()}; }
  G16_HD bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
  G16_HD bool operator==(const Fp2& o) const { return c0 == o.c0 && c1 == o.c1; }
  G16_HD bool operator!=(const Fp2& o) const { return !(*this == o); }
  G16_HD static Fp2 add(const Fp2& a, const Fp2& b) { return {B::add(a.c0, b.c0), B::add(a.c1, b.c1)}; }
  G16_HD static Fp2 sub(const Fp2& a, const Fp2& b) { return {B::sub(a.c0, b.c0), B::sub(a.c1, b.c1)}; }
  G16_HD static Fp2 neg(const Fp2& a) { return {B::neg(a.c0), B::neg(a.c1)}; }
  G16_HD static Fp2 dbl(const Fp2& a) { return {B::dbl(a.c0), B::dbl(a.c1)}; }
  G16_HD static B mul_nr(const B& a) { return NR == 1 ? a : B::mul_small(a, NR); }
  // Karatsuba: 3 base multiplications
  G16_HD static Fp2 mul(const Fp2& a, const Fp2& b) {
    B v0 = B::mul(a.c0, b.c0);
    B v1 = B::mul(a.c1, b.c1);
    B s = B::mul(B::add(a.c0, a.c1), B::add(b.c0, b.c1));
    Fp2 r;
    r.c0 = B::sub(v0, mul_nr(v1));
    r.c1 = B::sub(B::sub(s, v0), v1);
    return r;
  }
  // (a0 + a1 u)^2 = (a0 + a1)(a0 - NR a1) + (NR - 1) a0 a1  +  2 a0 a1 u : 2 base multiplications
  G16_HD static Fp2 sqr(const Fp2& a) {
    B t = B::mul(a.c0, a.c1);
    B s = B::mul(B::add(a.c0, a.c1), B::sub(a.c0, mul_nr(a.c1)));
    Fp2 r;
    r.c0 = (NR == 1) ? s : B::add(s, B::mul_small(t, NR - 1));
    r.c1 = B::dbl(t);
    return r;
  }
  G16_HD static Fp2 mul_small(const Fp2& a, int k) { return {B::mul_small(a.c0, k), B::mul_small(a.c1, k)}; }
  G16_HD static Fp2 inv(const Fp2& a) {
    B n = B::add(B::sqr(a.c0), mul_nr(B::sqr(a.c1)));
    B ni = B::inv(n);
    return {B::mul(a.c0, ni), B::neg(B::mul(a.c1, ni))};
  }
};

// Wide points: coordinates of 96 bytes, Fq2 over a 384-bit Fq (every G2) or BW6-761's 761-bit Fq (its G1 and G2 alike).
// They set the register budget and the load pattern of the MSM accumulation and batched-affine kernels (msm.cuh,
// msm_ba.cuh).
template <class F>
struct MsmWide { static constexpr bool value = false; };
template <class P, int NR>
struct MsmWide<Fp2<P, NR>> { static constexpr bool value = true; };
template <>
struct MsmWide<Fp<BW6_FqP>> { static constexpr bool value = true; };

// ------------------------------------------------------------------------------------------------
// Points
// ------------------------------------------------------------------------------------------------
template <class F>
struct alignas(16) Affine {
  F x, y;
  G16_HD bool is_inf() const { return x.is_zero() && y.is_zero(); }
  G16_HD static Affine inf() { return {F::zero(), F::zero()}; }
};

template <class F>
struct alignas(16) XYZZ {
  F X, Y, ZZ, ZZZ;
  G16_HD bool is_inf() const { return ZZ.is_zero(); }
  G16_HD static XYZZ inf() { return {F::zero(), F::zero(), F::zero(), F::zero()}; }
  G16_HD static XYZZ from_affine(const Affine<F>& p) {
    if (p.is_inf()) return inf();
    return {p.x, p.y, F::one(), F::one()};
  }

  // 2 * (affine p)        mdbl-2008-s-1
  G16_HD_NOINLINE static XYZZ dbl_affine(const Affine<F>& p) {
    if (p.is_inf() || p.y.is_zero()) return inf();
    F U = F::dbl(p.y);
    F V = F::sqr(U);
    F W = F::mul(U, V);
    F S = F::mul(p.x, V);
    F XX = F::sqr(p.x);
    F M = F::add(F::dbl(XX), XX);
    XYZZ r;
    r.X = F::sub(F::sqr(M), F::dbl(S));
    r.Y = F::sub(F::mul(M, F::sub(S, r.X)), F::mul(W, p.y));
    r.ZZ = V;
    r.ZZZ = W;
    return r;
  }
  // 2 * this              dbl-2008-s-1 (a = 0)
  G16_HD_NOINLINE void dbl_inplace() {
    if (is_inf()) return;
    if (Y.is_zero()) { *this = inf(); return; }
    F U = F::dbl(Y);
    F V = F::sqr(U);
    F W = F::mul(U, V);
    F S = F::mul(X, V);
    F XX = F::sqr(X);
    F M = F::add(F::dbl(XX), XX);
    F X3 = F::sub(F::sqr(M), F::dbl(S));
    F Y3 = F::sub(F::mul(M, F::sub(S, X3)), F::mul(W, Y));
    X = X3;
    Y = Y3;
    ZZ = F::mul(V, ZZ);
    ZZZ = F::mul(W, ZZZ);
  }
  // this += affine p  (p.y negated first when neg)      madd-2008-s, all exceptional cases handled
  G16_HD_NOINLINE void madd(const Affine<F>& p_in, bool neg = false) { madd_inline(p_in, neg); }
  G16_HD void madd_inline(const Affine<F>& p_in, bool neg = false) {
    if (p_in.is_inf()) return;
    Affine<F> p = p_in;
    if (neg) p.y = F::neg(p.y);
    if (is_inf()) {
      X = p.x; Y = p.y; ZZ = F::one(); ZZZ = F::one();
      return;
    }
    F Pd = F::sub(F::mul(p.x, ZZ), X);
    F R = F::sub(F::mul(p.y, ZZZ), Y);
    if (Pd.is_zero()) {
      if (R.is_zero()) *this = dbl_affine(p);
      else *this = inf();
      return;
    }
    F PP = F::sqr(Pd);
    F PPP = F::mul(Pd, PP);
    F Q = F::mul(X, PP);
    F X3 = F::sub(F::sub(F::sqr(R), PPP), F::dbl(Q));
    Y = F::sub(F::mul(R, F::sub(Q, X3)), F::mul(Y, PPP));
    X = X3;
    ZZ = F::mul(ZZ, PP);
    ZZZ = F::mul(ZZZ, PPP);
  }
  // Same mixed addition with the point's coordinates fetched on demand (x first, y only after x has been consumed):
  // shortens the live range of the 2 x 12 (G1) / 2 x 24 (G2) limb operand in the register-bound accumulation kernel.
  // LX(), LY() return the coordinates; the point is known not to be the identity mask-wise but may still be (0,0).
  template <class LX, class LY>
  G16_HD void madd_lazy(LX load_x, LY load_y, bool neg) {
    const F px = load_x();
    if (is_inf()) {
      F py = load_y();
      if (px.is_zero() && py.is_zero()) return;
      if (neg) py = F::neg(py);
      X = px; Y = py; ZZ = F::one(); ZZZ = F::one();
      return;
    }
    const F Pd = F::sub(F::mul(px, ZZ), X);
    F py = load_y();
    if (px.is_zero() && py.is_zero()) return;
    if (neg) py = F::neg(py);
    const F R = F::sub(F::mul(py, ZZZ), Y);
    if (Pd.is_zero()) {
      if (R.is_zero()) *this = dbl_affine(Affine<F>{px, py});
      else *this = inf();
      return;
    }
    const F PP = F::sqr(Pd);
    const F PPP = F::mul(Pd, PP);
    const F Q = F::mul(X, PP);
    const F X3 = F::sub(F::sub(F::sqr(R), PPP), F::dbl(Q));
    Y = F::sub(F::mul(R, F::sub(Q, X3)), F::mul(Y, PPP));
    X = X3;
    ZZ = F::mul(ZZ, PP);
    ZZZ = F::mul(ZZZ, PPP);
  }
  // this += q             add-2008-s, all exceptional cases handled
  G16_HD_NOINLINE void add(const XYZZ& q) {
    if (q.is_inf()) return;
    if (is_inf()) { *this = q; return; }
    F U1 = F::mul(X, q.ZZ);
    F U2 = F::mul(q.X, ZZ);
    F S1 = F::mul(Y, q.ZZZ);
    F S2 = F::mul(q.Y, ZZZ);
    F Pd = F::sub(U2, U1);
    F R = F::sub(S2, S1);
    if (Pd.is_zero()) {
      if (R.is_zero()) dbl_inplace();
      else *this = inf();
      return;
    }
    F PP = F::sqr(Pd);
    F PPP = F::mul(Pd, PP);
    F Q = F::mul(U1, PP);
    F X3 = F::sub(F::sub(F::sqr(R), PPP), F::dbl(Q));
    Y = F::sub(F::mul(R, F::sub(Q, X3)), F::mul(S1, PPP));
    X = X3;
    ZZ = F::mul(F::mul(ZZ, q.ZZ), PP);
    ZZZ = F::mul(F::mul(ZZZ, q.ZZZ), PPP);
  }
  G16_HD void negate() { Y = F::neg(Y); }

  // this * k for a little-endian u32 scalar of nl limbs (left-to-right double-and-add)
  G16_HD_NOINLINE XYZZ mul_u32(const uint32_t* k, int nl) const {
    XYZZ r = inf();
    bool started = false;
    for (int i = nl * 32 - 1; i >= 0; i--) {
      if (started) r.dbl_inplace();
      if ((k[i >> 5] >> (i & 31)) & 1) {
        r.add(*this);
        started = true;
      }
    }
    return r;
  }
  // canonical affine form (one inversion); ark `into_affine`, prover.rs:127-131
  G16_HD_NOINLINE Affine<F> to_affine() const {
    if (is_inf()) return Affine<F>::inf();
    F zi = F::inv(ZZZ);            // 1/Z^3
    F z = F::mul(zi, ZZ);          // 1/Z
    F zi2 = F::sqr(z);             // 1/Z^2
    return {F::mul(X, zi2), F::mul(Y, zi)};
  }
};

}  // namespace g16
