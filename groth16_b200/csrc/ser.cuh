// ser.cuh -- ark-serialize 0.5 point encodings of a Groth16 ProvingKey, decoded and encoded on the GPU.
//
// The formats are exactly groth16_b200/serialize.py's (ArkCodec.point / read_point):
//   * BLS12-381: zcash / IETF, big-endian, three flag bits in the first byte (0x80 compressed, 0x40 infinity, 0x20 y is the
//     larger of +-y), Fq2 as c1 || c0;
//   * BN254, BLS12-377, BW6-761: generic short Weierstrass, little-endian, SWFlags in the two top bits of the last byte
//     (0x80 y > -y, 0x40 infinity), Fq2 as c0 || c1.  BW6-761's G2 is over Fq: its points are encoded like G1 points.
// A compressed point is x alone, an uncompressed one x || y.  Decoding checks what serialize.py checks: the flag bits, zero
// bytes under the infinity flag, canonical coordinates (< q), that a compressed x has a curve point, that an uncompressed
// point is on the curve, and with G16_SER_VALIDATE that [r]P = O (skipped for BN254 G1, whose cofactor is 1).
//
// ser_decode / ser_encode are per-point host/device functions (tests/test_ser_codec.py runs them, and ser_sqrt, point by
// point in the host, emulated-PTX and device builds of tests/arith/arith_ops.cu); the kernels
// run one thread per point.  The host walk of the stream and the chunk planner are at the end.
#pragma once
#include <algorithm>
#include <string>
#include <type_traits>
#include <vector>
#include "ec.cuh"

namespace g16 {

// per-point result codes; ser_reason() gives serialize.py's message for each
enum : uint32_t {
  SER_OK = 0,
  SER_ERR_COMPRESSION_FLAG = 1,
  SER_ERR_BOTH_FLAGS = 2,
  SER_ERR_INFINITY_BYTES = 3,
  SER_ERR_SORT_FLAG = 4,
  SER_ERR_NONCANONICAL = 5,
  SER_ERR_NO_ROOT = 6,
  SER_ERR_OFF_CURVE = 7,
  SER_ERR_SUBGROUP = 8
};
inline const char* ser_reason(uint32_t code) {
  switch (code) {
    case SER_ERR_COMPRESSION_FLAG: return "compression flag mismatch";
    case SER_ERR_BOTH_FLAGS: return "both SWFlags set";
    case SER_ERR_INFINITY_BYTES: return "non-zero bytes in the encoding of the point at infinity";
    case SER_ERR_SORT_FLAG: return "sort flag set on an uncompressed point";
    case SER_ERR_NONCANONICAL: return "non-canonical field element (>= q)";
    case SER_ERR_NO_ROOT: return "x is not the abscissa of a curve point";
    case SER_ERR_OFF_CURVE: return "point is not on the curve";
    case SER_ERR_SUBGROUP: return "point is not in the prime-order subgroup";
    default: return "unknown error";
  }
}
// the G16_SER_* flags of include/g16b200.h
enum : uint32_t { SER_COMPRESSED = 1, SER_VALIDATE = 2 };

template <class CP>
struct SerFormat {
  static constexpr bool ZCASH = CP::CURVE_ID == 0;                           // BLS12-381
  static constexpr int NB = 4 * CP::FqP::N;                                  // bytes per Fq: 48 (BLS12-*), 32 (BN254), 96 (BW6)
  static constexpr bool G1_COFACTOR_ONE = CP::CURVE_ID == 1;                 // BN254
  static constexpr int G2_NC = sizeof(typename CP::G2F) / sizeof(Fp<typename CP::FqP>);   // Fq per G2 coordinate: 2 or 1
  static_assert(ZCASH || NB * 8 >= CP::FqP::BITS + 2, "no room for the SWFlags");
  G16_HD static constexpr int point_bytes(bool g2, bool compress) { return NB * (g2 ? G2_NC : 1) * (compress ? 1 : 2); }
};

template <class CP, bool G2>
using SerField = typename std::conditional<G2, typename CP::G2F, Fp<typename CP::FqP>>::type;

// ---- canonical integers ----------------------------------------------------------------------------------------------
template <class P>
G16_HD Fp<P> ser_read_fq(const uint8_t* p, bool be) {
  Fp<P> r;
  constexpr int NB = 4 * P::N;
#pragma unroll
  for (int i = 0; i < P::N; i++) {
    uint32_t w = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) w |= (uint32_t)p[be ? NB - 1 - (4 * i + j) : 4 * i + j] << (8 * j);
    r.v[i] = w;
  }
  return r;
}
template <class P>
G16_HD void ser_write_fq(const Fp<P>& a, uint8_t* p, bool be) {
  constexpr int NB = 4 * P::N;
#pragma unroll
  for (int i = 0; i < P::N; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) p[be ? NB - 1 - (4 * i + j) : 4 * i + j] = (uint8_t)(a.v[i] >> (8 * j));
}
template <class P>
G16_HD bool ser_lt_mod(const Fp<P>& a) {   // a < q as integers
  for (int i = P::N - 1; i >= 0; i--)
    if (a.v[i] != P::mod(i)) return a.v[i] < P::mod(i);
  return false;
}
// y > -y in ark's ordering: canonical y > (q - 1) / 2; Fq2 compares c1 first, c0 when c1 = 0
template <class P>
G16_HD bool ser_neg_gt(const Fp<P>& y) {
  const Fp<P> c = Fp<P>::from_mont(y);
  for (int i = P::N - 1; i >= 0; i--) {
    const uint32_t h = (P::mod(i) >> 1) | (i + 1 < P::N ? P::mod(i + 1) << 31 : 0u);   // (q - 1) / 2, q odd
    if (c.v[i] != h) return c.v[i] > h;
  }
  return false;
}
template <class P, int NR>
G16_HD bool ser_neg_gt(const Fp2<P, NR>& y) { return y.c1.is_zero() ? ser_neg_gt(y.c0) : ser_neg_gt(y.c1); }

// ---- square roots -----------------------------------------------------------------------------------------------------
// Tonelli-Shanks data for fields with q = 1 mod 4: 2-adicity S of q - 1 and c = z^t (t = (q - 1) / 2^S, z the smallest
// quadratic non-residue), canonical limbs.  Only BLS12-377's Fq needs it (z = 5, S = 46).
template <class P>
struct SqrtTS {
  static constexpr int S = 0;
  G16_HD static constexpr uint32_t root(int) { return 0; }
};
template <>
struct SqrtTS<BLS377_FqP> {
  static constexpr int S = 46;
  G16_HD static constexpr uint32_t root(int i) {
    constexpr uint32_t t[12] = {0x6b00bbe8u, 0xba6b5ef2u, 0xcc795186u, 0x1ea03d28u, 0x56228ac4u, 0xc6eaa2bcu,
                                0x7022110eu, 0xd14fcacau, 0xaa914b0au, 0x8fe9dee6u, 0x99cdbc5du, 0x00382d3du};
    return t[i];
  }
};
// (q - 1) >> sh plus `add` (add = 1 only with sh = 2: (q + 1) / 4 = ((q - 1) >> 2) + 1 for q = 3 mod 4)
template <class P>
G16_HD void ser_exp_shift(uint32_t* e, int sh, uint32_t add) {
  uint32_t m[P::N];
  for (int i = 0; i < P::N; i++) m[i] = P::mod(i);
  m[0] -= 1;   // q odd: no borrow
  const int w = sh >> 5, b = sh & 31;
  for (int i = 0; i < P::N; i++) {
    const uint32_t lo = i + w < P::N ? m[i + w] : 0u, hi = i + w + 1 < P::N ? m[i + w + 1] : 0u;
    e[i] = b ? (lo >> b) | (hi << (32 - b)) : lo;
  }
  uint64_t c = add;
  for (int i = 0; i < P::N && c; i++) { c += e[i]; e[i] = (uint32_t)c; c >>= 32; }
}
// r^2 = a, or false.  q = 3 mod 4: r = a^((q+1)/4).  Otherwise Tonelli-Shanks with a fixed schedule: S - 1 rounds
// (k = S - 1 .. 1) of k - 1 squarings each and a conditional multiplication, whatever a is.
template <class P>
G16_HD bool ser_sqrt(const Fp<P>& a, Fp<P>& r) {
  using F = Fp<P>;
  uint32_t e[P::N];
  if constexpr ((P::mod(0) & 3u) == 3u) {
    ser_exp_shift<P>(e, 2, 1);
    r = F::pow(a, e, P::N);
  } else {
    constexpr int S = SqrtTS<P>::S;
    static_assert(S > 1, "no Tonelli-Shanks data for this field");
    ser_exp_shift<P>(e, S + 1, 0);                 // (t - 1) / 2
    const F w = F::pow(a, e, P::N);                // a^((t-1)/2)
    F x = F::mul(a, w);                            // a^((t+1)/2)
    F b = F::mul(x, w);                            // a^t
    F z;
    for (int i = 0; i < P::N; i++) z.v[i] = SqrtTS<P>::root(i);
    z = F::to_mont(z);                             // order 2^S
    // invariant before round k: b has order dividing 2^k (a square), z has order 2^(k+1), x^2 = a b
    for (int k = S - 1; k >= 1; k--) {
      F t = b;
      for (int j = 0; j < k - 1; j++) t = F::sqr(t);
      const bool fix = t != F::one();              // b of order exactly 2^k: multiply by z^2 of the same order
      const F z2 = F::sqr(z);
      const F x2 = F::mul(x, z), b2 = F::mul(b, z2);
      x = fix ? x2 : x;
      b = fix ? b2 : b;
      z = z2;
    }
    r = x;
  }
  return F::sqr(r) == a;
}
// complex method in Fq[u]/(u^2 + NR), as serialize.py's _Fq2.sqrt
template <class P, int NR>
G16_HD bool ser_sqrt(const Fp2<P, NR>& a, Fp2<P, NR>& r) {
  using B = Fp<P>;
  using F2 = Fp2<P, NR>;
  if (a.c1.is_zero()) {
    B t;
    if (ser_sqrt(a.c0, t)) { r = {t, B::zero()}; return true; }
    // a0 = -NR t^2: sqrt = t u
    const B m = NR == 1 ? B::neg(a.c0) : B::mul(a.c0, B::inv(B::neg(F2::mul_nr(B::one()))));
    if (ser_sqrt(m, t)) { r = {B::zero(), t}; return true; }
    return false;
  }
  const B norm = B::add(B::sqr(a.c0), F2::mul_nr(B::sqr(a.c1)));
  B alpha;
  if (!ser_sqrt(norm, alpha)) return false;
  B half;   // 1/2 = (q + 1) / 2
  ser_exp_shift<P>(half.v, 1, 1);
  half = B::to_mont(half);
  B x0;
  B delta = B::mul(B::add(a.c0, alpha), half);
  if (!ser_sqrt(delta, x0)) {
    delta = B::mul(B::sub(a.c0, alpha), half);
    if (!ser_sqrt(delta, x0)) return false;
  }
  const B x1 = B::mul(a.c1, B::inv(B::dbl(x0)));
  r = {x0, x1};
  return F2::sqr(r) == a;
}

// ---- curve data -----------------------------------------------------------------------------------------------------
// b of G1, or of G2 in G2's own coordinate field (twist_b0 alone when G2 is over Fq)
template <class CP, bool G2>
G16_HD SerField<CP, G2> ser_b() {
  SerField<CP, G2> b;
  if constexpr (!G2) {
    for (int i = 0; i < CP::FqP::N; i++) b.v[i] = CP::FqP::curve_b(i);
  } else if constexpr (SerFormat<CP>::G2_NC == 1) {
    for (int i = 0; i < CP::FqP::N; i++) b.v[i] = CP::FqP::twist_b0(i);
  } else {
    for (int i = 0; i < CP::FqP::N; i++) { b.c0.v[i] = CP::FqP::twist_b0(i); b.c1.v[i] = CP::FqP::twist_b1(i); }
  }
  return b;
}
// [r]P = O by left-to-right double-and-add over the bits of r in XYZZ.  XYZZ::madd / dbl_inplace handle every exceptional
// case the chain meets with small-order points (acc = P: doubling, acc = -P: identity, y = 0: doubling to the identity).
template <class FrP, class F>
G16_HD bool ser_in_subgroup(const Affine<F>& p) {
  XYZZ<F> acc = XYZZ<F>::inf();
  for (int i = FrP::BITS - 1; i >= 0; i--) {
    acc.dbl_inplace();
    if ((FrP::mod(i >> 5) >> (i & 31)) & 1u) acc.madd(p);
  }
  return acc.is_inf();
}

// wire value k of the point -> field element (G1: x = value 0, y = value 1; G2 over Fq2: two values each)
template <class CP, bool G2>
G16_HD SerField<CP, G2> ser_pick(const Fp<typename CP::FqP>* v, int k) {
  if constexpr (G2 && SerFormat<CP>::G2_NC == 2) {
    if (SerFormat<CP>::ZCASH) return {v[2 * k + 1], v[2 * k]};
    return {v[2 * k], v[2 * k + 1]};
  } else {
    return v[k];
  }
}

// ---- one point ------------------------------------------------------------------------------------------------------
// raw: the point's bytes (SerFormat<CP>::point_bytes(G2, flags & SER_COMPRESSED) of them).  Returns SER_OK and the affine
// Montgomery point (all-zero limbs for the identity), or the first failing check in serialize.py's order.
template <class CP, bool G2>
G16_HD uint32_t ser_decode(const uint8_t* raw, uint32_t flags, Affine<SerField<CP, G2>>& out) {
  using Fq = Fp<typename CP::FqP>;
  using F = SerField<CP, G2>;
  using Fmt = SerFormat<CP>;
  constexpr int NB = Fmt::NB, NC = G2 ? Fmt::G2_NC : 1, N = CP::FqP::N;
  const bool compress = flags & SER_COMPRESSED;
  const int nv = compress ? NC : 2 * NC;
  uint32_t fl;
  if (Fmt::ZCASH) {
    fl = raw[0] & 0xE0u;
    if (((fl & 0x80u) != 0) != compress) return SER_ERR_COMPRESSION_FLAG;
  } else {
    fl = raw[nv * NB - 1] & 0xC0u;
    if (fl == 0xC0u) return SER_ERR_BOTH_FLAGS;
  }
  Fq v[2 * NC];
  bool any = false;
#pragma unroll
  for (int k = 0; k < 2 * NC; k++) {
    if (k < nv) {
      v[k] = ser_read_fq<typename CP::FqP>(raw + k * NB, Fmt::ZCASH);
      if (Fmt::ZCASH && k == 0) v[k].v[N - 1] &= 0x1FFFFFFFu;       // the three flag bits
      if (!Fmt::ZCASH && k == nv - 1) v[k].v[N - 1] &= 0x3FFFFFFFu;  // the two SWFlags
      any |= !v[k].is_zero();
    } else {
      v[k] = Fq::zero();
    }
  }
  if (fl & 0x40u) {
    if (any || (Fmt::ZCASH && (fl & 0x20u))) return SER_ERR_INFINITY_BYTES;
    out = Affine<F>::inf();
    return SER_OK;
  }
  if (Fmt::ZCASH && !compress && (fl & 0x20u)) return SER_ERR_SORT_FLAG;
#pragma unroll
  for (int k = 0; k < 2 * NC; k++)
    if (k < nv && !ser_lt_mod(v[k])) return SER_ERR_NONCANONICAL;
#pragma unroll
  for (int k = 0; k < 2 * NC; k++) v[k] = Fq::to_mont(v[k]);
  const F x = ser_pick<CP, G2>(v, 0);
  const F rhs = F::add(F::mul(F::sqr(x), x), ser_b<CP, G2>());
  F y;
  if (compress) {
    if (!ser_sqrt(rhs, y)) return SER_ERR_NO_ROOT;
    const bool neg = Fmt::ZCASH ? (fl & 0x20u) : (fl & 0x80u);
    if (ser_neg_gt(y) != neg) y = F::neg(y);
  } else {
    y = ser_pick<CP, G2>(v, 1);
    if (F::sqr(y) != rhs) return SER_ERR_OFF_CURVE;
  }
  out = Affine<F>{x, y};
  if ((flags & SER_VALIDATE) && !(!G2 && Fmt::G1_COFACTOR_ONE) && !ser_in_subgroup<typename CP::FrP>(out))
    return SER_ERR_SUBGROUP;
  return SER_OK;
}

// snarkjs .zkey points (zkey.cuh): every coordinate n8q = NB little-endian bytes already in Montgomery form (R = 2^(8 NB),
// which is the ABI's R), G1 x || y, G2 x.c0 || x.c1 || y.c0 || y.c1 on every curve; the identity is all-zero bytes.  No flag
// bits and no multiplication by R^2; otherwise the decisions of ser_decode: canonical coordinates (< q), on the curve, and
// with SER_VALIDATE [r]P = O.
template <class CP, bool G2>
G16_HD uint32_t ser_decode_mont(const uint8_t* raw, uint32_t flags, Affine<SerField<CP, G2>>& out) {
  using Fq = Fp<typename CP::FqP>;
  using F = SerField<CP, G2>;
  using Fmt = SerFormat<CP>;
  constexpr int NB = Fmt::NB, NC = G2 ? Fmt::G2_NC : 1;
  Fq v[2 * NC];
  bool any = false;
#pragma unroll
  for (int k = 0; k < 2 * NC; k++) {
    v[k] = ser_read_fq<typename CP::FqP>(raw + k * NB, false);
    any |= !v[k].is_zero();
  }
  if (!any) {
    out = Affine<F>::inf();
    return SER_OK;
  }
#pragma unroll
  for (int k = 0; k < 2 * NC; k++)
    if (!ser_lt_mod(v[k])) return SER_ERR_NONCANONICAL;
  F x, y;
  if constexpr (G2 && NC == 2) {
    x = {v[0], v[1]};
    y = {v[2], v[3]};
  } else {
    x = v[0];
    y = v[1];
  }
  if (F::sqr(y) != F::add(F::mul(F::sqr(x), x), ser_b<CP, G2>())) return SER_ERR_OFF_CURVE;
  out = Affine<F>{x, y};
  if ((flags & SER_VALIDATE) && !(!G2 && Fmt::G1_COFACTOR_ONE) && !ser_in_subgroup<typename CP::FrP>(out))
    return SER_ERR_SUBGROUP;
  return SER_OK;
}

// the point's encoding, exactly ArkCodec.point
template <class CP, bool G2>
G16_HD void ser_encode(const Affine<SerField<CP, G2>>& p, uint32_t flags, uint8_t* out) {
  using Fq = Fp<typename CP::FqP>;
  using Fmt = SerFormat<CP>;
  constexpr int NB = Fmt::NB, NC = G2 ? Fmt::G2_NC : 1;
  const bool compress = flags & SER_COMPRESSED;
  const int nv = compress ? NC : 2 * NC;
  const int size = nv * NB;
  if (p.is_inf()) {
    for (int i = 0; i < size; i++) out[i] = 0;
    if (Fmt::ZCASH) out[0] = (compress ? 0x80 : 0) | 0x40;
    else out[size - 1] = 0x40;
    return;
  }
  Fq v[2 * NC];
  if constexpr (NC == 2) {
    const Fq xs[4] = {p.x.c0, p.x.c1, p.y.c0, p.y.c1};
#pragma unroll
    for (int k = 0; k < 4; k++) v[Fmt::ZCASH ? (k ^ 1) : k] = xs[k];
  } else {
    v[0] = p.x;
    v[1] = p.y;
  }
#pragma unroll
  for (int k = 0; k < 2 * NC; k++)
    if (k < nv) ser_write_fq(Fq::from_mont(v[k]), out + k * NB, Fmt::ZCASH);
  const bool neg = ser_neg_gt(p.y);
  if (Fmt::ZCASH) {
    if (compress) out[0] |= 0x80 | (neg ? 0x20 : 0);
  } else if (neg) {
    out[size - 1] |= 0x80;   // set on uncompressed points too, as ark does
  }
}

// ---- where a decoded point goes -------------------------------------------------------------------------------------
// Element i of a query vector is MSM pair i - skip (skip = 1 for a / b queries, whose element 0 goes to the proof tail);
// pairs below `pairs` (the query truncated to the circuit) are dealt round-robin: rank j mod world keeps pair j in slot
// j / world.  Returns that slot for the point this rank keeps, -1 otherwise.
G16_HD int64_t ser_slot(uint64_t i, uint64_t skip, uint64_t pairs, uint32_t rank, uint32_t world) {
  if (i < skip) return -1;
  const uint64_t j = i - skip;
  if (j >= pairs || j % world != rank) return -1;
  return (int64_t)(j / world);
}
struct SerDest {
  void* bases = nullptr;                 // Affine<F>[...]: this rank's MSM slots (copy 0), or null
  uint64_t skip = 0, pairs = 0;
  uint32_t rank = 0, world = 1;
  void* aux = nullptr;                   // Affine<F>[aux_n]: elements 0 .. aux_n - 1 also land here (read back by the host)
  uint64_t aux_n = 0;
};

#ifdef __CUDACC__
// MONT: the .zkey encoding of ser_decode_mont (flags holds SER_VALIDATE at most) instead of the ark encodings
template <class CP, bool G2, bool MONT = false>
__global__ void __launch_bounds__(128) ser_decode_kernel(const uint8_t* src, uint64_t first, uint32_t count, uint32_t flags,
                                                         uint64_t off0, SerDest d, unsigned long long* err) {
  using A = Affine<SerField<CP, G2>>;
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= count) return;
  const uint32_t psize = SerFormat<CP>::point_bytes(G2, flags & SER_COMPRESSED);
  A p;
  uint32_t code;
  if constexpr (MONT) code = ser_decode_mont<CP, G2>(src + (uint64_t)t * psize, flags, p);
  else code = ser_decode<CP, G2>(src + (uint64_t)t * psize, flags, p);
  if (code) {   // the smallest (byte offset, code) is the first bad point in stream order
    atomicMin(err, ((off0 + (uint64_t)t * psize) << 8) | code);
    return;
  }
  const uint64_t i = first + t;
  if (i < d.aux_n) static_cast<A*>(d.aux)[i] = p;
  const int64_t s = ser_slot(i, d.skip, d.pairs, d.rank, d.world);
  if (s >= 0 && d.bases) static_cast<A*>(d.bases)[s] = p;
}
template <class CP, bool G2>
__global__ void __launch_bounds__(128) ser_encode_kernel(const Affine<SerField<CP, G2>>* src, uint32_t count, uint32_t flags,
                                                         uint8_t* out) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= count) return;
  const uint32_t psize = SerFormat<CP>::point_bytes(G2, flags & SER_COMPRESSED);
  ser_encode<CP, G2>(src[t], flags, out + (uint64_t)t * psize);
}
template <class CP, bool G2, bool MONT = false>
cudaError_t ser_decode_enqueue(cudaStream_t st, const uint8_t* src, uint64_t first, uint32_t count, uint32_t flags,
                               uint64_t off0, SerDest d, unsigned long long* err) {
  if (!count) return cudaSuccess;
  ser_decode_kernel<CP, G2, MONT><<<(count + 127) / 128, 128, 0, st>>>(src, first, count, flags, off0, d, err);
  return cudaGetLastError();
}
template <class CP, bool G2>
cudaError_t ser_encode_enqueue(cudaStream_t st, const void* src, uint32_t count, uint32_t flags, uint8_t* out) {
  if (!count) return cudaSuccess;
  ser_encode_kernel<CP, G2><<<(count + 127) / 128, 128, 0, st>>>(static_cast<const Affine<SerField<CP, G2>>*>(src), count,
                                                                 flags, out);
  return cudaGetLastError();
}
#define G16_SER_TEMPLATES(X, CP)                                                                                       \
  X cudaError_t ser_decode_enqueue<CP, false>(cudaStream_t, const uint8_t*, uint64_t, uint32_t, uint32_t, uint64_t,     \
                                              SerDest, unsigned long long*);                                            \
  X cudaError_t ser_decode_enqueue<CP, true>(cudaStream_t, const uint8_t*, uint64_t, uint32_t, uint32_t, uint64_t,      \
                                             SerDest, unsigned long long*);                                             \
  X cudaError_t ser_encode_enqueue<CP, false>(cudaStream_t, const void*, uint32_t, uint32_t, uint8_t*);                 \
  X cudaError_t ser_encode_enqueue<CP, true>(cudaStream_t, const void*, uint32_t, uint32_t, uint8_t*);
#endif

// ---- the stream: ProvingKey in derive order (data_structures.rs:125) -------------------------------------------------
// vk {alpha_g1, beta_g2, gamma_g2, delta_g2, gamma_abc_g1}, beta_g1, delta_g1, a_query, b_g1_query, b_g2_query, h_query,
// l_query.  Vectors are a u64 little-endian length and their points.
enum { SER_ALPHA_G1 = 0, SER_BETA_G2, SER_GAMMA_G2, SER_DELTA_G2, SER_GAMMA_ABC, SER_BETA_G1, SER_DELTA_G1, SER_A, SER_B_G1,
       SER_B_G2, SER_H, SER_L, SER_ITEMS };
struct SerItem {
  const char* name;
  bool g2, vec;
  uint64_t len = 1;    // points
  uint64_t off = 0;    // byte offset of the first point (after the length prefix of a vector)
  uint32_t psize = 0;  // bytes per point
};
static constexpr uint64_t SER_MAX_VEC = 1ull << 28;   // ArkCodec.MAX_VEC: absurd length prefixes are refused

inline void ser_items(SerItem it[SER_ITEMS]) {
  const SerItem t[SER_ITEMS] = {{"vk.alpha_g1", false, false}, {"vk.beta_g2", true, false}, {"vk.gamma_g2", true, false},
                                {"vk.delta_g2", true, false},  {"vk.gamma_abc_g1", false, true}, {"beta_g1", false, false},
                                {"delta_g1", false, false},    {"a_query", false, true},   {"b_g1_query", false, true},
                                {"b_g2_query", true, true},    {"h_query", false, true},   {"l_query", false, true}};
  for (int i = 0; i < SER_ITEMS; i++) it[i] = t[i];
}
// Walks the structure from the length prefixes alone (every point has a fixed size once the flag is known): fills
// it[].len / off / psize and returns "" or why the stream is malformed (truncated, trailing bytes, absurd prefix).
// g2_nc: Fq elements per G2 coordinate (SerFormat::G2_NC).
inline std::string ser_walk(const uint8_t* bytes, uint64_t len, int nb, bool compress, SerItem it[SER_ITEMS], int g2_nc = 2) {
  ser_items(it);
  uint64_t pos = 0;
  for (int m = 0; m < SER_ITEMS; m++) {
    SerItem& x = it[m];
    x.psize = (uint32_t)(nb * (x.g2 ? g2_nc : 1) * (compress ? 1 : 2));
    if (x.vec) {
      if (len - pos < 8)
        return std::string("truncated input: wanted 8 bytes, got ") + std::to_string(len - pos) + " (length of " + x.name + ")";
      uint64_t n = 0;
      for (int k = 0; k < 8; k++) n |= (uint64_t)bytes[pos + k] << (8 * k);
      if (n > SER_MAX_VEC) return std::string("vector length ") + std::to_string(n) + " exceeds the limit (" + x.name + ")";
      x.len = n;
      pos += 8;
    }
    x.off = pos;
    if ((len - pos) / x.psize < x.len) {
      const uint64_t i = (len - pos) / x.psize;
      return std::string("truncated input: wanted ") + std::to_string(x.psize) + " bytes, got " +
             std::to_string(len - pos - i * x.psize) + " (" + x.name + "[" + std::to_string(i) + "])";
    }
    pos += x.len * x.psize;
  }
  if (pos != len) return "trailing bytes after the proving key";
  return "";
}
// total size of a key with these lengths (g16_pk_export_serialized)
inline uint64_t ser_size(SerItem it[SER_ITEMS], int nb, bool compress, int g2_nc = 2) {
  uint64_t pos = 0;
  for (int m = 0; m < SER_ITEMS; m++) {
    SerItem& x = it[m];
    x.psize = (uint32_t)(nb * (x.g2 ? g2_nc : 1) * (compress ? 1 : 2));
    if (x.vec) pos += 8;
    x.off = pos;
    pos += x.len * x.psize;
  }
  return pos;
}
// Decode / encode work in chunks of at most `chunk` points; a chunk never spans two members.
struct SerChunk {
  int member;
  uint64_t first;    // index of its first point within the member
  uint32_t count;
  uint64_t off;      // byte offset of its first point in the stream
};
inline std::vector<SerChunk> ser_plan(const SerItem it[SER_ITEMS], uint32_t chunk) {
  std::vector<SerChunk> out;
  for (int m = 0; m < SER_ITEMS; m++)
    for (uint64_t f = 0; f < it[m].len; f += chunk)
      out.push_back({m, f, (uint32_t)std::min<uint64_t>(chunk, it[m].len - f), it[m].off + f * it[m].psize});
  return out;
}
// the member and index of the point that starts at byte `off`
inline std::string ser_locate(const SerItem it[SER_ITEMS], uint64_t off) {
  for (int m = SER_ITEMS - 1; m >= 0; m--)
    if (off >= it[m].off && it[m].len)
      return std::string(it[m].name) + "[" + std::to_string((off - it[m].off) / it[m].psize) + "]";
  return "?";
}

}  // namespace g16
