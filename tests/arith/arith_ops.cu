// Element-level harness of the product arithmetic: one field, Fq2 or point operation per vector, run through the very
// templates of fp.cuh, ec.cuh, fp_inv.cuh and msm_ba.cuh (no copies of their code).  tests/test_arith_ops.py feeds it
// raw Montgomery limbs and compares every output with Python big integers.
//
// Built three ways from this one file:
//   nvcc (Makefile)             : libg16arith.so, one device thread per vector -- the PTX carry chains, the out-of-line
//                                 base-field product mont_mul_call and the __ldg loads of ba_ld, as the kernels run them
//   g++                         : the plain 64-bit host back-end, a loop over the vectors
//   g++ -DG16_EMULATE_PTX       : the device algorithm with the PTX carry primitives emulated in C
//
// ABI: g16t_shape(field, op, &in_words, &out_words) gives the fixed number of u32 words per vector; g16t_run(field, op,
// in, out, n) reads n * in_words and writes n * out_words words (host arrays).  Every check of the inputs is done by the
// caller; the library only refuses unknown (field, op) pairs and negative counts.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include "../../groth16_b200/csrc/msm_ba.cuh"

using namespace g16;

namespace {

// fields: 0..5 Fp (Fr, Fq of BLS12-381, BN254, BLS12-377), 6..8 Fq2 of the same three curves; the point ops run on G1
// (coordinates in fields 1, 3, 5) and G2 (fields 6, 7, 8)
enum Op {
  ADD = 0, SUB = 1, NEG = 2, DBL = 3, MUL = 4, SQR = 5, MUL_SMALL = 6, FROM_MONT = 7, TO_MONT = 8, POW_U64 = 9, INV = 10,
  INV_GCD = 11, MUL_NR = 12, BA_INV = 13,
  MADD = 20, MADD_NEG = 21, MADD_LAZY = 22, MADD_LAZY_NEG = 23, PADD = 24, PDBL = 25, PDBL_AFFINE = 26, PMUL_U32 = 27,
  TO_AFFINE = 28,
};
constexpr int NUM_FIELDS = 9;

template <class T>
G16_HD T ld(const uint32_t* p) {
  T t;
  uint32_t* d = reinterpret_cast<uint32_t*>(&t);
  for (int i = 0; i < (int)(sizeof(T) / 4); i++) d[i] = p[i];
  return t;
}
template <class T>
G16_HD void st(uint32_t* p, const T& t) {
  const uint32_t* s = reinterpret_cast<const uint32_t*>(&t);
  for (int i = 0; i < (int)(sizeof(T) / 4); i++) p[i] = s[i];
}

// Vector layouts (E = words of one coordinate):  XYZZ = X Y ZZ ZZZ (4E), affine = x y (2E), scalar = 8 words LE.
template <class F>
G16_HD bool point_op(int op, const uint32_t* in, uint32_t* out) {
  constexpr int E = sizeof(F) / 4;
  using X = XYZZ<F>;
  using A = Affine<F>;
  switch (op) {
    case MADD:
    case MADD_NEG: {
      X acc = ld<X>(in);
      acc.madd(ld<A>(in + 4 * E), op == MADD_NEG);
      st(out, acc);
      return true;
    }
    case MADD_LAZY:
    case MADD_LAZY_NEG: {   // the accumulation kernel's form: coordinates fetched on demand through ba_ld (__ldg)
      X acc = ld<X>(in);
      const A* p = reinterpret_cast<const A*>(in + 4 * E);
      acc.madd_lazy([&]() { return ba_ld(&p->x); }, [&]() { return ba_ld(&p->y); }, op == MADD_LAZY_NEG);
      st(out, acc);
      return true;
    }
    case PADD: {
      X acc = ld<X>(in);
      acc.add(ld<X>(in + 4 * E));
      st(out, acc);
      return true;
    }
    case PDBL: {
      X acc = ld<X>(in);
      acc.dbl_inplace();
      st(out, acc);
      return true;
    }
    case PDBL_AFFINE: st(out, X::dbl_affine(ld<A>(in))); return true;
    case PMUL_U32: st(out, ld<X>(in).mul_u32(in + 4 * E, 8)); return true;
    case TO_AFFINE: st(out, ld<X>(in).to_affine()); return true;
  }
  return false;
}

template <class P>
G16_HD bool fp_op(int op, const uint32_t* in, uint32_t* out) {
  using F = Fp<P>;
  constexpr int E = P::N;
  switch (op) {
    case ADD: st(out, F::add(ld<F>(in), ld<F>(in + E))); return true;
    case SUB: st(out, F::sub(ld<F>(in), ld<F>(in + E))); return true;
    case NEG: st(out, F::neg(ld<F>(in))); return true;
    case DBL: st(out, F::dbl(ld<F>(in))); return true;
    case MUL: st(out, F::mul(ld<F>(in), ld<F>(in + E))); return true;
    case SQR: st(out, F::sqr(ld<F>(in))); return true;
    case MUL_SMALL: st(out, F::mul_small(ld<F>(in), (int)in[E])); return true;
    case FROM_MONT: st(out, F::from_mont(ld<F>(in))); return true;
    case TO_MONT: st(out, F::to_mont(ld<F>(in))); return true;
    case POW_U64: st(out, F::pow_u64(ld<F>(in), (uint64_t)in[E] | (uint64_t)in[E + 1] << 32)); return true;
    case INV: st(out, F::inv(ld<F>(in))); return true;
    case INV_GCD: st(out, fp_inv_safegcd<P>(ld<F>(in))); return true;
  }
  if constexpr (is_base_field<P>()) return point_op<F>(op, in, out);
  return false;
}

template <class P, int NR>
G16_HD bool fq2_op(int op, const uint32_t* in, uint32_t* out) {
  using F = Fp2<P, NR>;
  constexpr int E = 2 * P::N;
  switch (op) {
    case ADD: st(out, F::add(ld<F>(in), ld<F>(in + E))); return true;
    case SUB: st(out, F::sub(ld<F>(in), ld<F>(in + E))); return true;
    case NEG: st(out, F::neg(ld<F>(in))); return true;
    case DBL: st(out, F::dbl(ld<F>(in))); return true;
    case MUL: st(out, F::mul(ld<F>(in), ld<F>(in + E))); return true;
    case SQR: st(out, F::sqr(ld<F>(in))); return true;
    case INV: st(out, F::inv(ld<F>(in))); return true;
    case MUL_NR: st(out, F::mul_nr(ld<Fp<P>>(in))); return true;
    case BA_INV: st(out, ba_inv(ld<F>(in), in[E] != 0)); return true;
  }
  return point_op<F>(op, in, out);
}

template <int FIELD>
G16_HD bool run_one(int op, const uint32_t* in, uint32_t* out) {
  if constexpr (FIELD == 0) return fp_op<BLS381_FrP>(op, in, out);
  else if constexpr (FIELD == 1) return fp_op<BLS381_FqP>(op, in, out);
  else if constexpr (FIELD == 2) return fp_op<BN254_FrP>(op, in, out);
  else if constexpr (FIELD == 3) return fp_op<BN254_FqP>(op, in, out);
  else if constexpr (FIELD == 4) return fp_op<BLS377_FrP>(op, in, out);
  else if constexpr (FIELD == 5) return fp_op<BLS377_FqP>(op, in, out);
  else if constexpr (FIELD == 6) return fq2_op<BLS381_FqP, BLS381_Params::FQ2_NONRESIDUE_NEG>(op, in, out);
  else if constexpr (FIELD == 7) return fq2_op<BN254_FqP, BN254_Params::FQ2_NONRESIDUE_NEG>(op, in, out);
  else return fq2_op<BLS377_FqP, BLS377_Params::FQ2_NONRESIDUE_NEG>(op, in, out);
}

// words per element of each field
constexpr int ELEM_WORDS[NUM_FIELDS] = {BLS381_FrP::N, BLS381_FqP::N, BN254_FrP::N, BN254_FqP::N, BLS377_FrP::N,
                                        BLS377_FqP::N, 2 * BLS381_FqP::N, 2 * BN254_FqP::N, 2 * BLS377_FqP::N};

#ifdef __CUDACC__
template <int FIELD>
__global__ void __launch_bounds__(128) arith_kernel(int op, const uint32_t* in, uint32_t* out, int64_t n, int iw, int ow) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  run_one<FIELD>(op, in + i * iw, out + i * ow);
}
template <int FIELD>
void exec(int op, const uint32_t* in, uint32_t* out, int64_t n, int iw, int ow) {   // in, out: device arrays
  arith_kernel<FIELD><<<(unsigned)((n + 127) / 128), 128>>>(op, in, out, n, iw, ow);
}
#else
template <int FIELD>
void exec(int op, const uint32_t* in, uint32_t* out, int64_t n, int iw, int ow) {
  for (int64_t i = 0; i < n; i++) run_one<FIELD>(op, in + i * iw, out + i * ow);
}
#endif

}  // namespace

extern "C" {

// 0 = plain host back-end, 1 = emulated PTX, 2 = device
int g16t_backend() {
#if defined(__CUDACC__)
  return 2;
#elif defined(G16_EMULATE_PTX)
  return 1;
#else
  return 0;
#endif
}

// words per vector of (field, op); returns -1 for a pair the harness does not run
int g16t_shape(int field, int op, int* in_words, int* out_words) {
  if (field < 0 || field >= NUM_FIELDS) return -1;
  const int E = ELEM_WORDS[field];
  const bool fp = field < 6, fq2 = field >= 6, curve = fq2 || (field & 1);
  int i = -1, o = E;
  switch (op) {
    case ADD: case SUB: case MUL: i = 2 * E; break;
    case NEG: case DBL: case SQR: case INV: i = E; break;
    case MUL_SMALL: if (fp) i = E + 1; break;
    case FROM_MONT: case TO_MONT: case INV_GCD: if (fp) i = E; break;
    case POW_U64: if (fp) i = E + 2; break;
    case MUL_NR: if (fq2) { i = E / 2; o = E / 2; } break;
    case BA_INV: if (fq2) i = E + 1; break;
    case MADD: case MADD_NEG: case MADD_LAZY: case MADD_LAZY_NEG: if (curve) { i = 6 * E; o = 4 * E; } break;
    case PADD: if (curve) { i = 8 * E; o = 4 * E; } break;
    case PDBL: if (curve) { i = 4 * E; o = 4 * E; } break;
    case PDBL_AFFINE: if (curve) { i = 2 * E; o = 4 * E; } break;
    case PMUL_U32: if (curve) { i = 4 * E + 8; o = 4 * E; } break;
    case TO_AFFINE: if (curve) { i = 4 * E; o = 2 * E; } break;
  }
  if (i < 0) return -1;
  *in_words = i;
  *out_words = o;
  return 0;
}

// 0 on success, -1 for an unknown (field, op) or a negative count, otherwise the CUDA error code
int g16t_run(int field, int op, const uint32_t* in, uint32_t* out, int64_t n) {
  int iw = 0, ow = 0;
  if (n < 0 || g16t_shape(field, op, &iw, &ow) != 0) return -1;
  if (n == 0) return 0;
  const size_t ib = (size_t)n * iw * 4, ob = (size_t)n * ow * 4;
  using Exec = void (*)(int, const uint32_t*, uint32_t*, int64_t, int, int);
  static const Exec table[NUM_FIELDS] = {exec<0>, exec<1>, exec<2>, exec<3>, exec<4>, exec<5>, exec<6>, exec<7>, exec<8>};
  const Exec run = table[field];
#ifdef __CUDACC__
  uint32_t *din = nullptr, *dout = nullptr;
  cudaError_t e = cudaMalloc(&din, ib);
  if (e == cudaSuccess) e = cudaMalloc(&dout, ob);
  if (e == cudaSuccess) e = cudaMemcpy(din, in, ib, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemset(dout, 0xff, ob);   // a vector the kernel skipped reads back as non-canonical
  if (e == cudaSuccess) {
    run(op, din, dout, n, iw, ow);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = cudaMemcpy(out, dout, ob, cudaMemcpyDeviceToHost);
  cudaFree(din);
  cudaFree(dout);
  return (int)e;
#else
  // 64-byte aligned copy: the point operands are read through Affine<F> / XYZZ<F> (alignas(16)) pointers
  uint32_t* buf = static_cast<uint32_t*>(aligned_alloc(64, (ib + 63) / 64 * 64));
  if (!buf) return -1;
  memcpy(buf, in, ib);
  memset(out, 0xff, ob);
  run(op, buf, out, n, iw, ow);
  free(buf);
  return 0;
#endif
}

}  // extern "C"
