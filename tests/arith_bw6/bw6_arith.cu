// Element-level harness of BW6-761's arithmetic: the 12-limb Fr and the 24-limb Fq of fp.cuh, the safegcd inversion of
// fp_inv.cuh and the XYZZ point operations of ec.cuh over that Fq (G1 and G2 share them), run through the product's own
// templates.  tests/test_bw6_arith.py feeds raw Montgomery limbs at carry-chain edge operands and compares every output with
// Python big integers.
//
// Built three ways from this one file:
//   nvcc (Makefile)        : libg16bw6arith.so, one device thread per vector -- the PTX carry chains and the out-of-line
//                            base-field product mont_mul_call, as the kernels run them
//   g++                    : the plain 64-bit CIOS host back-end
//   g++ -DG16_EMULATE_PTX  : the device algorithm with the PTX carry primitives emulated in C
//
// ABI: bw6t_shape(field, op, &in_words, &out_words) gives the u32 words per vector; bw6t_run(field, op, in, out, n) reads
// n * in_words and writes n * out_words words (host arrays).  Returns 0, or -1 for an unknown (field, op) or a CUDA failure.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include "../../groth16_b200/csrc/ec.cuh"
#include "../../groth16_b200/csrc/fp_inv.cuh"
#ifdef __CUDACC__
#include <cuda_runtime.h>
#endif

using namespace g16;

namespace {

// fields: 0 = Fr (12 limbs), 1 = Fq (24 limbs); point ops need field 1
enum Op {
  ADD = 0, SUB = 1, NEG = 2, DBL = 3, MUL = 4, SQR = 5, FROM_MONT = 6, TO_MONT = 7, INV = 8, INV_GCD = 9,
  MADD = 20, MADD_LAZY = 21, PADD = 22, PDBL = 23,
};
using Fr = Fp<BW6_FrP>;
using Fq = Fp<BW6_FqP>;

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

// field ops: in = a || b, out = result.  Point ops (Fq): in = XYZZ P || (affine Q || padding, or XYZZ Q), out = XYZZ.
template <class F>
G16_HD bool field_op(int op, const uint32_t* in, uint32_t* out) {
  constexpr int E = sizeof(F) / 4;
  const F a = ld<F>(in), b = ld<F>(in + E);
  F r;
  switch (op) {
    case ADD: r = F::add(a, b); break;
    case SUB: r = F::sub(a, b); break;
    case NEG: r = F::neg(a); break;
    case DBL: r = F::dbl(a); break;
    case MUL: r = F::mul(a, b); break;
    case SQR: r = F::sqr(a); break;
    case FROM_MONT: r = F::from_mont(a); break;
    case TO_MONT: r = F::to_mont(a); break;
    case INV: r = F::inv(a); break;
    case INV_GCD: r = fp_inv_safegcd<typename F::Params>(a); break;
    default: return false;
  }
  st(out, r);
  return true;
}
G16_HD bool point_op(int op, const uint32_t* in, uint32_t* out) {
  constexpr int E = sizeof(Fq) / 4;
  using X = XYZZ<Fq>;
  using A = Affine<Fq>;
  X acc = ld<X>(in);
  switch (op) {
    case MADD: acc.madd(ld<A>(in + 4 * E)); break;
    case MADD_LAZY: {
      const A q = ld<A>(in + 4 * E);
      acc.madd_lazy([&]() { return q.x; }, [&]() { return q.y; }, false);
      break;
    }
    case PADD: acc.add(ld<X>(in + 4 * E)); break;
    case PDBL: acc.dbl_inplace(); break;
    default: return false;
  }
  st(out, acc);
  return true;
}
G16_HD bool run_one(int field, int op, const uint32_t* in, uint32_t* out) {
  if (op >= MADD) return field == 1 && point_op(op, in, out);
  return field == 0 ? field_op<Fr>(op, in, out) : field_op<Fq>(op, in, out);
}
bool shape(int field, int op, int* iw, int* ow) {
  if (field != 0 && field != 1) return false;
  const int E = field == 0 ? Fr::N : Fq::N;
  if (op >= MADD) {
    if (field != 1 || op > PDBL) return false;
    *iw = 8 * E;
    *ow = 4 * E;
    return true;
  }
  if (op < ADD || op > INV_GCD) return false;
  *iw = 2 * E;
  *ow = E;
  return true;
}

#ifdef __CUDACC__
__global__ void __launch_bounds__(64) bw6_kernel(int field, int op, const uint32_t* in, uint32_t* out, int64_t n, int iw, int ow) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) run_one(field, op, in + i * iw, out + i * ow);
}
#endif

}  // namespace

extern "C" {
int bw6t_shape(int field, int op, int* in_words, int* out_words) { return shape(field, op, in_words, out_words) ? 0 : -1; }
int bw6t_run(int field, int op, const uint32_t* in, uint32_t* out, int64_t n) {
  int iw = 0, ow = 0;
  if (n < 0 || !shape(field, op, &iw, &ow)) return -1;
#ifdef __CUDACC__
  if (n == 0) return 0;
  uint32_t *din = nullptr, *dout = nullptr;
  const size_t ib = (size_t)n * iw * 4, ob = (size_t)n * ow * 4;
  cudaError_t e = cudaMalloc(&din, ib);
  if (e == cudaSuccess) e = cudaMalloc(&dout, ob);
  if (e == cudaSuccess) e = cudaMemcpy(din, in, ib, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    bw6_kernel<<<(unsigned)((n + 63) / 64), 64>>>(field, op, din, dout, n, iw, ow);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpy(out, dout, ob, cudaMemcpyDeviceToHost);
  if (din) cudaFree(din);
  if (dout) cudaFree(dout);
  return e == cudaSuccess ? 0 : -1;
#else
  for (int64_t i = 0; i < n; i++) run_one(field, op, in + i * iw, out + i * ow);
  return 0;
#endif
}
}  // extern "C"
