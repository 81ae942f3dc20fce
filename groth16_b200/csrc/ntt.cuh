// ntt.cuh -- radix-2 NTT / iNTT over Fr and the R1CS->QAP witness map on sm_90a.
//
// Replaces ark-poly 0.5.0 `Radix2EvaluationDomain::{fft,ifft}_in_place`, `get_coset`, `mul_polynomials_in_
// evaluation_domain` and `evaluate_vanishing_polynomial` as called from
// /root/reference/src/r1cs_to_qap.rs:172-235 (LibsnarkReduction::witness_map_from_matrices), and the sparse row
// evaluation `evaluate_constraint` (r1cs_to_qap.rs:28-67, called at :186-193 and :214-218).
// Conventions that the proving key bakes in and that therefore must match ark (SURVEY.md section 8c): the domain
// generator is TWO_ADIC_ROOT^(2^(s - log n)), constraint i <-> omega^i, natural order in and out.
//
// A transform of 2^L points is L decimation-in-frequency stages split into passes; each pass keeps a tile of 1024
// field elements in shared memory (limb-major, bank-conflict free), runs up to 10 stages on it and writes it back:
//   strided passes   tile = 2^k rows x C columns (C*32 B contiguous per row), k <= 7
//   last pass        tile = 1024 contiguous points, k <= 10; stores to the bit-reversed address so that the output is
//                    in natural order, with the n^-1 / coset scalings fused into that store
// The element-wise work of the witness map -- coset pre-scaling by g^i (r1cs_to_qap.rs:204-207), (a*b - c)/Z
// (r1cs_to_qap.rs:209,223-230), n^-1 g^-i (r1cs_to_qap.rs:232) -- is fused into the first-pass load / last-pass store.
#pragma once
#include <cuda_runtime.h>
#include "fp.cuh"

namespace g16 {

enum NttLoad { NTT_LOAD_PLAIN = 0, NTT_LOAD_MUL_TABLE = 1, NTT_LOAD_AB_MINUS_C = 2 };
enum NttStore { NTT_STORE_PLAIN = 0, NTT_STORE_MUL_CONST = 1, NTT_STORE_MUL_TABLE = 2 };

template <class Fr>
struct NttPass {
  const Fr* in;      // input (NTT_LOAD_AB_MINUS_C: the `a` vector)
  const Fr* in_b;    // AB_MINUS_C only
  const Fr* in_c;    // AB_MINUS_C only
  Fr* out;
  const Fr* tw;      // tw[i] = root^i, i < n/2
  const Fr* ltab;    // load table, natural index
  const Fr* stab;    // store table, natural (bit-reversed-address) index
  Fr lcst;           // AB_MINUS_C: Z^-1
  Fr scst;           // STORE_MUL_CONST: n^-1
  int L, s0, k, logC;
  int load_mode, store_mode;
  int bitrev_store;  // 1 on the last pass
};

template <class Fr>
__device__ __forceinline__ Fr ntt_ldg(const Fr* p) {
  Fr r;
  const uint4* s = reinterpret_cast<const uint4*>(p);
  uint4 a = __ldg(s), b = __ldg(s + 1);
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}
template <class Fr>
__device__ __forceinline__ void ntt_stg(Fr* p, const Fr& r) {
  uint4* d = reinterpret_cast<uint4*>(p);
  d[0] = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]);
  d[1] = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
}

static constexpr int NTT_TILE_LOG = 10;
static constexpr int NTT_TILE = 1 << NTT_TILE_LOG;

// One pass: stages s0 .. s0+k-1 of an L-stage DIF transform.  blockDim.x = min(256, tile/2).
template <class Fr>
__global__ void __launch_bounds__(256) ntt_pass_kernel(NttPass<Fr> a) {
  static_assert(Fr::N == 8, "Fr must be 8 x 32-bit limbs");
  __shared__ uint32_t sm[8][NTT_TILE];
  const int k = a.k, logC = a.logC;
  const uint32_t C = 1u << logC;
  const int tile_log = k + logC;
  const uint32_t tile = 1u << tile_log;
  const int low_bits = a.L - a.s0 - k;              // bits below the k transformed bits
  const uint32_t lowblks = 1u << (low_bits - logC);
  const uint32_t top = blockIdx.x / lowblks, lowblk = blockIdx.x % lowblks;
  const uint64_t gbase = ((uint64_t)top << (a.L - a.s0)) + ((uint64_t)lowblk << logC);
  const uint32_t T = blockDim.x;

  // ---- load ----
  for (uint32_t e = threadIdx.x; e < tile; e += T) {
    const uint32_t mid = e >> logC, cl = e & (C - 1);
    const uint64_t gi = gbase + ((uint64_t)mid << low_bits) + cl;
    Fr x = ntt_ldg(a.in + gi);
    if (a.load_mode == NTT_LOAD_MUL_TABLE) {
      x = Fr::mul(x, ntt_ldg(a.ltab + gi));
    } else if (a.load_mode == NTT_LOAD_AB_MINUS_C) {
      Fr y = ntt_ldg(a.in_b + gi), z = ntt_ldg(a.in_c + gi);
      x = Fr::mul(Fr::sub(Fr::mul(x, y), z), a.lcst);
    }
#pragma unroll
    for (int w = 0; w < 8; w++) sm[w][e] = x.v[w];
  }
  __syncthreads();

  // ---- k butterfly stages ----
  const uint32_t nbf = tile >> 1;
  for (int t = 0; t < k; t++) {
    const int hb = k - 1 - t;   // bit of `mid` that separates the pair
    const int s = a.s0 + t;     // global stage
    for (uint32_t bf = threadIdx.x; bf < nbf; bf += T) {
      const uint32_t cl = bf & (C - 1), mp = bf >> logC;
      const uint32_t mlow = mp & ((1u << hb) - 1);
      const uint32_t mid0 = ((mp >> hb) << (hb + 1)) | mlow;
      const uint32_t e0 = (mid0 << logC) | cl, e1 = e0 | (1u << (hb + logC));
      // twiddle exponent (j mod d) << s with d = 2^(L-s-1)
      const uint64_t jm = ((uint64_t)mlow << low_bits) + ((uint64_t)lowblk << logC) + cl;
      const Fr w = ntt_ldg(a.tw + (jm << s));
      Fr x0, x1;
#pragma unroll
      for (int q = 0; q < 8; q++) { x0.v[q] = sm[q][e0]; x1.v[q] = sm[q][e1]; }
      const Fr u = Fr::add(x0, x1);
      Fr v = Fr::sub(x0, x1);
      if (s != a.L - 1) v = Fr::mul(v, w);   // the last stage of a transform only has the twiddle omega^0 = 1
#pragma unroll
      for (int q = 0; q < 8; q++) { sm[q][e0] = u.v[q]; sm[q][e1] = v.v[q]; }
    }
    __syncthreads();
  }

  // ---- store ----
  for (uint32_t e = threadIdx.x; e < tile; e += T) {
    const uint32_t mid = e >> logC, cl = e & (C - 1);
    uint64_t gi = gbase + ((uint64_t)mid << low_bits) + cl;
    Fr x;
#pragma unroll
    for (int w = 0; w < 8; w++) x.v[w] = sm[w][e];
    if (a.bitrev_store && a.L > 0) gi = __brevll(gi) >> (64 - a.L);
    if (a.store_mode == NTT_STORE_MUL_CONST) x = Fr::mul(x, a.scst);
    else if (a.store_mode == NTT_STORE_MUL_TABLE) x = Fr::mul(x, ntt_ldg(a.stab + gi));
    ntt_stg(a.out + gi, x);
  }
}

// out[i] = c0 * base^i, i < n  (twiddle and coset tables)
template <class Fr>
__global__ void ntt_powers_kernel(Fr* out, uint64_t n, Fr base, Fr c0) {
  constexpr int RUN = 32;
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t i0 = t * RUN;
  if (i0 >= n) return;
  Fr x = Fr::mul(c0, Fr::pow_u64(base, i0));
  for (int j = 0; j < RUN && i0 + j < n; j++) {
    ntt_stg(out + i0 + j, x);
    x = Fr::mul(x, base);
  }
}

// Sparse rows times the assignment (evaluate_constraint, r1cs_to_qap.rs:28-67) for the three matrices at once,
// plus the instance copy a[nc + i] = z[i] (r1cs_to_qap.rs:195-199) and the zero tail up to the domain size.
struct CsrDev {
  const uint32_t* row_ptr;  // nc + 1
  const uint32_t* col;
  const void* val;          // Fr, Montgomery
};
template <class Fr>
__global__ void __launch_bounds__(256) r1cs_matvec_kernel(CsrDev A, CsrDev B, CsrDev Cm, const Fr* __restrict__ z,
                                                          uint32_t nc, uint32_t num_inputs, uint32_t n, Fr* a, Fr* b,
                                                          Fr* c) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr ra = Fr::zero(), rb = Fr::zero(), rc = Fr::zero();
  if (i < nc) {
    const CsrDev* ms[3] = {&A, &B, &Cm};
    Fr* outs[3] = {&ra, &rb, &rc};
#pragma unroll
    for (int m = 0; m < 3; m++) {
      const uint32_t lo = ms[m]->row_ptr[i], hi = ms[m]->row_ptr[i + 1];
      const Fr* vals = reinterpret_cast<const Fr*>(ms[m]->val);
      Fr acc = Fr::zero();
      for (uint32_t e = lo; e < hi; e++) acc = Fr::add(acc, Fr::mul(ntt_ldg(vals + e), ntt_ldg(z + ms[m]->col[e])));
      *outs[m] = acc;
    }
  } else if (i < nc + num_inputs) {
    ra = ntt_ldg(z + (i - nc));
  }
  ntt_stg(a + i, ra);
  ntt_stg(b + i, rb);
  ntt_stg(c + i, rc);
}

// ------------------------------------------------------------------------------------------------
// host side: per-size tables and transform drivers
// ------------------------------------------------------------------------------------------------
template <class Fr>
struct NttDomain {
  int L = -1;
  uint64_t n = 0;
  Fr* tw_fwd = nullptr;     // omega^i      i < n/2
  Fr* tw_inv = nullptr;     // omega^-i     i < n/2
  Fr* coset_fwd = nullptr;  // g^i          i < n
  Fr* coset_inv = nullptr;  // n^-1 g^-i    i < n
  Fr* coset_fwd_ninv = nullptr;  // n^-1 g^i  i < n: iFFT's n^-1 and the following coset pre-scaling in one multiplication
  Fr n_inv, z_inv;          // n^-1 ; (g^n - 1)^-1   (Montgomery form, host copies)
  Fr omega;
  void release() {
    if (tw_fwd) cudaFree(tw_fwd);
    if (tw_inv) cudaFree(tw_inv);
    if (coset_fwd) cudaFree(coset_fwd);
    if (coset_inv) cudaFree(coset_inv);
    if (coset_fwd_ninv) cudaFree(coset_fwd_ninv);
    tw_fwd = tw_inv = coset_fwd = coset_inv = coset_fwd_ninv = nullptr;
    L = -1;
  }
};

// Host-side field helpers (plain host back-end of Fp)
template <class Fr>
Fr fr_from_u64(uint64_t x) {
  Fr r = Fr::zero();
  r.v[0] = (uint32_t)x;
  r.v[1] = (uint32_t)(x >> 32);
  return Fr::to_mont(r);
}
template <class Fr>
Fr fr_generator() {
  Fr r;
  for (int i = 0; i < Fr::N; i++) r.v[i] = Fr::Params::generator(i);
  return r;
}
// omega = TWO_ADIC_ROOT^(2^(s - L))   (ark-ff get_root_of_unity, SURVEY.md section 2a)
template <class Fr>
Fr fr_domain_root(int L) {
  Fr r;
  for (int i = 0; i < Fr::N; i++) r.v[i] = Fr::Params::two_adic_root(i);
  for (int i = 0; i < Fr::Params::TWO_ADICITY - L; i++) r = Fr::sqr(r);
  return r;
}

template <class Fr>
cudaError_t ntt_domain_build(NttDomain<Fr>& d, int L, cudaStream_t st, unsigned long long* launches) {
  if (d.L == L) return cudaSuccess;
  d.release();
  d.n = 1ull << L;
  cudaError_t e;
  const uint64_t half = d.n > 1 ? d.n / 2 : 1;
  if ((e = cudaMalloc(&d.tw_fwd, half * sizeof(Fr))) != cudaSuccess) return e;
  if ((e = cudaMalloc(&d.tw_inv, half * sizeof(Fr))) != cudaSuccess) return e;
  if ((e = cudaMalloc(&d.coset_fwd, d.n * sizeof(Fr))) != cudaSuccess) return e;
  if ((e = cudaMalloc(&d.coset_inv, d.n * sizeof(Fr))) != cudaSuccess) return e;
  if ((e = cudaMalloc(&d.coset_fwd_ninv, d.n * sizeof(Fr))) != cudaSuccess) return e;
  const Fr omega = fr_domain_root<Fr>(L);
  const Fr omega_inv = Fr::inv(omega);
  const Fr g = fr_generator<Fr>();
  const Fr g_inv = Fr::inv(g);
  d.omega = omega;
  d.n_inv = Fr::inv(fr_from_u64<Fr>(d.n));
  // vanishing polynomial of the base domain at g: g^n - 1 (r1cs_to_qap.rs:223-226)
  Fr gn = g;
  for (int i = 0; i < L; i++) gn = Fr::sqr(gn);
  d.z_inv = Fr::inv(Fr::sub(gn, Fr::one()));
  auto launch = [&](Fr* out, uint64_t cnt, const Fr& base, const Fr& c0) {
    const uint64_t threads = (cnt + 31) / 32;
    ntt_powers_kernel<Fr><<<(unsigned)((threads + 127) / 128), 128, 0, st>>>(out, cnt, base, c0);
    if (launches) (*launches)++;
  };
  launch(d.tw_fwd, half, omega, Fr::one());
  launch(d.tw_inv, half, omega_inv, Fr::one());
  launch(d.coset_fwd, d.n, g, Fr::one());
  launch(d.coset_inv, d.n, g_inv, d.n_inv);
  launch(d.coset_fwd_ninv, d.n, g, d.n_inv);
  d.L = L;
  return cudaGetLastError();
}

struct NttPlan {
  int npass;
  int k[8];
  int logC[8];
};
inline NttPlan ntt_plan(int L) {
  NttPlan p;
  p.npass = 0;
  const int klast = L < NTT_TILE_LOG ? L : NTT_TILE_LOG;
  int rest = L - klast;
  if (rest > 0) {
    const int np = (rest + 6) / 7;
    for (int i = 0; i < np; i++) {
      const int ki = rest / np + (i < rest % np ? 1 : 0);
      p.k[p.npass] = ki;
      p.logC[p.npass] = NTT_TILE_LOG - ki;
      p.npass++;
    }
  }
  p.k[p.npass] = klast;
  p.logC[p.npass] = 0;
  p.npass++;
  return p;
}

// Full transform, natural order in -> natural order out.  `src` is read by the first pass only; `work` (n
// elements) carries the intermediate passes in place; the last pass scatters into `dst` (dst != work; dst may
// equal src when there is more than one pass).  For a single-pass transform src -> dst directly (dst != src).
template <class Fr>
void ntt_run(cudaStream_t st, const NttDomain<Fr>& d, bool inverse, const Fr* src, Fr* work, Fr* dst, int load_mode,
             const Fr* ltab, const Fr* in_b, const Fr* in_c, const Fr& load_cst, int store_mode, const Fr* stab,
             const Fr& store_cst, unsigned long long* launches) {
  const NttPlan p = ntt_plan(d.L);
  int s0 = 0;
  for (int i = 0; i < p.npass; i++) {
    NttPass<Fr> a;
    const bool first = i == 0, last = i == p.npass - 1;
    a.in = first ? src : work;
    a.in_b = in_b;
    a.in_c = in_c;
    a.out = last ? dst : work;
    a.tw = inverse ? d.tw_inv : d.tw_fwd;
    a.ltab = ltab;
    a.stab = stab;
    a.lcst = load_cst;
    a.scst = store_cst;
    a.L = d.L;
    a.s0 = s0;
    a.k = p.k[i];
    a.logC = p.logC[i];
    a.load_mode = first ? load_mode : NTT_LOAD_PLAIN;
    a.store_mode = last ? store_mode : NTT_STORE_PLAIN;
    a.bitrev_store = last ? 1 : 0;
    const int tile_log = a.k + a.logC;
    const uint64_t blocks = d.n >> tile_log;
    uint32_t threads = (1u << tile_log) / 2;
    if (threads > 256) threads = 256;
    if (threads < 32) threads = 32;
    ntt_pass_kernel<Fr><<<(unsigned)blocks, threads, 0, st>>>(a);
    if (launches) (*launches)++;
    s0 += a.k;
  }
}


template <class Fr>
void r1cs_matvec(cudaStream_t st, const CsrDev* cs, const Fr* z, uint32_t nc, uint32_t num_inputs, uint32_t n, Fr* a, Fr* b,
                 Fr* c) {
  r1cs_matvec_kernel<Fr><<<(n + 255) / 256, 256, 0, st>>>(cs[0], cs[1], cs[2], z, nc, num_inputs, n, a, b, c);
}

#define G16_NTT_TEMPLATES(X, Fr)                                                                                       \
  X void ntt_run<Fr>(cudaStream_t, const NttDomain<Fr>&, bool, const Fr*, Fr*, Fr*, int, const Fr*, const Fr*, const Fr*, \
                     const Fr&, int, const Fr*, const Fr&, unsigned long long*);                                       \
  X cudaError_t ntt_domain_build<Fr>(NttDomain<Fr>&, int, cudaStream_t, unsigned long long*);                          \
  X void r1cs_matvec<Fr>(cudaStream_t, const CsrDev*, const Fr*, uint32_t, uint32_t, uint32_t, Fr*, Fr*, Fr*);

}  // namespace g16
