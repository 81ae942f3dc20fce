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
// The same holds for ark-circom's CircomReduction: c = a o b is formed by the load of c's iFFT (NTT_LOAD_AB), the
// n^-1 omega_2n^i pre-scaling by the load of each forward transform, and h = A*B - C by the last-pass store of c's forward
// transform (NTT_STORE_AB_MINUS).  Those two modes live in a separate instantiation of the pass kernel (CIRCOM = true), so
// the kernel the libsnark reduction runs is compiled exactly as before.
#pragma once
#include <cuda_runtime.h>
#include "fp.cuh"

namespace g16 {

enum NttLoad { NTT_LOAD_PLAIN = 0, NTT_LOAD_MUL_TABLE = 1, NTT_LOAD_AB_MINUS_C = 2, NTT_LOAD_AB = 3 };
enum NttStore { NTT_STORE_PLAIN = 0, NTT_STORE_MUL_CONST = 1, NTT_STORE_MUL_TABLE = 2, NTT_STORE_AB_MINUS = 3 };
// NTT_LOAD_AB: x = in[i] * in_b[i] (natural index).  NTT_STORE_AB_MINUS: out[i] = st_a[i] * st_b[i] - x (natural index).
static inline bool ntt_circom_mode(int load_mode, int store_mode) {
  return load_mode == NTT_LOAD_AB || store_mode == NTT_STORE_AB_MINUS;
}

template <class Fr>
struct NttPass {
  const Fr* in;      // input (NTT_LOAD_AB_MINUS_C: the `a` vector)
  const Fr* in_b;    // AB_MINUS_C and AB only
  const Fr* in_c;    // AB_MINUS_C only
  Fr* out;
  const Fr* st_a;    // STORE_AB_MINUS only
  const Fr* st_b;
  const Fr* tw;      // tw[i] = root^i, i < n/2
  const Fr* ltab;    // load table, natural index
  const Fr* stab;    // store table, natural (bit-reversed-address) index
  Fr lcst;           // AB_MINUS_C: Z^-1
  Fr scst;           // STORE_MUL_CONST: n^-1
  int L, s0, k, logC;
  int load_mode, store_mode;
  int bitrev_store;  // 1 on the last pass
  uint64_t vstride;  // elements between the vectors of a batch: blockIdx.y selects in / in_b / in_c / out / st_a / st_b;
                     // tables are shared
};

template <class Fr>
__device__ __forceinline__ Fr ntt_ldg(const Fr* p) {
  Fr r;
  const uint4* s = reinterpret_cast<const uint4*>(p);
#pragma unroll
  for (int j = 0; j < Fr::N / 4; j++) {
    const uint4 a = __ldg(s + j);
    r.v[4 * j] = a.x; r.v[4 * j + 1] = a.y; r.v[4 * j + 2] = a.z; r.v[4 * j + 3] = a.w;
  }
  return r;
}
template <class Fr>
__device__ __forceinline__ void ntt_stg(Fr* p, const Fr& r) {
  uint4* d = reinterpret_cast<uint4*>(p);
#pragma unroll
  for (int j = 0; j < Fr::N / 4; j++) d[j] = make_uint4(r.v[4 * j], r.v[4 * j + 1], r.v[4 * j + 2], r.v[4 * j + 3]);
}

static constexpr int NTT_TILE_LOG = 10;
static constexpr int NTT_TILE = 1 << NTT_TILE_LOG;

// One pass: stages s0 .. s0+k-1 of an L-stage DIF transform.  blockDim.x = min(256, tile/2).
// CIRCOM = false: the libsnark load / store modes; CIRCOM = true: NTT_LOAD_AB / NTT_STORE_AB_MINUS (plus plain / table loads)
template <class Fr, bool CIRCOM>
__global__ void __launch_bounds__(256) ntt_pass_kernel(NttPass<Fr> a) {
  // 8 limbs (256-bit Fr): 32 KB of tile; 12 limbs (BW6-761's 377-bit Fr): 48 KB, the static shared-memory limit
  static_assert(Fr::N == 8 || Fr::N == 12, "Fr must be 8 or 12 x 32-bit limbs");
  __shared__ uint32_t sm[Fr::N][NTT_TILE];
  const int k = a.k, logC = a.logC;
  const uint32_t C = 1u << logC;
  const int tile_log = k + logC;
  const uint32_t tile = 1u << tile_log;
  const int low_bits = a.L - a.s0 - k;              // bits below the k transformed bits
  const uint32_t lowblks = 1u << (low_bits - logC);
  const uint32_t top = blockIdx.x / lowblks, lowblk = blockIdx.x % lowblks;
  const uint64_t gbase = ((uint64_t)top << (a.L - a.s0)) + ((uint64_t)lowblk << logC);
  const uint32_t T = blockDim.x;
  const uint64_t voff = blockIdx.y * a.vstride;

  // ---- load ----
  for (uint32_t e = threadIdx.x; e < tile; e += T) {
    const uint32_t mid = e >> logC, cl = e & (C - 1);
    const uint64_t gi = gbase + ((uint64_t)mid << low_bits) + cl;
    Fr x = ntt_ldg(a.in + voff + gi);
    if (a.load_mode == NTT_LOAD_MUL_TABLE) {
      x = Fr::mul(x, ntt_ldg(a.ltab + gi));
    } else if constexpr (CIRCOM) {
      if (a.load_mode == NTT_LOAD_AB) x = Fr::mul(x, ntt_ldg(a.in_b + voff + gi));
    } else if (a.load_mode == NTT_LOAD_AB_MINUS_C) {
      Fr y = ntt_ldg(a.in_b + voff + gi), z = ntt_ldg(a.in_c + voff + gi);
      x = Fr::mul(Fr::sub(Fr::mul(x, y), z), a.lcst);
    }
#pragma unroll
    for (int w = 0; w < Fr::N; w++) sm[w][e] = x.v[w];
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
      for (int q = 0; q < Fr::N; q++) { x0.v[q] = sm[q][e0]; x1.v[q] = sm[q][e1]; }
      const Fr u = Fr::add(x0, x1);
      Fr v = Fr::sub(x0, x1);
      if (s != a.L - 1) v = Fr::mul(v, w);   // the last stage of a transform only has the twiddle omega^0 = 1
#pragma unroll
      for (int q = 0; q < Fr::N; q++) { sm[q][e0] = u.v[q]; sm[q][e1] = v.v[q]; }
    }
    __syncthreads();
  }

  // ---- store ----
  for (uint32_t e = threadIdx.x; e < tile; e += T) {
    const uint32_t mid = e >> logC, cl = e & (C - 1);
    uint64_t gi = gbase + ((uint64_t)mid << low_bits) + cl;
    Fr x;
#pragma unroll
    for (int w = 0; w < Fr::N; w++) x.v[w] = sm[w][e];
    if (a.bitrev_store && a.L > 0) gi = __brevll(gi) >> (64 - a.L);
    if constexpr (CIRCOM) {
      if (a.store_mode == NTT_STORE_AB_MINUS) x = Fr::sub(Fr::mul(ntt_ldg(a.st_a + voff + gi), ntt_ldg(a.st_b + voff + gi)), x);
    } else {
      if (a.store_mode == NTT_STORE_MUL_CONST) x = Fr::mul(x, a.scst);
      else if (a.store_mode == NTT_STORE_MUL_TABLE) x = Fr::mul(x, ntt_ldg(a.stab + gi));
    }
    ntt_stg(a.out + voff + gi, x);
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
// blockIdx.y = proof k of a batch: it reads z + k * nv and writes a, b, c + k * n.
// WITH_C = false (CircomReduction, which never reads matrix C): only a and b; c is neither read nor written.
struct CsrDev {
  const uint32_t* row_ptr;  // nc + 1
  const uint32_t* col;
  const void* val;          // Fr, Montgomery
};
// <M_i, z>: row i of one CSR matrix times the assignment
template <class Fr>
__device__ __forceinline__ Fr r1cs_row_dot(const CsrDev& M, uint32_t i, const Fr* __restrict__ z) {
  const uint32_t lo = M.row_ptr[i], hi = M.row_ptr[i + 1];
  const Fr* vals = reinterpret_cast<const Fr*>(M.val);
  Fr acc = Fr::zero();
  for (uint32_t e = lo; e < hi; e++) acc = Fr::add(acc, Fr::mul(ntt_ldg(vals + e), ntt_ldg(z + M.col[e])));
  return acc;
}

template <class Fr, bool WITH_C>
__global__ void __launch_bounds__(256) r1cs_matvec_kernel(CsrDev A, CsrDev B, CsrDev Cm, const Fr* __restrict__ z,
                                                          uint32_t nc, uint32_t num_inputs, uint32_t n, Fr* a, Fr* b,
                                                          Fr* c, uint32_t nv) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  z += (size_t)blockIdx.y * nv;
  a += (size_t)blockIdx.y * n;
  b += (size_t)blockIdx.y * n;
  c += (size_t)blockIdx.y * n;
  Fr ra = Fr::zero(), rb = Fr::zero(), rc = Fr::zero();
  if (i < nc) {
    ra = r1cs_row_dot(A, i, z);
    rb = r1cs_row_dot(B, i, z);
    if (WITH_C) rc = r1cs_row_dot(Cm, i, z);
  } else if (i < nc + num_inputs) {
    ra = ntt_ldg(z + (i - nc));
  }
  ntt_stg(a + i, ra);
  ntt_stg(b + i, rb);
  if (WITH_C) ntt_stg(c + i, rc);
}

// The limbs of x, read as an integer, are >= the modulus: x is not a canonical field element
template <class Fr>
__device__ __forceinline__ bool fr_noncanonical(const Fr& x) {
  const Fr p = Fr::modulus();
  bool ge = true;   // equal so far
#pragma unroll
  for (int w = 0; w < Fr::N; w++) ge = x.v[w] > p.v[w] || (x.v[w] == p.v[w] && ge);   // little-endian limbs
  return ge;
}

// R1CS satisfiability of `count` assignments (ark-relations ConstraintSystem::is_satisfied / which_is_unsatisfied), one
// launch for rows and elements.  blockIdx.y = proof k: it reads z + k * nv and writes out[3k .. 3k + 2].
//   rows     thread i < nc: constraint i is unsatisfied when <A_i,z> <B_i,z> != <C_i,z> (values are fully reduced, so ==
//            compares them).  Only constraint rows: the instance rows the witness map appends are not constraints.
//   elements grid-stride over j < nv: z[j] is malformed when its limbs are >= r, z[0] also when it is not One.
// out[3k] = lowest unsatisfied row, out[3k + 1] = ~(unsatisfied rows), out[3k + 2] = lowest malformed element.  All three
// start at 0xffffffff (one memset), which is why the count is kept as its complement and counted down.  The lanes of a warp
// hold consecutive indices, so a warp's lowest index is its base plus the first set bit of its ballot: one atomic per warp
// and value.  Malformed limbs make the row values meaningless (the field operations assume inputs < p) but never an index:
// the columns were checked at g16_circuit_load.
template <class Fr>
__global__ void __launch_bounds__(256) r1cs_check_kernel(CsrDev A, CsrDev B, CsrDev Cm, const Fr* __restrict__ z,
                                                         uint32_t nc, uint32_t nv, uint32_t* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31;
  z += (size_t)blockIdx.y * nv;
  out += 3 * (size_t)blockIdx.y;
  const bool bad = i < nc && Fr::mul(r1cs_row_dot(A, i, z), r1cs_row_dot(B, i, z)) != r1cs_row_dot(Cm, i, z);
  const uint32_t rows = __ballot_sync(0xffffffffu, bad);
  if (rows && lane == 0) {
    atomicMin(out, i + __ffs(rows) - 1);
    atomicSub(out + 1, (uint32_t)__popc(rows));
  }
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t j0 = i - lane; j0 < nv; j0 += stride) {   // j0: the warp's base, so every lane runs the same iterations
    const uint64_t j = j0 + lane;
    bool mal = false;
    if (j < nv) {
      const Fr x = ntt_ldg(z + j);
      mal = j == 0 ? x != Fr::one() : fr_noncanonical(x);
    }
    const uint32_t els = __ballot_sync(0xffffffffu, mal);
    if (els) {   // later iterations of this warp only see higher indices
      if (lane == 0) atomicMin(out + 2, (uint32_t)j0 + __ffs(els) - 1);
      break;
    }
  }
}

// h[i] = a[i] * b[i] - c[i], i < n: the pointwise step of CircomReduction when a, b, c were transformed on different GPUs
template <class Fr>
__global__ void ntt_ab_minus_c_kernel(const Fr* a, const Fr* b, const Fr* c, Fr* h, uint64_t n) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ntt_stg(h + i, Fr::sub(Fr::mul(ntt_ldg(a + i), ntt_ldg(b + i)), ntt_ldg(c + i)));
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
  Fr* odd_fwd_ninv = nullptr;    // n^-1 omega_2n^i  i < n: the same for CircomReduction's odd-point evaluation (built on
                                 // demand by ntt_domain_build_odd, for a CircomReduction circuit only)
  Fr n_inv, z_inv;          // n^-1 ; (g^n - 1)^-1   (Montgomery form, host copies)
  Fr omega;
  void release() {
    if (tw_fwd) cudaFree(tw_fwd);
    if (tw_inv) cudaFree(tw_inv);
    if (coset_fwd) cudaFree(coset_fwd);
    if (coset_inv) cudaFree(coset_inv);
    if (coset_fwd_ninv) cudaFree(coset_fwd_ninv);
    if (odd_fwd_ninv) cudaFree(odd_fwd_ninv);
    tw_fwd = tw_inv = coset_fwd = coset_inv = coset_fwd_ninv = odd_fwd_ninv = nullptr;
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

// The table n^-1 omega_2n^i of a built domain (CircomReduction); the caller has checked that L + 1 <= the two-adicity
template <class Fr>
cudaError_t ntt_domain_build_odd(NttDomain<Fr>& d, cudaStream_t st, unsigned long long* launches) {
  if (d.odd_fwd_ninv) return cudaSuccess;
  cudaError_t e;
  if ((e = cudaMalloc(&d.odd_fwd_ninv, d.n * sizeof(Fr))) != cudaSuccess) return e;
  const uint64_t threads = (d.n + 31) / 32;
  ntt_powers_kernel<Fr><<<(unsigned)((threads + 127) / 128), 128, 0, st>>>(d.odd_fwd_ninv, d.n, fr_domain_root<Fr>(d.L + 1), d.n_inv);
  if (launches) (*launches)++;
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
// nvec > 1: the same transform of nvec vectors stored n elements apart in every buffer, one launch per pass.
template <class Fr>
void ntt_run(cudaStream_t st, const NttDomain<Fr>& d, bool inverse, const Fr* src, Fr* work, Fr* dst, int load_mode,
             const Fr* ltab, const Fr* in_b, const Fr* in_c, const Fr& load_cst, int store_mode, const Fr* stab,
             const Fr& store_cst, unsigned long long* launches, uint32_t nvec, const Fr* st_a, const Fr* st_b) {
  const NttPlan p = ntt_plan(d.L);
  int s0 = 0;
  for (int i = 0; i < p.npass; i++) {
    NttPass<Fr> a;
    const bool first = i == 0, last = i == p.npass - 1;
    a.in = first ? src : work;
    a.in_b = in_b;
    a.in_c = in_c;
    a.out = last ? dst : work;
    a.st_a = st_a;
    a.st_b = st_b;
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
    a.vstride = nvec > 1 ? d.n : 0;
    const int tile_log = a.k + a.logC;
    const uint64_t blocks = d.n >> tile_log;
    uint32_t threads = (1u << tile_log) / 2;
    if (threads > 256) threads = 256;
    if (threads < 32) threads = 32;
    const dim3 grid((unsigned)blocks, nvec > 1 ? nvec : 1u);
    if (ntt_circom_mode(a.load_mode, a.store_mode)) ntt_pass_kernel<Fr, true><<<grid, threads, 0, st>>>(a);
    else ntt_pass_kernel<Fr, false><<<grid, threads, 0, st>>>(a);
    if (launches) (*launches)++;
    s0 += a.k;
  }
}


// `count` assignments of nv elements each (z, contiguous) -> count row evaluations of n elements each (a, b and, with
// with_c, c)
template <class Fr>
void r1cs_matvec(cudaStream_t st, const CsrDev* cs, const Fr* z, uint32_t nc, uint32_t num_inputs, uint32_t n, Fr* a, Fr* b,
                 Fr* c, uint32_t count, uint32_t nv, bool with_c) {
  const dim3 grid((n + 255) / 256, count > 1 ? count : 1u);
  if (with_c) r1cs_matvec_kernel<Fr, true><<<grid, 256, 0, st>>>(cs[0], cs[1], cs[2], z, nc, num_inputs, n, a, b, c, nv);
  else r1cs_matvec_kernel<Fr, false><<<grid, 256, 0, st>>>(cs[0], cs[1], cs[2], z, nc, num_inputs, n, a, b, c, nv);
}

// Satisfiability of `count` assignments (z, nv elements apart) into out (count * 3 u32, device; see r1cs_check_kernel):
// the memset, then one launch per 65535 proofs (the grid-y limit)
static constexpr uint32_t R1CS_CHECK_MAX_Y = 65535;
template <class Fr>
cudaError_t r1cs_check(cudaStream_t st, const CsrDev* cs, const Fr* z, uint32_t nc, uint32_t nv, uint32_t count, uint32_t* out,
                       unsigned long long* launches) {
  cudaError_t e = cudaMemsetAsync(out, 0xff, (size_t)count * 3 * sizeof(uint32_t), st);
  if (e != cudaSuccess) return e;
  const unsigned bx = (nc > 0 ? (nc + 255) / 256 : 1u);
  for (uint32_t k = 0; k < count; k += R1CS_CHECK_MAX_Y) {
    const uint32_t ky = count - k < R1CS_CHECK_MAX_Y ? count - k : R1CS_CHECK_MAX_Y;
    r1cs_check_kernel<Fr><<<dim3(bx, ky), 256, 0, st>>>(cs[0], cs[1], cs[2], z + (size_t)k * nv, nc, nv, out + 3 * (size_t)k);
    if (launches) (*launches)++;
  }
  return cudaGetLastError();
}

// h = a o b - c over `count` vectors of n elements (one launch)
template <class Fr>
void ntt_ab_minus_c(cudaStream_t st, const Fr* a, const Fr* b, const Fr* c, Fr* h, uint64_t n) {
  ntt_ab_minus_c_kernel<Fr><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, b, c, h, n);
}

#define G16_NTT_TEMPLATES(X, Fr)                                                                                       \
  X void ntt_run<Fr>(cudaStream_t, const NttDomain<Fr>&, bool, const Fr*, Fr*, Fr*, int, const Fr*, const Fr*, const Fr*, \
                     const Fr&, int, const Fr*, const Fr&, unsigned long long*, uint32_t, const Fr*, const Fr*);       \
  X cudaError_t ntt_domain_build<Fr>(NttDomain<Fr>&, int, cudaStream_t, unsigned long long*);                          \
  X cudaError_t ntt_domain_build_odd<Fr>(NttDomain<Fr>&, cudaStream_t, unsigned long long*);                           \
  X void r1cs_matvec<Fr>(cudaStream_t, const CsrDev*, const Fr*, uint32_t, uint32_t, uint32_t, Fr*, Fr*, Fr*, uint32_t, uint32_t, \
                         bool);                                                                                         \
  X cudaError_t r1cs_check<Fr>(cudaStream_t, const CsrDev*, const Fr*, uint32_t, uint32_t, uint32_t, uint32_t*,            \
                               unsigned long long*);                                                                    \
  X void ntt_ab_minus_c<Fr>(cudaStream_t, const Fr*, const Fr*, const Fr*, Fr*, uint64_t);

}  // namespace g16
