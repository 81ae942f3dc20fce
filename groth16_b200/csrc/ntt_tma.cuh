// ntt_tma.cuh -- radix-2 NTT passes on 128 KB shared-memory tiles moved by TMA (sm_90a), for transforms of 2^14 points up.
//
// Same mathematics and conventions as ntt.cuh (ark-poly Radix2EvaluationDomain as called at
// /root/reference/src/r1cs_to_qap.rs:201-207,220-221,232; natural order in and out, L decimation-in-frequency stages), a
// different data movement.  A transform of 2^L points is ceil((L-10)/10) STRIDED passes followed by one LAST pass:
//
//   strided pass (stages s0 .. s0+k-1, k <= 10): the array is the matrix [R = 2^(s0+k) rows][W = 2^(L-s0-k) columns] of
//       32-byte elements; a CTA owns the tile rows seg*2^k .. +2^k  x  columns cb*C .. +C  with C = 4096 / 2^k: 4096
//       elements = 128 KB.  The tile is fetched as 2-D boxes by cp.async.bulk.tensor (TMA, completion on an mbarrier), the
//       k stages run on it in shared memory, and it is written back in place by TMA stores.  At L = 20 this is ONE pass with
//       k = 10, C = 4 (128-byte row segments).
//   last pass (stages L-10 .. L-1): a CTA owns FOUR contiguous 1024-point blocks b, b + N/4, b + 2N/4, b + 3N/4
//       (N = 2^(L-10) blocks), fetched by four 32 KB bulk copies (cp.async.bulk, TMA 1-D).  After the ten stages the
//       transform's output lives at the bit-reversed index: element e of block b + j N/4 belongs at
//       brev10(e) * N + brev(b) * 4 + brev2(j) -- for the four blocks together that is a 1024-row x 4-column box of the
//       [1024][N] output matrix.  An in-place 12-bit bit-reversal permutation of the tile (swaps) puts the tile in exactly
//       that box layout, and the box is written by TMA stores.  No scattered 32-byte stores, no separate transpose.
//
// Traffic per transform at 2^20: 2 passes x (read + write) = 4 x 32 MiB (the three-pass plan of ntt.cuh moves 6 x).
// The element-wise work of the witness map stays fused: coset scaling / (a*b - c) * Z^-1 after the first pass's load,
// n^-1 / n^-1 g^-i scaling before the last pass's store (r1cs_to_qap.rs:204-209,223-232).
// Twiddles: strided passes read omega^((i mod d) << s) from the domain's table (L2-resident); the last pass needs only the
// 512 powers of the 1024-th root and keeps them in shared memory.
#pragma once
#include <cuda.h>            // CUtensorMap (types only: the encoder is fetched through the runtime, libcuda is not linked)
#include <cuda_runtime.h>
#include "ntt.cuh"

namespace g16 {

static constexpr int NTT2_TILE_LOG = 12;                  // 4096 elements = 128 KB
static constexpr int NTT2_TILE = 1 << NTT2_TILE_LOG;
static constexpr int NTT2_LAST_LOG = 10;                  // the last pass transforms 1024-point blocks
static constexpr int NTT2_THREADS = 512;
static constexpr int NTT2_MIN_L = 14;

// ---- PTX wrappers (sm_90+ TMA / mbarrier) ------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "NTT2_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra NTT2_DONE;\n\t"
      "bra NTT2_WAIT;\n\t"
      "NTT2_DONE:\n\t"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, int c0, int c1, const void* smem_src) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];" ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1),
               "r"(smem_u32(smem_src))
               : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes),
               "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void tma_store_commit_and_wait() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void fence_async_proxy() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// shared-memory tile: array of 32-byte field elements, accessed with two 128-bit transactions per element
template <class Fr>
__device__ __forceinline__ Fr tile_ld(const uint4* tile, uint32_t e) {
  const uint4 a = tile[2 * e], b = tile[2 * e + 1];
  Fr r;
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}
template <class Fr>
__device__ __forceinline__ void tile_st(uint4* tile, uint32_t e, const Fr& r) {
  tile[2 * e] = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]);
  tile[2 * e + 1] = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
}
#endif

template <class Fr>
struct Ntt2Strided {
  const Fr* tw;        // omega^i, i < n/2 (forward or inverse table of the domain)
  const Fr* ltab;      // load table (coset g^i), natural index
  const Fr* in_b;      // AB_MINUS_C only
  const Fr* in_c;
  Fr lcst;             // AB_MINUS_C: Z^-1
  int L, s0, k;        // this pass runs stages s0 .. s0+k-1
  int load_mode;       // NTT_LOAD_*: applied by the FIRST pass only
};
template <class Fr>
struct Ntt2Last {
  const Fr* tw;        // omega^i, i < n/2
  const Fr* stab;      // store table, natural index (n^-1 g^-i)
  Fr scst;             // STORE_MUL_CONST: n^-1
  int L;
  int store_mode;      // NTT_STORE_*
};

#ifdef __CUDACC__
// One strided pass.  grid.x = (W / C) column blocks x 2^s0 segments; 512 threads; dynamic shared memory = 128 KB + 64 B.
template <class Fr>
__global__ void __launch_bounds__(NTT2_THREADS, 1) ntt2_strided_kernel(const __grid_constant__ CUtensorMap map_in,
                                                                       const __grid_constant__ CUtensorMap map_out, Ntt2Strided<Fr> a) {
  extern __shared__ __align__(128) unsigned char ntt2_smem[];
  uint4* tile = reinterpret_cast<uint4*>(ntt2_smem);
  uint64_t* bar = reinterpret_cast<uint64_t*>(ntt2_smem + (size_t)NTT2_TILE * 32);
  const int k = a.k;
  const int logC = NTT2_TILE_LOG - k;
  const uint32_t C = 1u << logC, rows = 1u << k;
  const int low_bits = a.L - a.s0 - k;                       // log2 W
  const uint32_t colblks = 1u << (low_bits - logC);
  const uint32_t seg = blockIdx.x / colblks, cb = blockIdx.x % colblks;
  // boxes: at most 256 rows x 64 columns (256 u64) each
  const uint32_t box_rows = rows < 256 ? rows : 256, box_cols = C < 64 ? C : 64;
  const uint32_t nbr = rows / box_rows, nbc = C / box_cols;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, (uint32_t)NTT2_TILE * 32);
    // shared-memory layout of the tile: box-major, every box row-major [box_rows][box_cols]
    for (uint32_t br = 0; br < nbr; br++)
      for (uint32_t bc = 0; bc < nbc; bc++)
        tma_load_2d(ntt2_smem + ((size_t)(br * nbc + bc) * box_rows * box_cols) * 32, &map_in, (int)((cb * C + bc * box_cols) * 4),
                    (int)(seg * rows + br * box_rows), bar);
  }
  mbar_wait(bar, 0);
  // element (row r, column c) of the tile -> index in shared memory
  auto at = [&](uint32_t r, uint32_t c) -> uint32_t {
    const uint32_t br = r / box_rows, rr = r % box_rows, bc = c / box_cols, cc = c % box_cols;
    return ((br * nbc + bc) * box_rows + rr) * box_cols + cc;
  };
  const uint64_t gbase = ((uint64_t)seg << (a.L - a.s0)) + ((uint64_t)cb << logC);
  if (a.load_mode != NTT_LOAD_PLAIN) {
    for (uint32_t e = threadIdx.x; e < (uint32_t)NTT2_TILE; e += NTT2_THREADS) {
      const uint32_t r = e >> logC, c = e & (C - 1);
      const uint64_t gi = gbase + ((uint64_t)r << low_bits) + c;
      const uint32_t se = at(r, c);
      Fr x = tile_ld<Fr>(tile, se);
      if (a.load_mode == NTT_LOAD_MUL_TABLE) {
        x = Fr::mul(x, ntt_ldg(a.ltab + gi));
      } else {
        const Fr y = ntt_ldg(a.in_b + gi), z = ntt_ldg(a.in_c + gi);
        x = Fr::mul(Fr::sub(Fr::mul(x, y), z), a.lcst);
      }
      tile_st<Fr>(tile, se, x);
    }
  }
  __syncthreads();
  const uint32_t nbf = NTT2_TILE >> 1;
  for (int t = 0; t < k; t++) {
    const int hb = k - 1 - t;                  // row bit that separates the pair
    const int s = a.s0 + t;                    // global stage
    const bool trivial = s == a.L - 1;         // last stage of the whole transform: every twiddle is 1 (only when the
                                               // strided pass is also the last one, which the plan never produces)
    for (uint32_t bf = threadIdx.x; bf < nbf; bf += NTT2_THREADS) {
      const uint32_t c = bf & (C - 1), mp = bf >> logC;
      const uint32_t mlow = mp & ((1u << hb) - 1);
      const uint32_t r0 = ((mp >> hb) << (hb + 1)) | mlow, r1 = r0 | (1u << hb);
      const uint32_t e0 = at(r0, c), e1 = at(r1, c);
      const uint64_t jm = ((uint64_t)mlow << low_bits) + ((uint64_t)cb << logC) + c;   // (i mod d)
      const Fr x0 = tile_ld<Fr>(tile, e0), x1 = tile_ld<Fr>(tile, e1);
      const Fr u = Fr::add(x0, x1);
      Fr v = Fr::sub(x0, x1);
      if (!trivial) v = Fr::mul(v, ntt_ldg(a.tw + (jm << s)));
      tile_st<Fr>(tile, e0, u);
      tile_st<Fr>(tile, e1, v);
    }
    __syncthreads();
  }
  fence_async_proxy();                          // generic-proxy writes to the tile -> visible to the TMA store
  __syncthreads();
  if (threadIdx.x == 0) {
    for (uint32_t br = 0; br < nbr; br++)
      for (uint32_t bc = 0; bc < nbc; bc++)
        tma_store_2d(&map_out, (int)((cb * C + bc * box_cols) * 4), (int)(seg * rows + br * box_rows),
                     ntt2_smem + ((size_t)(br * nbc + bc) * box_rows * box_cols) * 32);
    tma_store_commit_and_wait();
  }
}

// The last pass.  grid.x = N / 4 (N = 2^(L-10) blocks of 1024 points); 512 threads; dynamic smem = 128 KB + 16 KB + 64 B.
template <class Fr>
__global__ void __launch_bounds__(NTT2_THREADS, 1) ntt2_last_kernel(const Fr* __restrict__ in, const __grid_constant__ CUtensorMap map_out,
                                                                    Ntt2Last<Fr> a) {
  extern __shared__ __align__(128) unsigned char ntt2_smem[];
  uint4* tile = reinterpret_cast<uint4*>(ntt2_smem);
  uint4* twl = reinterpret_cast<uint4*>(ntt2_smem + (size_t)NTT2_TILE * 32);                    // 512 powers of the 1024-th root
  uint64_t* bar = reinterpret_cast<uint64_t*>(ntt2_smem + (size_t)NTT2_TILE * 32 + 512 * 32);
  const int nb_log = a.L - NTT2_LAST_LOG;                  // log2 N
  const uint32_t quarter = 1u << (nb_log - 2);
  const uint32_t blo = blockIdx.x;                         // < N / 4
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, (uint32_t)NTT2_TILE * 32);
    for (uint32_t j = 0; j < 4; j++)
      tma_load_1d(ntt2_smem + (size_t)j * 1024 * 32, in + ((size_t)(blo + j * quarter) << NTT2_LAST_LOG), 1024 * 32, bar);
  }
  // twiddles of the ten last stages: omega^(jm << s) with s >= L-10 only involves omega_1024 = omega^(2^(L-10))
  for (uint32_t i = threadIdx.x; i < 512; i += NTT2_THREADS) tile_st<Fr>(twl, i, ntt_ldg(a.tw + ((uint64_t)i << nb_log)));
  mbar_wait(bar, 0);
  __syncthreads();
  for (int t = 0; t < NTT2_LAST_LOG; t++) {
    const int hb = NTT2_LAST_LOG - 1 - t;
    const bool trivial = t == NTT2_LAST_LOG - 1;            // the very last stage: twiddle 1
    for (uint32_t bf = threadIdx.x; bf < (uint32_t)(NTT2_TILE >> 1); bf += NTT2_THREADS) {
      const uint32_t blk = bf >> 9, mp = bf & 511;
      const uint32_t mlow = mp & ((1u << hb) - 1);
      const uint32_t e0 = (blk << 10) | ((mp >> hb) << (hb + 1)) | mlow, e1 = e0 | (1u << hb);
      const Fr x0 = tile_ld<Fr>(tile, e0), x1 = tile_ld<Fr>(tile, e1);
      const Fr u = Fr::add(x0, x1);
      Fr v = Fr::sub(x0, x1);
      if (!trivial) v = Fr::mul(v, tile_ld<Fr>(twl, mlow << t));   // exponent (i mod d) * 2^(s - (L-10))
      tile_st<Fr>(tile, e0, u);
      tile_st<Fr>(tile, e1, v);
    }
    __syncthreads();
  }
  // output scalings, by natural output index: element e of block blo + j*quarter lands at brev10(e) * N + brev(blo) * 4 + brev2(j)
  const uint32_t col0 = (nb_log > 2 ? (__brev(blo) >> (32 - (nb_log - 2))) : 0u) << 2;
  if (a.store_mode != NTT_STORE_PLAIN) {
    for (uint32_t idx = threadIdx.x; idx < (uint32_t)NTT2_TILE; idx += NTT2_THREADS) {
      const uint32_t j = idx >> 10, e = idx & 1023;
      Fr x = tile_ld<Fr>(tile, idx);
      if (a.store_mode == NTT_STORE_MUL_CONST) {
        x = Fr::mul(x, a.scst);
      } else {
        const uint64_t gi = ((uint64_t)(__brev(e) >> 22) << nb_log) + col0 + (__brev(j) >> 30);
        x = Fr::mul(x, ntt_ldg(a.stab + gi));
      }
      tile_st<Fr>(tile, idx, x);
    }
    __syncthreads();
  }
  // in-place 12-bit bit-reversal permutation: tile index (j, e) -> (brev10(e), brev2(j)) = row-major [1024 rows][4 columns]
  for (uint32_t idx = threadIdx.x; idx < (uint32_t)NTT2_TILE; idx += NTT2_THREADS) {
    const uint32_t rev = __brev(idx) >> (32 - NTT2_TILE_LOG);
    if (idx < rev) {
      const Fr x = tile_ld<Fr>(tile, idx), y = tile_ld<Fr>(tile, rev);
      tile_st<Fr>(tile, idx, y);
      tile_st<Fr>(tile, rev, x);
    }
  }
  fence_async_proxy();
  __syncthreads();
  if (threadIdx.x == 0) {
    for (uint32_t br = 0; br < 4; br++) tma_store_2d(&map_out, (int)(col0 * 4), (int)(br * 256), ntt2_smem + (size_t)br * 256 * 4 * 32);
    tma_store_commit_and_wait();
  }
}
#endif  // __CUDACC__

// ---- host side -----------------------------------------------------------------------------------------------------------
struct Ntt2Plan {
  int npass;        // strided passes
  int k[4];
};
inline bool ntt2_usable(int L) { return L >= NTT2_MIN_L && L <= 28; }
inline Ntt2Plan ntt2_plan(int L) {
  Ntt2Plan p{};
  const int rest = L - NTT2_LAST_LOG;                       // stages of the strided passes, each 2..10 (C = 4096 >> k <= 1024)
  p.npass = (rest + 9) / 10;
  for (int i = 0; i < p.npass; i++) p.k[i] = rest / p.npass + (i < rest % p.npass ? 1 : 0);
  return p;
}

typedef CUresult (*ntt2_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline ntt2_encode_fn ntt2_encoder() {
  static ntt2_encode_fn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) p = nullptr;
    return reinterpret_cast<ntt2_encode_fn>(p);
  }();
  return fn;
}
// 2-D map over `base` seen as [rows][cols_elems * 4] u64, box = [box_rows][box_cols_elems * 4]
inline bool ntt2_make_map(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols_elems, uint32_t box_rows, uint32_t box_cols_elems) {
  ntt2_encode_fn enc = ntt2_encoder();
  if (!enc) return false;
  const cuuint64_t gdim[2] = {cols_elems * 4, rows};
  const cuuint64_t gstride[1] = {cols_elems * 32};
  const cuuint32_t box[2] = {box_cols_elems * 4, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Full transform with the TMA passes; same contract as ntt_run (src read by the first pass only, `work` carries the
// intermediate passes in place, the last pass writes dst != work).  Returns false when the path is unavailable (size out
// of range or no tensor-map encoder), in which case the caller uses ntt_run.
template <class Fr>
bool ntt2_run(cudaStream_t st, const NttDomain<Fr>& d, bool inverse, const Fr* src, Fr* work, Fr* dst, int load_mode, const Fr* ltab,
              const Fr* in_b, const Fr* in_c, const Fr& load_cst, int store_mode, const Fr* stab, const Fr& store_cst,
              unsigned long long* launches) {
  if (!ntt2_usable(d.L) || !ntt2_encoder()) return false;
  static bool attr_set = [] {
    const int bytes_s = NTT2_TILE * 32 + 64, bytes_l = NTT2_TILE * 32 + 512 * 32 + 64;
    return cudaFuncSetAttribute(ntt2_strided_kernel<Fr>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes_s) == cudaSuccess &&
           cudaFuncSetAttribute(ntt2_last_kernel<Fr>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes_l) == cudaSuccess;
  }();
  if (!attr_set) return false;
  const Ntt2Plan p = ntt2_plan(d.L);
  const Fr* tw = inverse ? d.tw_inv : d.tw_fwd;
  int s0 = 0;
  for (int i = 0; i < p.npass; i++) {
    const int k = p.k[i];
    const int low_bits = d.L - s0 - k;
    const uint64_t R = 1ull << (s0 + k), W = 1ull << low_bits;
    const uint32_t rows = 1u << k, C = (uint32_t)NTT2_TILE >> k;
    const uint32_t box_rows = rows < 256 ? rows : 256, box_cols = C < 64 ? C : 64;
    CUtensorMap mi, mo;
    if (!ntt2_make_map(&mi, i == 0 ? src : work, R, W, box_rows, box_cols) || !ntt2_make_map(&mo, work, R, W, box_rows, box_cols)) return false;
    Ntt2Strided<Fr> a;
    a.tw = tw; a.ltab = ltab; a.in_b = in_b; a.in_c = in_c; a.lcst = load_cst;
    a.L = d.L; a.s0 = s0; a.k = k;
    a.load_mode = i == 0 ? load_mode : NTT_LOAD_PLAIN;
    const unsigned blocks = (unsigned)((W / C) << s0);
    ntt2_strided_kernel<Fr><<<blocks, NTT2_THREADS, NTT2_TILE * 32 + 64, st>>>(mi, mo, a);
    if (launches) (*launches)++;
    s0 += k;
  }
  {
    const uint64_t N = 1ull << (d.L - NTT2_LAST_LOG);
    CUtensorMap mo;
    if (!ntt2_make_map(&mo, dst, 1024, N, 256, 4)) return false;
    Ntt2Last<Fr> a;
    a.tw = tw; a.stab = stab; a.scst = store_cst; a.L = d.L; a.store_mode = store_mode;
    ntt2_last_kernel<Fr><<<(unsigned)(N / 4), NTT2_THREADS, NTT2_TILE * 32 + 512 * 32 + 64, st>>>(work, mo, a);
    if (launches) (*launches)++;
  }
  return true;
}

#define G16_NTT2_TEMPLATES(X, Fr)                                                                                              \
  X bool ntt2_run<Fr>(cudaStream_t, const NttDomain<Fr>&, bool, const Fr*, Fr*, Fr*, int, const Fr*, const Fr*, const Fr*, const Fr&, \
                      int, const Fr*, const Fr&, unsigned long long*);

}  // namespace g16
