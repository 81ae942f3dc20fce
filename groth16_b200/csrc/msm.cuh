// msm.cuh -- variable-base multi-scalar multiplication on sm_90a (Pippenger, signed digits, sort-by-bucket).
//
// Replaces ark-ec 0.5.0 `VariableBaseMSM::msm_bigint` as called at /root/reference/src/prover.rs:66 (H query),
// :74 (L query) and :262 (A, B-in-G1, B-in-G2 via calculate_coeff).  The group element returned is identical to
// the reference's (EC addition is exactly associative/commutative), whatever the window size or summation order.
//
// Resident bases come with precomputed multiples 2^(c*ne*j) * P (msm_precompute, copy-major), so that the W windows of a
// scalar fall into only `ne` bucket sets (ne = 1 by default: one set of 2^(c-1) buckets for the whole MSM).
// Pipeline (all on one stream, no host synchronisation until the leaf sums of the bucket reduction are read back):
//   1. msm_digits<COUNT>   scalar -> W signed c-bit digits; histogram of (bucket set, |digit|) keys (warp-aggregated atomics)
//   2. msm_scan_*          exclusive prefix sum of the histogram -> bucket offsets (three small launches)
//   3. msm_digits<SCATTER> counting-sort scatter: sorted (copy * n + base index | sign) per entry; msm_pad_fill then writes
//                          the key of every sorted slot bucket by bucket and marks the bucket padding empty
//   4. msm_accum_l0        load-balanced segmented reduction: every thread owns K0 consecutive sorted entries,
//                          mixed-adds them (XYZZ += affine, gathered from the resident base array), writes buckets
//                          that are complete inside its chunk and emits <= 2 boundary partials
//   5. msm_accum_ln/_tail  the same reduction over the partial list, level by level (empty levels return at once)
//   6. msm_sum_strided     bucket reduction sum_b (b+1) B_b as two rounds of row / column block-tree sums
//   host: weighted sums of the <= 64-point leaf arrays, Horner over effective windows; prover.rs semantics preserved.
// Skewed scalar distributions (boolean witnesses, the reference's DummyCircuit whose witness is constant,
// benches/bench.rs:43-54) cost the same as uniform ones: work is split by sorted position, not by bucket.
#pragma once
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdlib>
#include "ec.cuh"

namespace g16 {

static constexpr uint32_t MSM_INVALID = 0xffffffffu;

struct MsmGeom {
  uint32_t n;        // number of (scalar, base) pairs
  int c;             // window bits
  int W;             // number of c-bit windows of a scalar
  int ne;            // effective windows: window w = j*ne + e lands in bucket set e and uses base copy j
  int copies;        // ceil(W / ne) precomputed multiples 2^(c*ne*j) * P of every base (1 = no precomputation)
  uint32_t B;        // buckets per effective window = 2^(c-1)  (digit magnitudes 1..B)
  uint32_t nkeys;    // ne * B
  uint64_t max_entries;  // n * W
  int k0;            // sorted entries per thread in the level-0 accumulation (64 for large MSMs, less to fill the GPU)
  int ba;            // batched-affine pre-reduction rounds before the accumulation (msm_ba.cuh); 0 = none
  int ba_pad;        // buckets are padded to multiples of 2^ba_pad sorted slots (>= ba; larger when the sorted list is
                     // shared with an MSM that runs more rounds)
  int ba_m;          // batched-affine: additions per thread and round
  int ba_G;          // batched-affine: thread products per field inversion
  int ba_gcd;        // batched-affine: 1 = safegcd inversion, 0 = Fermat
  int acc_block;     // threads per block of the level-0 accumulation (32 / 64 / 128)
  uint32_t batch;    // MSMs over the same bases in one pass (proof k owns bucket sets k*ne .. k*ne+ne-1); 0 and 1 = one
  // bucket sets of the whole pass (a zero-initialised MsmGeom is one MSM)
  __host__ __device__ uint32_t sets() const { return (uint32_t)ne * (batch > 1 ? batch : 1u); }
};

static constexpr int MSM_K0_MAX = 64;
// Entries per thread so that the level-0 grid is at least ~2 waves of `resident_threads` (small MSMs, e.g. the per-rank
// shards of a multi-GPU proof, would otherwise run as a fraction of one wave: time = one 64-entry chunk regardless of size).
inline int msm_pick_k0(uint64_t max_entries, uint64_t resident_threads, int k0_min) {
  int k0 = MSM_K0_MAX;
  while (k0 > k0_min && max_entries / k0 < resident_threads * 2) k0 >>= 1;
  return k0;
}
static constexpr int MSM_K0_AUTO_MIN_G1 = 8, MSM_K0_AUTO_MIN_G2 = 16;   // k0_min of the automatic rule (Engine::with_k0)
// the smallest k0 an MSM can run with under acc_k0 = k0_knob (0: automatic; 4 .. 1024: exactly that many)
inline int msm_k0_floor(bool g2, long long k0_knob) {
  return (k0_knob >= 4 && k0_knob <= 1024) ? (int)k0_knob : (g2 ? MSM_K0_AUTO_MIN_G2 : MSM_K0_AUTO_MIN_G1);
}
inline int msm_pick_c(uint64_t n) {
  int lg = 0;
  while ((1ull << lg) < n) lg++;
  int c = lg - 4;
  if (c < 3) c = 3;
  if (c > 16) c = 16;
  return c;
}
// ne_req <= 0: no precomputation (ne = W).  Otherwise the requested number of effective windows (1 = every window
// of a scalar shares one bucket set, which needs W precomputed multiples per base).
inline MsmGeom msm_geom(uint64_t n, int scalar_bits, int c_override = 0, int ne_req = 0) {
  MsmGeom g;
  g.n = (uint32_t)n;
  g.c = c_override > 0 ? c_override : msm_pick_c(n);
  g.W = (scalar_bits + 1 + g.c - 1) / g.c;   // +1: room for the top signed-digit carry
  g.ne = (ne_req <= 0 || ne_req > g.W) ? g.W : ne_req;
  g.copies = (g.W + g.ne - 1) / g.ne;
  g.B = 1u << (g.c - 1);
  g.batch = 1;
  g.nkeys = g.sets() * g.B;
  g.max_entries = (uint64_t)n * g.W;
  g.k0 = MSM_K0_MAX;
  g.ba = 0;
  g.ba_pad = 0;
  g.ba_m = 32;
  g.ba_G = 16;
  g.ba_gcd = 1;
  g.acc_block = 128;
  return g;
}
// `batch` MSMs of one geometry over the same bases, sorted and reduced together (k0 / rounds are re-derived by the caller)
inline MsmGeom msm_geom_batch(MsmGeom g, uint32_t batch) {
  g.batch = batch;
  g.nkeys = g.sets() * g.B;
  g.max_entries = (uint64_t)g.n * g.W * (batch > 1 ? batch : 1u);
  return g;
}

// ------------------------------------------------------------------------------------------------
// 1/3. digit extraction + histogram / scatter
// ------------------------------------------------------------------------------------------------
// Signed-digit recoding of a canonical scalar k < 2^bits:  k = sum_w d_w 2^(c w), d_w in [-2^(c-1), 2^(c-1)].
// blockIdx.y = MSM k of a batch: its scalars start batch_stride 32-bit words after those of MSM k-1, its keys lie in bucket
// sets k*ne .. k*ne+ne-1; the sorted index is the same (copy * n + i | sign) for every k, since the bases are shared.
template <class FrF, bool SCATTER>
__global__ void __launch_bounds__(256) msm_digits(const uint32_t* __restrict__ scalars, uint32_t scalar_stride, int scalars_mont,
                                                  const uint8_t* __restrict__ skip, MsmGeom g,
                                                  uint32_t* __restrict__ counters,  // COUNT: histogram; SCATTER: cursors
                                                  uint32_t* __restrict__ sidx, uint64_t batch_stride) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t set0 = blockIdx.y * (uint32_t)g.ne;
  scalars += blockIdx.y * batch_stride;
  bool live = i < g.n;
  FrF s = FrF::zero();
  if (live) {
    constexpr int NV = FrF::N / 4;   // 16-byte words per scalar
    const uint4* p = reinterpret_cast<const uint4*>(scalars) + (size_t)i * scalar_stride * NV;
#pragma unroll
    for (int j = 0; j < NV; j++) {
      const uint4 x = __ldg(p + j);
      s.v[4 * j] = x.x; s.v[4 * j + 1] = x.y; s.v[4 * j + 2] = x.z; s.v[4 * j + 3] = x.w;
    }
    if (skip && skip[i]) live = false;
  }
  if (scalars_mont) s = FrF::from_mont(s);   // `into_bigint`, prover.rs:64,71,82
  uint32_t carry = 0;
  for (int w = 0; w < g.W; w++) {
    // c <= 16 bits starting at bit w*c
    const int bit = w * g.c;
    const int limb = bit >> 5, sh = bit & 31;
    uint32_t raw = 0;
    if (limb < FrF::N) {
      uint64_t two = s.v[limb];
      if (limb + 1 < FrF::N) two |= (uint64_t)s.v[limb + 1] << 32;
      raw = (uint32_t)(two >> sh) & ((1u << g.c) - 1);
    }
    raw += carry;
    uint32_t neg = 0;
    carry = 0;
    if (raw > g.B) { raw = (1u << g.c) - raw; neg = 1; carry = 1; }
    const bool emit = live && raw != 0;
    const int e = w % g.ne, j = w / g.ne;
    const uint32_t key = emit ? (set0 + (uint32_t)e) * g.B + (raw - 1) : MSM_INVALID;
    // warp-aggregated atomic: one atomicAdd per distinct key in the warp
    const uint32_t peers = __match_any_sync(0xffffffffu, key);
    if (emit) {
      const uint32_t rank = __popc(peers & ((1u << lane) - 1));
      const int leader = __ffs(peers) - 1;
      uint32_t base = 0;
      if ((int)lane == leader) base = atomicAdd(&counters[key], (uint32_t)__popc(peers));
      base = __shfl_sync(peers, base, leader);
      if (SCATTER) sidx[base + rank] = ((uint32_t)j * g.n + i) | (neg << 31);   // its key: msm_pad_fill
    }
  }
}

// 2. exclusive scan in three small launches: per-block scan (4096 keys per block), scan of the block totals, fix-up.
// `cursors` may alias `hist` (the histogram is turned into the scatter cursors in place).  offsets[nkeys] = total.
static constexpr int SCAN_ITEMS = 4;
static constexpr int SCAN_BLOCK = 1024 * SCAN_ITEMS;
static __device__ __forceinline__ uint32_t block_exclusive_scan_1024(uint32_t v, uint32_t* sh, uint32_t* total) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= (uint32_t)d) x += y;
  }
  if (lane == 31) sh[wid] = x;
  __syncthreads();
  if (wid == 0) {
    uint32_t w = sh[lane];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      uint32_t y = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= (uint32_t)d) w += y;
    }
    sh[32 + lane] = w;
  }
  __syncthreads();
  const uint32_t warp_off = wid ? sh[32 + wid - 1] : 0;
  *total = sh[63];
  return warp_off + x - v;
}
// pad_mask = 2^R - 1: every bucket is padded to a multiple of 2^R slots (regular layout of the batched-affine rounds)
static __global__ void __launch_bounds__(1024) msm_scan_blocks(const uint32_t* hist, uint32_t nkeys, uint32_t* offsets,
                                                               uint32_t* block_tot, uint32_t pad_mask) {
  __shared__ uint32_t sh[64];
  const uint32_t base = blockIdx.x * SCAN_BLOCK + threadIdx.x * SCAN_ITEMS;
  uint32_t v[SCAN_ITEMS], s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) { v[k] = (base + k < nkeys) ? ((hist[base + k] + pad_mask) & ~pad_mask) : 0; s += v[k]; }
  uint32_t tot;
  uint32_t run = block_exclusive_scan_1024(s, sh, &tot);
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) { if (base + k < nkeys) offsets[base + k] = run; run += v[k]; }
  if (threadIdx.x == 0) block_tot[blockIdx.x] = tot;
}
static __global__ void __launch_bounds__(1024) msm_scan_tops(uint32_t* block_tot, uint32_t nblocks, uint32_t* total_out) {
  __shared__ uint32_t sh[64];
  __shared__ uint32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (uint32_t b0 = 0; b0 < nblocks; b0 += 1024) {
    const uint32_t i = b0 + threadIdx.x;
    const uint32_t v = i < nblocks ? block_tot[i] : 0;
    uint32_t tot;
    const uint32_t ex = block_exclusive_scan_1024(v, sh, &tot);
    const uint32_t c = carry;
    __syncthreads();
    if (i < nblocks) block_tot[i] = c + ex;
    if (threadIdx.x == 0) carry = c + tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total_out = carry;
}
static __global__ void __launch_bounds__(1024) msm_scan_fix(uint32_t* offsets, uint32_t nkeys, const uint32_t* block_tot,
                                                            uint32_t* cursors) {
  const uint32_t add = block_tot[blockIdx.x];
  const uint32_t base = blockIdx.x * SCAN_BLOCK + threadIdx.x * SCAN_ITEMS;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++)
    if (base + k < nkeys) {
      const uint32_t o = offsets[base + k] + add;
      offsets[base + k] = o;
      cursors[base + k] = o;
    }
}

// Every sorted slot of bucket b, [offsets[b], offsets[b + 1]), gets its key b here, one warp per bucket, in unit-stride
// stores.  The scatter does not write keys: there every entry is a random 4-byte store, and the sorted list is larger
// than L2, so each such store costs DRAM traffic.  After the scatter the cursor of bucket b stands at the end of its
// real entries; the slots from there to the start of the next bucket are padding and are marked empty.
static constexpr uint32_t MSM_FILL_BLOCK = 256;
static __global__ void __launch_bounds__(MSM_FILL_BLOCK) msm_pad_fill(const uint32_t* __restrict__ cursors,
                                                                      const uint32_t* __restrict__ offsets, uint32_t nkeys,
                                                                      uint32_t* __restrict__ sidx, uint32_t* __restrict__ skey) {
  const uint64_t b = ((uint64_t)blockIdx.x * MSM_FILL_BLOCK + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if (b >= nkeys) return;
  const uint32_t real_end = cursors[b], end = offsets[b + 1];
  for (uint32_t p = offsets[b] + lane; p < end; p += 32) {
    skey[p] = (uint32_t)b;
    if (p >= real_end) sidx[p] = MSM_INVALID;
  }
}

}  // namespace g16
#include "msm_ba.cuh"   // batched-affine pre-reduction of the sorted entries
namespace g16 {

// ------------------------------------------------------------------------------------------------
// 4/5. load-balanced segmented bucket accumulation
// ------------------------------------------------------------------------------------------------
// Every thread t of a level owns two output slots (2t: "head" partial, 2t+1: "tail" partial) and always writes
// both keys (MSM_INVALID when unused), so no memset of the partial lists is needed.
template <class F>
struct MsmEmit {
  XYZZ<F>* buckets;
  uint32_t* okeys;
  XYZZ<F>* opts;
  uint64_t t;
  bool wrote_head, wrote_tail;
  __device__ __forceinline__ void flush(uint32_t key, const XYZZ<F>& acc, bool head, bool tail) {
    if (!head && !tail) {
      buckets[key] = acc;   // the whole bucket was summed here: written exactly once, no atomics
    } else {
      const uint64_t slot = 2 * t + (head ? 0 : 1);
      okeys[slot] = key;
      opts[slot] = acc;
      if (head) wrote_head = true; else wrote_tail = true;
    }
  }
  // returns the number of partials this thread emitted
  __device__ __forceinline__ uint32_t finish() {
    if (!wrote_head) okeys[2 * t] = MSM_INVALID;
    if (!wrote_tail) okeys[2 * t + 1] = MSM_INVALID;
    return (wrote_head ? 1u : 0u) + (wrote_tail ? 1u : 0u);
  }
};

template <class F>
__device__ __forceinline__ Affine<F> load_affine(const Affine<F>* __restrict__ bases, uint32_t idx) {
  Affine<F> p;
  constexpr int NV = sizeof(Affine<F>) / 16;
  const uint4* src = reinterpret_cast<const uint4*>(bases + idx);
  uint4* dst = reinterpret_cast<uint4*>(&p);
#pragma unroll
  for (int j = 0; j < NV; j++) dst[j] = __ldg(src + j);
  return p;
}

// Level 0: grid covers T0 = ceil(max_entries / K0) threads; threads past the real entry count only clear their slots.
// Register budget: 3 resident blocks per SM for narrow points (G1), 2 for wide ones (G2, BW6-761).  (Staging the gathered
// bases through shared memory with cp.async was measured and is slower: with 3 warps per scheduler the gather latency
// is already hidden and the kernel is bound by the IMAD.WIDE pipe.  Also measured and slower: the running sum
// kept in shared memory for one more resident block per SM; lazily reduced double-width products.)
template <class F>
struct MsmAccumCfg { static constexpr int MIN_BLOCKS = MsmWide<F>::value ? 2 : 3; };
// coordinates of the gathered base fetched on demand (x, then y) for wide points: 24 fewer live registers at the peak
template <class F>
__host__ __device__ constexpr bool msm_lazy_load() { return MsmWide<F>::value; }
// `sidx` == nullptr: the entries are the points of `bases` themselves (last list of the batched-affine rounds) and the
// key of entry e is skey[e << key_shift]; empty slots (MSM_INVALID index, or the point (0,0)) add nothing.
template <class F>
__global__ void __launch_bounds__(128, MsmAccumCfg<F>::MIN_BLOCKS) msm_accum_l0(const Affine<F>* __restrict__ bases,
                                                    const uint32_t* __restrict__ sidx,
                                                    const uint32_t* __restrict__ skey, uint32_t key_shift,
                                                    const uint32_t* __restrict__ total_ptr, uint64_t T0, uint32_t K0,
                                                    XYZZ<F>* __restrict__ buckets, uint32_t* __restrict__ okeys,
                                                    XYZZ<F>* __restrict__ opts, uint32_t* pending0) {
  const uint32_t M = *total_ptr >> key_shift;
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t == 0) *pending0 = 1;   // level 0 always hands a (possibly empty) partial list to level 1
  if (t >= T0) return;
  MsmEmit<F> em{buckets, okeys, opts, t, false, false};
  const uint64_t begin = t * (uint64_t)K0;
  if (begin >= M) { em.finish(); return; }
  const uint32_t end = (uint32_t)min((uint64_t)M, begin + K0);
  auto key_at = [&](uint64_t e) { return skey[e << key_shift]; };
  const uint32_t prev = begin > 0 ? key_at(begin - 1) : MSM_INVALID;
  const uint32_t next = end < M ? key_at(end) : MSM_INVALID;
  uint32_t cur = key_at(begin);
  bool first_seg = true;
  XYZZ<F> acc = XYZZ<F>::inf();
#pragma unroll 1
  for (uint32_t e = (uint32_t)begin; e < end; e++) {
    const uint32_t k = key_at(e);
    if (k != cur) {
      em.flush(cur, acc, first_seg && prev == cur, false);
      first_seg = false;
      cur = k;
      acc = XYZZ<F>::inf();
    }
    const uint32_t ix = sidx ? sidx[e] : e;
    if (ix == MSM_INVALID) continue;
    if (msm_lazy_load<F>()) {
      const uint4* src = reinterpret_cast<const uint4*>(bases + (ix & 0x7fffffffu));
      constexpr int NVH = sizeof(F) / 16;
      auto ld = [&](int half) {
        F v;
        uint4* d = reinterpret_cast<uint4*>(&v);
#pragma unroll
        for (int j = 0; j < NVH; j++) d[j] = __ldg(src + half * NVH + j);
        return v;
      };
      acc.madd_lazy([&]() { return ld(0); }, [&]() { return ld(1); }, sidx && (ix >> 31) != 0);
    } else {
      const Affine<F> p = load_affine(bases, ix & 0x7fffffffu);
      acc.madd_inline(p, sidx && (ix >> 31) != 0);
    }
  }
  em.flush(cur, acc, first_seg && prev == cur, next == cur);
  em.finish();
}

// One level >= 1 for thread t over slots [1 + t*KF, 1 + (t+1)*KF) of a partial list of S slots (slot 0, the head of
// thread 0, is never valid).  The one-slot shift makes chunk boundaries fall between a thread's (head, tail) pair instead
// of between tail_t and head_{t+1}: with evenly filled buckets every run (tail_t, head_{t+1}) is then interior to a chunk
// and the whole list resolves in ONE level.  Keys may contain MSM_INVALID holes; inside a run of equal keys there is at
// most one hole between neighbours (DESIGN.md), so a look-back / look-ahead of two slots decides whether a run continues
// across the chunk boundary.  Returns the number of partials emitted.
template <class F, int KF>
__device__ __forceinline__ uint32_t msm_level_step(const uint32_t* ikeys, const XYZZ<F>* ipts, uint64_t S, uint64_t t,
                                                   XYZZ<F>* buckets, uint32_t* okeys, XYZZ<F>* opts) {
  MsmEmit<F> em{buckets, okeys, opts, t, false, false};
  const uint64_t begin = 1 + t * KF;
  if (begin >= S) return em.finish();
  const uint64_t end = min(S, begin + KF);
  uint32_t prev = ikeys[begin - 1], next = MSM_INVALID;
  if (prev == MSM_INVALID && begin >= 2) prev = ikeys[begin - 2];
  if (end < S) next = ikeys[end];
  if (next == MSM_INVALID && end + 1 < S) next = ikeys[end + 1];
  uint32_t cur = MSM_INVALID;
  bool have = false, first_seg = true;
  XYZZ<F> acc = XYZZ<F>::inf();
  for (uint64_t e = begin; e < end; e++) {
    const uint32_t k = ikeys[e];
    if (k == MSM_INVALID) continue;
    if (!have) {
      have = true;
      cur = k;
      acc = ipts[e];
    } else if (k != cur) {
      em.flush(cur, acc, first_seg && prev == cur, false);
      first_seg = false;
      cur = k;
      acc = ipts[e];
    } else {
      acc.add(ipts[e]);
    }
  }
  if (have) em.flush(cur, acc, first_seg && prev == cur, next == cur);
  return em.finish();
}
__host__ __device__ inline uint64_t msm_level_threads(uint64_t S, int KF) { return S <= 1 ? 1 : (S - 1 + KF - 1) / KF; }

// pending[0] = partials emitted by the previous level (level 0 stores a non-zero dummy), pending[1] = ours.
// A level whose input is empty returns at once; so do all later levels (their input counter stays 0).
template <class F, int KF>
__global__ void __launch_bounds__(128) msm_accum_ln(const uint32_t* __restrict__ ikeys,
                                                    const XYZZ<F>* __restrict__ ipts, uint64_t S, uint64_t T,
                                                    XYZZ<F>* __restrict__ buckets, uint32_t* __restrict__ okeys,
                                                    XYZZ<F>* __restrict__ opts, uint32_t* pending) {
  if (pending[0] == 0) return;
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t emitted = 0;
  if (t < T) emitted = msm_level_step<F, KF>(ikeys, ipts, S, t, buckets, okeys, opts);
  const uint32_t any = __syncthreads_count(emitted != 0);
  if (threadIdx.x == 0 && any) atomicAdd(&pending[1], any);
}
// All remaining levels in one block once the partial list is short: no launch gaps.
template <class F, int KF>
__global__ void __launch_bounds__(256) msm_accum_tail(uint32_t* k0, XYZZ<F>* p0, uint32_t* k1, XYZZ<F>* p1, uint64_t S,
                                                      XYZZ<F>* buckets, const uint32_t* pending) {
  if (pending[0] == 0) return;
  uint32_t *ik = k0, *ok = k1;
  XYZZ<F>*ip = p0, *op = p1;
  while (true) {
    const uint64_t T = msm_level_threads(S, KF);
    uint32_t emitted = 0;
    for (uint64_t t = threadIdx.x; t < T; t += blockDim.x) emitted += msm_level_step<F, KF>(ik, ip, S, t, buckets, ok, op);
    const uint32_t any = __syncthreads_count(emitted != 0);
    if (T == 1 || any == 0) break;
    S = 2 * T;
    uint32_t* tk = ik; ik = ok; ok = tk;
    XYZZ<F>* tp = ip; ip = op; op = tp;
  }
}

// ------------------------------------------------------------------------------------------------
// 6/7. bucket reduction:  sum_b (b + 1) * bucket[b]  per effective window
// ------------------------------------------------------------------------------------------------
// Written as plain sums only, so that every step is a shallow tree instead of a long dependent chain of point
// additions (a single warp needs ~15 us per XYZZ addition):  with b = hi * 2^a0 + lo,
//     sum_b (b+1) B_b = 2^a0 * sum_hi hi * R_hi + sum_lo (lo+1) * C_lo,   R_hi = sum_lo B[hi,lo],  C_lo = sum_hi B[hi,lo]
// and the two weighted sums over the short arrays R and C are split the same way once more; what is left (arrays of
// <= 64 points) is finished on the host, where a point addition costs ~0.6 us.  Each bucket enters two additions, like
// in the classic running-sum trick.
//
// job: out[o] = sum_{j < len} in[w * win_stride + r * base_mul + j * stride],  o = w * per_win_out + r.
// `tpo` threads cooperate on one output: strided serial part, then a shared-memory tree.  Up to 4 independent jobs
// (the row and the column sums of one or two arrays) share a launch: blocks [first_block, first_block + n_blocks).
template <class F>
struct MsmSumJob {
  const XYZZ<F>* in;
  XYZZ<F>* out;
  uint32_t n_out, per_win_out, win_stride, len, stride, base_mul, tpo, first_block;
};
template <class F>
struct MsmSumJobs {
  MsmSumJob<F> j[4];
  int n;
};
template <class F, int TPB>
__global__ void __launch_bounds__(TPB) msm_sum_strided(MsmSumJobs<F> jobs) {
  __shared__ XYZZ<F> sm[TPB];
  int ji = 0;
#pragma unroll
  for (int k = 1; k < 4; k++)
    if (k < jobs.n && blockIdx.x >= jobs.j[k].first_block) ji = k;
  const MsmSumJob<F>& jb = jobs.j[ji];
  const uint32_t tpo = jb.tpo;
  const uint32_t g = threadIdx.x / tpo, l = threadIdx.x % tpo;
  const uint32_t o = (blockIdx.x - jb.first_block) * (TPB / tpo) + g;
  XYZZ<F> acc = XYZZ<F>::inf();
  if (o < jb.n_out) {
    const uint32_t w = o / jb.per_win_out, r = o % jb.per_win_out;
    const XYZZ<F>* base = jb.in + (size_t)w * jb.win_stride + (size_t)r * jb.base_mul;
    for (uint32_t j = l; j < jb.len; j += tpo) acc.add(base[(size_t)j * jb.stride]);
  }
  for (uint32_t sft = tpo >> 1; sft > 0; sft >>= 1) {
    sm[threadIdx.x] = acc;
    __syncthreads();
    if (l < sft) acc.add(sm[threadIdx.x + sft]);
    __syncthreads();
  }
  if (l == 0 && o < jb.n_out) jb.out[o] = acc;
}

// Reduction plan for one effective window of 2^m buckets: a binary tree of arrays (node 0 = the buckets).
static constexpr int MSM_LEAF_LOG = 6;   // arrays of <= 64 points go to the host
struct MsmRedNode {
  int log_len, a0, a1;      // a0 = low bits (row length), a1 = high bits (column length)
  int child_r, child_c;     // -1 for leaves
  size_t off;               // offset (points, per window) in the device scratch; leaves: offset in the leaf region
  bool leaf;
};
struct MsmRedPlan {
  MsmRedNode nodes[16];
  int n_nodes = 0;
  size_t inner_pts = 0, leaf_pts = 0;   // per window
  int build(int log_len) {
    const int id = n_nodes++;
    MsmRedNode& nd = nodes[id];
    nd.log_len = log_len;
    nd.child_r = nd.child_c = -1;
    nd.leaf = log_len <= MSM_LEAF_LOG;
    nd.a0 = nd.a1 = 0;
    nd.off = 0;
    if (!nd.leaf) {
      const int a0 = log_len / 2, a1 = log_len - a0;
      nodes[id].a0 = a0;
      nodes[id].a1 = a1;
      const int r = build(a1);
      const int c = build(a0);
      nodes[id].child_r = r;
      nodes[id].child_c = c;
    }
    return id;
  }
  void layout() {
    inner_pts = leaf_pts = 0;
    for (int i = 1; i < n_nodes; i++)
      if (!nodes[i].leaf) { nodes[i].off = inner_pts; inner_pts += (size_t)1 << nodes[i].log_len; }
    for (int i = 0; i < n_nodes; i++)
      if (nodes[i].leaf) { nodes[i].off = leaf_pts; leaf_pts += (size_t)1 << nodes[i].log_len; }
  }
  void make(int m) { n_nodes = 0; build(m); layout(); }
};

// infinity mask of a base array (x == y == 0), computed once when a query is made resident
template <class F>
__global__ void msm_inf_mask(const Affine<F>* __restrict__ bases, uint32_t n, uint8_t* __restrict__ mask) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Affine<F> p = load_affine(bases, i);
  mask[i] = p.is_inf() ? 1 : 0;
}

// Base precomputation: out[j*n + i] = 2^(shift*j) * in[i] for j < copies, as affine points (one inversion per base:
// the copies of a base are normalised together with Montgomery's trick).  `out` copy 0 may alias `in`.
static constexpr int MSM_MAX_COPIES = 20;
template <class F>
__global__ void __launch_bounds__(128) msm_precompute(const Affine<F>* in, uint32_t n, int copies, int shift,
                                                      Affine<F>* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Affine<F> p = load_affine(in, i);
  out[i] = p;
  XYZZ<F> q = XYZZ<F>::from_affine(p);
  F Xs[MSM_MAX_COPIES], Ys[MSM_MAX_COPIES], ZZs[MSM_MAX_COPIES], ZZZs[MSM_MAX_COPIES], pref[MSM_MAX_COPIES];
  F acc = F::one();
  int live = 0;   // copies 1..live are finite
  for (int j = 1; j < copies; j++) {
    for (int s = 0; s < shift; s++) q.dbl_inplace();
    if (q.is_inf()) break;
    Xs[j] = q.X; Ys[j] = q.Y; ZZs[j] = q.ZZ; ZZZs[j] = q.ZZZ;
    pref[j] = acc;
    acc = F::mul(acc, q.ZZZ);
    live = j;
  }
  for (int j = live + 1; j < copies; j++) out[(size_t)j * n + i] = Affine<F>::inf();
  if (live == 0) return;
  F inv = F::inv(acc);
  for (int j = live; j >= 1; j--) {
    const F zi = F::mul(inv, pref[j]);   // 1 / ZZZ_j
    inv = F::mul(inv, ZZZs[j]);
    const F z = F::mul(zi, ZZs[j]);      // 1 / Z_j
    const F zi2 = F::sqr(z);
    Affine<F> a{F::mul(Xs[j], zi2), F::mul(Ys[j], zi)};
    out[(size_t)j * n + i] = a;
  }
}

// ------------------------------------------------------------------------------------------------
// host driver
// ------------------------------------------------------------------------------------------------
struct DevBuf {   // owns one device allocation: freed when the buffer goes out of scope, moved but never copied
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) {
      release();
      p = o.p; cap = o.cap;
      o.p = nullptr; o.cap = 0;
    }
    return *this;
  }
  ~DevBuf() { release(); }
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e == cudaSuccess) cap = bytes;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <class T>
  T* as() const { return reinterpret_cast<T*>(p); }
};

static constexpr int MSM_KF = 4;       // partial slots per thread, levels >= 1
static constexpr int MSM_TAIL_S = 2048;  // partial-list length at which the remaining levels fuse into one block

// Host-side plan of the batched-affine rounds of one MSM (msm_ba.cuh): upper bounds of the list lengths (the true
// lengths live on the device), outputs per thread of every round and the entries per thread of the accumulation
// that finishes the last list.
static constexpr int MSM_BA_MAX_ROUNDS = 6;
struct MsmBaPlan {
  int R = 0, pad = 0;
  uint64_t len[MSM_BA_MAX_ROUNDS + 1] = {0};   // len[r] = slots of list r (len[0]: padded sorted slots), upper bounds
  uint32_t m[MSM_BA_MAX_ROUNDS] = {0};
  uint64_t threads_max = 0;
  int k0_final = 0;
  void make(const MsmGeom& g) {
    R = g.ba < 0 ? 0 : (g.ba > MSM_BA_MAX_ROUNDS ? MSM_BA_MAX_ROUNDS : g.ba);
    pad = g.ba_pad > R ? (g.ba_pad > MSM_BA_MAX_ROUNDS ? MSM_BA_MAX_ROUNDS : g.ba_pad) : R;
    // every bucket is padded to a multiple of 2^pad slots: at most 2^pad - 1 extra slots per bucket
    len[0] = pad > 0 ? ((g.max_entries + (uint64_t)g.nkeys * ((1u << pad) - 1)) >> pad) << pad : g.max_entries;
    threads_max = 0;
    for (int r = 0; r < R; r++) {
      len[r + 1] = len[r] >> 1;
      uint32_t mm = (uint32_t)(g.ba_m < 1 ? 1 : g.ba_m);
      while (mm > 4 && len[r + 1] / mm < 200000) mm >>= 1;   // keep at least ~200k threads per round
      m[r] = mm;
      const uint64_t T = ba_threads(len[r + 1], mm);
      if (T > threads_max) threads_max = T;
    }
    k0_final = g.k0 >> R;
    if (k0_final < 8) k0_final = g.k0 < 8 ? g.k0 : 8;
  }
  // threads of the level-0 accumulation.  Without rounds the list is still padded when it is shared with an MSM that runs
  // them (pad > 0): the threads must cover the padded length len[0], not just max_entries
  uint64_t l0_threads(const MsmGeom& g) const {
    return R > 0 ? (len[R] + k0_final - 1) / k0_final : (len[0] + g.k0 - 1) / g.k0;
  }
  // device bytes the rounds need on top of the plain pipeline (per MSM and proof slot)
  template <class F>
  uint64_t extra_bytes() const {
    if (R == 0) return 0;
    return len[1] * (sizeof(F) + sizeof(Affine<F>)) + (R > 1 ? len[2] * sizeof(Affine<F>) : 0) + 2 * threads_max * sizeof(F);
  }
};

// Device bytes of every buffer MsmWorkspace::prepare reserves for geometry g, with bap = the rounds' plan of g and plan =
// the reduction plan of 2^(c-1) buckets.  prepare reserves exactly these sizes and the batch prover's group bound is taken
// from them (msm_batch_bytes_per_proof), so the bound cannot drift from the allocation.
struct MsmWsBytes {
  uint64_t ba_pre, ba_prod, ba_pre2, ba_l0, ba_l1;          // batched-affine rounds (0 without rounds)
  uint64_t counters, offsets, blocktot, sidx, skey, buckets;
  uint64_t pk0, pp0, pk1, pp1, pending;                     // partial lists of the accumulation levels
  uint64_t red_inner, red_leaf;                             // bucket reduction
  uint64_t total() const {
    return ba_pre + ba_prod + ba_pre2 + ba_l0 + ba_l1 + counters + offsets + blocktot + sidx + skey + buckets + pk0 + pp0 +
           pk1 + pp1 + pending + red_inner + red_leaf;
  }
};
template <class F>
MsmWsBytes msm_ws_bytes(const MsmGeom& g, const MsmBaPlan& bap, const MsmRedPlan& plan) {
  MsmWsBytes b{};
  const uint64_t T0 = bap.l0_threads(g);
  const uint64_t S1 = 2 * T0;
  const uint64_t S2 = 2 * msm_level_threads(S1, MSM_KF);
  if (bap.R > 0) {
    b.ba_pre = bap.len[1] * sizeof(F) + 16;
    b.ba_prod = b.ba_pre2 = bap.threads_max * sizeof(F) + 16;
    b.ba_l0 = bap.len[1] * sizeof(Affine<F>) + 16;
    if (bap.R > 1) b.ba_l1 = bap.len[2] * sizeof(Affine<F>) + 16;
  }
  b.counters = b.offsets = ((uint64_t)g.nkeys + 1) * 4;
  b.blocktot = (((uint64_t)g.nkeys + SCAN_BLOCK - 1) / SCAN_BLOCK + 1) * 4;
  b.sidx = b.skey = bap.len[0] * 4 + 16;
  b.buckets = (uint64_t)g.nkeys * sizeof(XYZZ<F>);
  b.pk0 = S1 * 4 + 16;
  b.pp0 = S1 * sizeof(XYZZ<F>);
  b.pk1 = S2 * 4 + 16;
  b.pp1 = S2 * sizeof(XYZZ<F>);
  b.pending = 64 * 4;   // one partial-list counter per accumulation level
  b.red_inner = (plan.inner_pts * g.sets() + 1) * sizeof(XYZZ<F>);
  b.red_leaf = (plan.leaf_pts * g.sets() + 1) * sizeof(XYZZ<F>);
  return b;
}
// Device workspace per proof of a batched pass of MSM g (g16_prove_batch): an upper bound of msm_ws_bytes / G for the pass
// of any group of G proofs (msm_geom_batch(g, G)) with at least k0_min sorted entries per level-0 thread, at every round
// count 0 .. MSM_BA_MAX_ROUNDS and, when the MSM's sorted list is shared with another MSM (`shared_pad`), at every larger
// bucket padding too: a list padded for the other MSM's rounds is walked at its padded length, with or without rounds.
// Each term of msm_ws_bytes grows at most G-fold from one proof to G at the same k0, rounds and padding, and falls with k0,
// but for the padded length MsmBaPlan::make rounds down to a multiple of 2^pad: G proofs' sum can round to up to 2^pad - 1
// slots more than G times one proof's, so one proof is counted with that many entries more.
template <class F>
uint64_t msm_batch_bytes_per_proof(MsmGeom g, int k0_min, bool shared_pad) {
  g = msm_geom_batch(g, 1);
  g.k0 = k0_min;
  const uint64_t entries = g.max_entries;
  MsmRedPlan plan;
  plan.make(g.c - 1);
  uint64_t worst = 0;
  for (int R = 0; R <= MSM_BA_MAX_ROUNDS; R++)
    for (int pad = R; pad <= (shared_pad ? MSM_BA_MAX_ROUNDS : R); pad++) {
      g.ba = R;
      g.ba_pad = pad;
      g.max_entries = entries + (1u << pad) - 1;
      MsmBaPlan bap;
      bap.make(g);
      worst = std::max(worst, msm_ws_bytes<F>(g, bap, plan).total());
    }
  return worst;
}

template <class F>
struct MsmWorkspace {
  DevBuf counters, offsets, blocktot, sidx, skey, buckets, pk0, pp0, pk1, pp1, pending, red_inner, red_leaf;
  DevBuf ba_pre, ba_prod, ba_pre2, ba_l0, ba_l1;
  MsmBaPlan bap;
  MsmRedPlan plan;
  int plan_m = -1, plan_ne = 0;
  XYZZ<F>* h_leaf = nullptr;  // pinned host copy of the leaf arrays: [node][window][element]
  size_t h_cap = 0;
  uint32_t* h_total = nullptr;  // pinned: number of sorted slots of the last MSM (entries + bucket padding)
  cudaError_t prepare(const MsmGeom& g) {
    cudaError_t e;
    bap.make(g);
    if (plan_m != g.c - 1 || plan_ne != g.ne) {
      plan.make(g.c - 1);
      plan_m = g.c - 1;
      plan_ne = g.ne;
    }
    const MsmWsBytes b = msm_ws_bytes<F>(g, bap, plan);   // 0 bytes (no rounds): reserve keeps what the buffer has
#define G16_TRY(x) if ((e = (x)) != cudaSuccess) return e
    G16_TRY(ba_pre.reserve(b.ba_pre));
    G16_TRY(ba_prod.reserve(b.ba_prod));
    G16_TRY(ba_pre2.reserve(b.ba_pre2));
    G16_TRY(ba_l0.reserve(b.ba_l0));
    G16_TRY(ba_l1.reserve(b.ba_l1));
    G16_TRY(counters.reserve(b.counters));
    G16_TRY(offsets.reserve(b.offsets));
    G16_TRY(blocktot.reserve(b.blocktot));
    G16_TRY(sidx.reserve(b.sidx));
    G16_TRY(skey.reserve(b.skey));
    G16_TRY(buckets.reserve(b.buckets));
    G16_TRY(pk0.reserve(b.pk0));
    G16_TRY(pp0.reserve(b.pp0));
    G16_TRY(pk1.reserve(b.pk1));
    G16_TRY(pp1.reserve(b.pp1));
    G16_TRY(pending.reserve(b.pending));
    G16_TRY(red_inner.reserve(b.red_inner));
    G16_TRY(red_leaf.reserve(b.red_leaf));
    if (!h_total) G16_TRY(cudaMallocHost(&h_total, 16));
    const size_t need = plan.leaf_pts * g.sets();
    if (h_cap < need) {
      if (h_leaf) cudaFreeHost(h_leaf);
      h_leaf = nullptr;
      G16_TRY(cudaMallocHost(&h_leaf, need * sizeof(XYZZ<F>)));
      h_cap = need;
    }
#undef G16_TRY
    return cudaSuccess;
  }
  ~MsmWorkspace() {   // the DevBuf members free themselves
    if (h_leaf) cudaFreeHost(h_leaf);
    if (h_total) cudaFreeHost(h_total);
  }
};

struct MsmCounters {  // launch bookkeeping for bench.py's gpu_launches
  unsigned long long launches = 0;
};

// Enqueue one MSM on `st`.  d_bases holds g.copies * g.n affine points (copy-major); d_scalars / d_skip are device
// pointers, pair i uses the scalar at d_scalars + FrF::N * i * scalar_stride (stride = world size for a sharded key); the leaf arrays of the bucket reduction land in ws.h_leaf once the stream is synchronised (msm_finish).
// The sorted (bucket-major, padded) entry list of an MSM, as another MSM over the SAME scalars, skip mask and geometry may
// borrow it: B in G1 and B in G2 (prover.rs:101,113) share scalars, and their queries share the identity pattern
// (b_g1_query[i] and b_g2_query[i] are both b_i(tau) times a generator), so one counting sort serves both.
struct MsmSorted {
  const uint32_t* sidx = nullptr;
  const uint32_t* skey = nullptr;
  const uint32_t* total0 = nullptr;
  cudaEvent_t ready = nullptr;   // recorded on the lender's stream once the list is complete
};
// A batched geometry (g.batch > 1) runs g.batch MSMs over the same bases in one pass: MSM k reads its scalars at
// d_scalars + k * batch_stride (32-bit words) and its result is msm_finish(ws, g, k).
template <class F, class FrF>
cudaError_t msm_enqueue(cudaStream_t st, MsmWorkspace<F>& ws, const MsmGeom& g, const Affine<F>* d_bases,
                        const uint8_t* d_skip, const uint32_t* d_scalars, uint32_t scalar_stride, bool scalars_mont,
                        MsmCounters* ctr, cudaEvent_t ev_acc0, cudaEvent_t ev_acc1, MsmSorted* lend, const MsmSorted* borrow,
                        cudaEvent_t gate_accum, uint64_t batch_stride) {
  cudaError_t e;
  if (g.n == 0) return cudaSuccess;
  if ((e = ws.prepare(g)) != cudaSuccess) return e;
  uint32_t* counters = ws.counters.template as<uint32_t>();
  uint32_t* offsets = ws.offsets.template as<uint32_t>();
  uint32_t* blocktot = ws.blocktot.template as<uint32_t>();
  uint32_t* sidx = ws.sidx.template as<uint32_t>();
  uint32_t* skey = ws.skey.template as<uint32_t>();
  uint32_t* pending = ws.pending.template as<uint32_t>();
  XYZZ<F>* buckets = ws.buckets.template as<XYZZ<F>>();
  unsigned long long nl = 0;
  cudaMemsetAsync(pending, 0, 64 * 4, st);
  cudaMemsetAsync(buckets, 0, (size_t)g.nkeys * sizeof(XYZZ<F>), st);
  const MsmBaPlan& bp = ws.bap;
  const uint32_t* total0 = offsets + g.nkeys;
  if (borrow) {
    // same scalars, mask and geometry as the lender: wait for its list instead of sorting again
    cudaStreamWaitEvent(st, borrow->ready, 0);
    sidx = const_cast<uint32_t*>(borrow->sidx);
    skey = const_cast<uint32_t*>(borrow->skey);
    total0 = borrow->total0;
  } else {
    cudaMemsetAsync(counters, 0, (size_t)(g.nkeys + 1) * 4, st);
    const dim3 nb((g.n + 255) / 256, g.batch > 1 ? g.batch : 1u);
    msm_digits<FrF, false><<<nb, 256, 0, st>>>(d_scalars, scalar_stride, scalars_mont ? 1 : 0, d_skip, g, counters, nullptr, batch_stride);
    const uint32_t pad_mask = bp.pad > 0 ? (1u << bp.pad) - 1 : 0;
    const uint32_t sb = (g.nkeys + SCAN_BLOCK - 1) / SCAN_BLOCK;
    msm_scan_blocks<<<sb, 1024, 0, st>>>(counters, g.nkeys, offsets, blocktot, pad_mask);
    msm_scan_tops<<<1, 1024, 0, st>>>(blocktot, sb, offsets + g.nkeys);
    msm_scan_fix<<<sb, 1024, 0, st>>>(offsets, g.nkeys, blocktot, counters);
    msm_digits<FrF, true><<<nb, 256, 0, st>>>(d_scalars, scalar_stride, scalars_mont ? 1 : 0, d_skip, g, counters, sidx, batch_stride);
    const uint64_t fill_warps_per_block = MSM_FILL_BLOCK / 32;
    msm_pad_fill<<<(unsigned)((g.nkeys + fill_warps_per_block - 1) / fill_warps_per_block), MSM_FILL_BLOCK, 0, st>>>(counters, offsets, g.nkeys, sidx, skey);
    nl += 6;
    if (lend) {
      lend->sidx = sidx;
      lend->skey = skey;
      lend->total0 = total0;
      if (lend->ready) cudaEventRecord(lend->ready, st);
    }
  }
  // batched-affine rounds: the (padded) sorted slots shrink 2^R-fold to a list of partial bucket sums (msm_ba.cuh)
  const Affine<F>* acc_bases = d_bases;
  const uint32_t* acc_sidx = sidx;
  // optional gate between the sort and the accumulation (engine: "witness map first" schedule of small / sharded proofs)
  if (gate_accum) cudaStreamWaitEvent(st, gate_accum, 0);
  if (ev_acc0) cudaEventRecord(ev_acc0, st);
  if (bp.R > 0) {
    Affine<F>* lists[2] = {ws.ba_l0.template as<Affine<F>>(), ws.ba_l1.template as<Affine<F>>()};
    for (int r = 0; r < bp.R; r++) {
      BaRound<F> a;
      a.in = r == 0 ? d_bases : lists[(r - 1) & 1];
      a.sidx = r == 0 ? sidx : nullptr;
      a.total0 = total0;
      a.shift = (uint32_t)(r + 1);
      a.m = bp.m[r];
      a.G = (uint32_t)(g.ba_G < 1 ? 1 : g.ba_G);
      a.inv_gcd = (uint32_t)g.ba_gcd;
      a.pre = ws.ba_pre.template as<F>();
      a.prod = ws.ba_prod.template as<F>();
      a.pre2 = ws.ba_pre2.template as<F>();
      a.out = lists[r & 1];
      const uint64_t T = ba_threads(bp.len[r + 1], a.m), lanes = (T + a.G - 1) / a.G;
      const unsigned nblk = (unsigned)((T + 127) / 128);
      ba_forward_kernel<F><<<nblk, 128, 0, st>>>(a);
      ba_combine_kernel<F><<<(unsigned)((lanes + 31) / 32), 32, 0, st>>>(a);
      ba_backward_kernel<F><<<nblk, 128, 0, st>>>(a);
      nl += 3;
    }
    acc_bases = lists[(bp.R - 1) & 1];
    acc_sidx = nullptr;
  }
  // level 0
  const uint64_t T0 = bp.l0_threads(g);
  const uint32_t K0 = bp.R > 0 ? (uint32_t)bp.k0_final : (uint32_t)g.k0;
  uint32_t* kk[2] = {ws.pk0.template as<uint32_t>(), ws.pk1.template as<uint32_t>()};
  XYZZ<F>* pp[2] = {ws.pp0.template as<XYZZ<F>>(), ws.pp1.template as<XYZZ<F>>()};
  {
    const unsigned tpb = (g.acc_block == 32 || g.acc_block == 64) ? (unsigned)g.acc_block : 128u;
    msm_accum_l0<F><<<(unsigned)((T0 + tpb - 1) / tpb), tpb, 0, st>>>(acc_bases, acc_sidx, skey, (uint32_t)bp.R, total0, T0, K0, buckets, kk[0], pp[0], pending);
  }
  if (ev_acc1) cudaEventRecord(ev_acc1, st);
  nl += 1;
  // levels >= 1: ping-pong between the two partial buffers, then one fused tail; empty levels return immediately
  uint64_t S = 2 * T0;
  int cur = 0, lvl = 0;
  while (S > (uint64_t)MSM_TAIL_S && lvl < 60) {
    const uint64_t T = msm_level_threads(S, MSM_KF);
    msm_accum_ln<F, MSM_KF><<<(unsigned)((T + 127) / 128), 128, 0, st>>>(kk[cur], pp[cur], S, T, buckets, kk[cur ^ 1], pp[cur ^ 1], pending + lvl);
    nl += 1;
    S = 2 * T;
    cur ^= 1;
    lvl++;
  }
  msm_accum_tail<F, MSM_KF><<<1, 256, 0, st>>>(kk[cur], pp[cur], kk[cur ^ 1], pp[cur ^ 1], S, buckets, pending + lvl);
  nl += 1;
  // bucket reduction: row / column sums down the plan, leaves to the host
  constexpr int TPB = sizeof(XYZZ<F>) > 192 ? 64 : 128;
  const MsmRedPlan& pl = ws.plan;
  XYZZ<F>* inner = ws.red_inner.template as<XYZZ<F>>();
  XYZZ<F>* leaf = ws.red_leaf.template as<XYZZ<F>>();
  auto arr = [&](int id) -> XYZZ<F>* {
    if (id == 0) return buckets;
    const MsmRedNode& nd = pl.nodes[id];
    return (nd.leaf ? leaf : inner) + nd.off * g.sets();
  };
  // one launch per depth of the plan: the row and column sums of every non-leaf node at that depth are independent jobs
  {
    int depth_of[16];
    int max_depth = 0;
    depth_of[0] = 0;
    for (int id = 0; id < pl.n_nodes; id++) {   // parents precede children in the node array
      const MsmRedNode& nd = pl.nodes[id];
      if (nd.leaf) continue;
      depth_of[nd.child_r] = depth_of[nd.child_c] = depth_of[id] + 1;
      if (depth_of[id] > max_depth) max_depth = depth_of[id];
    }
    for (int d = 0; d <= max_depth; d++) {
      MsmSumJobs<F> jobs;
      jobs.n = 0;
      uint32_t blocks = 0;
      auto flush = [&]() {
        if (jobs.n) {
          msm_sum_strided<F, TPB><<<blocks, TPB, 0, st>>>(jobs);
          nl += 1;
        }
        jobs.n = 0;
        blocks = 0;
      };
      for (int id = 0; id < pl.n_nodes; id++) {
        const MsmRedNode& nd = pl.nodes[id];
        if (nd.leaf || depth_of[id] != d) continue;
        for (int side = 0; side < 2; side++) {
          const bool rows = side == 0;
          MsmSumJob<F>& jb = jobs.j[jobs.n];
          jb.in = arr(id);
          jb.out = arr(rows ? nd.child_r : nd.child_c);
          jb.per_win_out = rows ? (1u << nd.a1) : (1u << nd.a0);
          jb.win_stride = 1u << nd.log_len;
          jb.len = rows ? (1u << nd.a0) : (1u << nd.a1);
          jb.stride = rows ? 1u : (1u << nd.a0);
          jb.base_mul = rows ? (1u << nd.a0) : 1u;
          jb.n_out = jb.per_win_out * g.sets();
          uint32_t tpo = TPB;
          while (tpo > jb.len) tpo >>= 1;
          jb.tpo = tpo;
          jb.first_block = blocks;
          blocks += (jb.n_out + TPB / tpo - 1) / (TPB / tpo);
          if (++jobs.n == 4) flush();
        }
      }
      flush();
    }
  }
  if (ctr) ctr->launches += nl;
  const XYZZ<F>* leaf_src = pl.nodes[0].leaf ? buckets : leaf;
  cudaMemcpyAsync(ws.h_total, total0, 4, cudaMemcpyDeviceToHost, st);
  e = cudaMemcpyAsync(ws.h_leaf, leaf_src, pl.leaf_pts * g.sets() * sizeof(XYZZ<F>), cudaMemcpyDeviceToHost, st);
  if (e != cudaSuccess) return e;
  return cudaGetLastError();
}

// Host end of the bucket reduction (stream must be synchronised): weighted sums of the leaf arrays, recombination up
// the plan, then Horner over the effective windows: sum_e 2^(c e) S_e.
template <class F>
struct MsmHostRed {
  const MsmWorkspace<F>& ws;
  const MsmGeom& g;
  int w;   // bucket set (of all g.sets() in the pass)
  // returns T(node) = sum_i (i + 1) X_i and sets total = sum_i X_i
  XYZZ<F> T(int id, XYZZ<F>& total) const {
    const MsmRedNode& nd = ws.plan.nodes[id];
    if (nd.leaf) {
      const size_t len = (size_t)1 << nd.log_len;
      const XYZZ<F>* x = ws.h_leaf + nd.off * g.sets() + (size_t)w * len;
      XYZZ<F> running = XYZZ<F>::inf(), acc = XYZZ<F>::inf();
      for (size_t i = len; i-- > 0;) {
        running.add(x[i]);
        acc.add(running);
      }
      total = running;
      return acc;
    }
    XYZZ<F> tot_r, tot_c;
    XYZZ<F> tr = T(nd.child_r, tot_r);   // sum (hi + 1) R_hi
    XYZZ<F> tc = T(nd.child_c, tot_c);   // sum (lo + 1) C_lo
    tot_r.negate();
    tr.add(tot_r);                       // sum hi R_hi
    for (int k = 0; k < nd.a0; k++) tr.dbl_inplace();
    tr.add(tc);
    total = tot_c;
    return tr;
  }
};
// `k`: which MSM of a batched pass (its bucket sets are k*ne .. k*ne+ne-1)
template <class F>
XYZZ<F> msm_finish(const MsmWorkspace<F>& ws, const MsmGeom& g, uint32_t k = 0) {
  XYZZ<F> acc = XYZZ<F>::inf();
  if (g.n == 0) return acc;
  for (int w = g.ne - 1; w >= 0; w--) {
    for (int i = 0; i < g.c; i++) acc.dbl_inplace();
    MsmHostRed<F> hr{ws, g, (int)(k * g.ne) + w};
    XYZZ<F> tot;
    acc.add(hr.T(0, tot));
  }
  return acc;
}

// Make a query resident: identity mask of copy 0 and (copies > 1) the precomputed multiples 2^(shift*j) * P.
template <class F>
cudaError_t msm_prepare_query(cudaStream_t st, Affine<F>* d_bases, uint32_t cnt, int copies, int shift, uint8_t* d_mask) {
  if (!cnt) return cudaSuccess;
  msm_inf_mask<F><<<(cnt + 255) / 256, 256, 0, st>>>(d_bases, cnt, d_mask);
  if (copies > 1) msm_precompute<F><<<(cnt + 127) / 128, 128, 0, st>>>(d_bases, cnt, copies, shift, d_bases);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// fixed-base batch multiplication (BatchMulPreprocessing::batch_mul, generator.rs:129-183)
// ------------------------------------------------------------------------------------------------
// 8-bit windows over the scalar's limbs: 32 for a 256-bit Fr, 48 for BW6-761's 384-bit one
template <class FrF>
constexpr int fb_windows() { return 4 * FrF::N; }
template <class F, int NW>
__global__ void fb_table_kernel(Affine<F> g, XYZZ<F>* table /* [NW][255] */) {
  const int w = threadIdx.x;
  if (w >= NW) return;
  XYZZ<F> base = XYZZ<F>::from_affine(g);
  for (int i = 0; i < 8 * w; i++) base.dbl_inplace();
  XYZZ<F> acc = base;
  for (int d = 1; d <= 255; d++) {
    table[w * 255 + d - 1] = acc;
    acc.add(base);
  }
}
template <class F, class FrF>
__global__ void __launch_bounds__(128) fb_mul_kernel(const XYZZ<F>* __restrict__ table, const FrF* __restrict__ scalars,
                                                     uint32_t n, Affine<F>* __restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  FrF s;
  {
    const uint4* p = reinterpret_cast<const uint4*>(scalars + i);
#pragma unroll
    for (int j = 0; j < FrF::N / 4; j++) {
      const uint4 x = __ldg(p + j);
      s.v[4 * j] = x.x; s.v[4 * j + 1] = x.y; s.v[4 * j + 2] = x.z; s.v[4 * j + 3] = x.w;
    }
  }
  s = FrF::from_mont(s);
  XYZZ<F> acc = XYZZ<F>::inf();
  for (int w = 0; w < fb_windows<FrF>(); w++) {
    const uint32_t d = (s.v[w >> 2] >> (8 * (w & 3))) & 0xff;
    if (d) acc.add(table[w * 255 + d - 1]);
  }
  out[i] = acc.to_affine();
}
// d_table: fb_windows<FrF>() * 255 XYZZ points of scratch
template <class F, class FrF>
cudaError_t fb_batch_mul(cudaStream_t st, const Affine<F>& gen, const FrF* d_scalars, uint64_t cnt, Affine<F>* d_out,
                         XYZZ<F>* d_table) {
  fb_table_kernel<F, fb_windows<FrF>()><<<1, fb_windows<FrF>(), 0, st>>>(gen, d_table);
  if (cnt) fb_mul_kernel<F, FrF><<<(unsigned)((cnt + 127) / 128), 128, 0, st>>>(d_table, d_scalars, (uint32_t)cnt, d_out);
  return cudaGetLastError();
}
// d_out[i] = d_scalars[i] * gen for a table fb_batch_mul already built (batch proving: one table per key point)
template <class F, class FrF>
cudaError_t fb_mul(cudaStream_t st, const XYZZ<F>* d_table, const FrF* d_scalars, uint64_t cnt, Affine<F>* d_out) {
  if (cnt) fb_mul_kernel<F, FrF><<<(unsigned)((cnt + 127) / 128), 128, 0, st>>>(d_table, d_scalars, (uint32_t)cnt, d_out);
  return cudaGetLastError();
}

// Explicit-instantiation lists: kernels are compiled in their own translation units (k_msm_*.cu), the engine TU only
// declares them `extern template` (keeps ptxas work parallel across make jobs).
#define G16_MSM_TEMPLATES(X, F, FrF)                                                                                     \
  X cudaError_t msm_enqueue<F, FrF>(cudaStream_t, MsmWorkspace<F>&, const MsmGeom&, const Affine<F>*, const uint8_t*,    \
                                    const uint32_t*, uint32_t, bool, MsmCounters*, cudaEvent_t, cudaEvent_t, MsmSorted*, \
                                    const MsmSorted*, cudaEvent_t, uint64_t);                                            \
  X cudaError_t msm_prepare_query<F>(cudaStream_t, Affine<F>*, uint32_t, int, int, uint8_t*);                            \
  X cudaError_t fb_batch_mul<F, FrF>(cudaStream_t, const Affine<F>&, const FrF*, uint64_t, Affine<F>*, XYZZ<F>*);       \
  X cudaError_t fb_mul<F, FrF>(cudaStream_t, const XYZZ<F>*, const FrF*, uint64_t, Affine<F>*);

}  // namespace g16
