// zkey.cuh -- snarkjs .zkey files (Groth16, as snarkjs zkey_utils.js writes them and ark-circom's read_zkey reads them):
// the host walk of the section table and header, and the device decode of the coefficient section into the resident CSR
// matrices A and B.  The points go through ser.cuh (ser_decode_mont) and the serialized-key staging of engine.cuh.
//
// File: "zkey", version u32 = 1, nSections u32, then nSections records {id u32, size u64, size bytes}; ids 1 .. 9 exactly
// once each, in any order; ids >= 10 are skipped (10: the MPC contributions).  All integers little-endian.
//   1  protocol u32 = 1 (Groth16), size 4
//   2  n8q, q, n8r, r, nVars, nPublic, domainSize, alpha1, beta1, beta2, gamma2, delta1, delta2 (exact size)
//   3  IC: nPublic + 1 G1                    5 A: nVars G1      6 B1: nVars G1      7 B2: nVars G2
//   4  nCoefs u32, then nCoefs records {matrix u32 (0 = A, 1 = B), constraint u32, signal u32, value (n8r bytes)}; value
//      is the canonical c R_r^2 mod r, so one Montgomery reduction gives the ABI's c R_r
//   8  C: nVars - nPublic - 1 G1            9 H: domainSize G1
// snarkjs appends to A, for s = 0 .. nPublic, row nConstraints + s = {(s, 1)}; B has no entries there.  The reader derives
// num_constraints = (largest constraint index) - nPublic and drops those rows: CircomReduction appends them itself.
#pragma once
#include <cstring>
#include <string>
#include <vector>
#include "ser.cuh"

namespace g16 {

// ---- one coefficient record ------------------------------------------------------------------------------------------
// per-record result codes, in the order they are checked; zkey_coef_reason() gives the field each refers to
enum : uint32_t { ZK_OK = 0, ZK_ERR_MATRIX = 1, ZK_ERR_CONSTRAINT = 2, ZK_ERR_SIGNAL = 3, ZK_ERR_VALUE = 4 };
G16_HD uint32_t zk_u32(const uint8_t* p) {
#ifdef __CUDA_ARCH__
  return *reinterpret_cast<const uint32_t*>(p);   // records start 4-byte aligned in the device copy
#else
  uint32_t w;
  memcpy(&w, p, 4);
  return w;
#endif
}
struct ZkeyCoef {
  uint32_t matrix, constraint, signal;
};
// rec: 12 + 4 Fr::N bytes.  Returns ZK_OK with the indices and the Montgomery value c R_r, or the first failing check.
template <class P>
G16_HD uint32_t zkey_coef_decode(const uint8_t* rec, uint32_t domain_size, uint32_t nvars, ZkeyCoef& c, Fp<P>& val) {
  c.matrix = zk_u32(rec);
  c.constraint = zk_u32(rec + 4);
  c.signal = zk_u32(rec + 8);
  if (c.matrix >= 2) return ZK_ERR_MATRIX;
  if (c.constraint >= domain_size) return ZK_ERR_CONSTRAINT;
  if (c.signal >= nvars) return ZK_ERR_SIGNAL;
  Fp<P> v;
#pragma unroll
  for (int i = 0; i < P::N; i++) v.v[i] = zk_u32(rec + 12 + 4 * i);
  if (!ser_lt_mod(v)) return ZK_ERR_VALUE;
  val = Fp<P>::from_mont(v);   // (c R^2) R^-1
  return ZK_OK;
}

#ifdef __CUDACC__
// One thread per record of a chunk (rec: the chunk's device copy, rs bytes per record; off0: byte offset of its first
// record in the file).  A refused record lands in *err as (byte offset << 8 | code), the smallest winning; an accepted one
// has its value replaced in place by c R_r (the first 4 Fr::N bytes after the indices), is counted in counts[matrix
// domain_size + constraint], and raises *row_end to constraint + 1.
template <class Fr>
__global__ void __launch_bounds__(256) zkey_coef_kernel(uint8_t* rec, uint32_t count, uint32_t rs, uint64_t off0,
                                                        uint32_t domain_size, uint32_t nvars, uint32_t* counts,
                                                        uint32_t* row_end, unsigned long long* err) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t end = 0;
  if (t < count) {
    uint8_t* r = rec + (uint64_t)t * rs;
    ZkeyCoef c;
    Fr v;
    const uint32_t code = zkey_coef_decode(r, domain_size, nvars, c, v);
    if (code) {
      atomicMin(err, ((off0 + (uint64_t)t * rs) << 8) | code);
    } else {
      uint32_t* w = reinterpret_cast<uint32_t*>(r + 12);
#pragma unroll
      for (int i = 0; i < Fr::N; i++) w[i] = v.v[i];
      atomicAdd(counts + (size_t)c.matrix * domain_size + c.constraint, 1u);
      end = c.constraint + 1;
    }
  }
  end = __reduce_max_sync(0xffffffffu, end);   // one atomic per warp: every record hits the same word
  if ((threadIdx.x & 31) == 0 && end) atomicMax(row_end, end);
}

// Places each decoded record of a chunk: rows below nc into the CSR arrays of its matrix (position row_ptr[row] plus a
// slot taken by counting counts[row] back down to 0; the order within a row is free, field sums being exact), rows nc + s
// (the appended public-input rows) checked against A = {(s, 1)}, B = {}: a mismatch lands in *pub_err as 2 s + matrix.
struct ZkeyCsr {
  const uint32_t* row_ptr;
  uint32_t* col;
  void* val;
};
template <class Fr>
__global__ void __launch_bounds__(256) zkey_scatter_kernel(const uint8_t* rec, uint32_t count, uint32_t rs, uint32_t nc,
                                                           ZkeyCsr a, ZkeyCsr b, uint32_t* counts, uint32_t domain_size,
                                                           uint32_t* pub_err) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= count) return;
  const uint8_t* r = rec + (uint64_t)t * rs;
  const uint32_t m = zk_u32(r), row = zk_u32(r + 4), col = zk_u32(r + 8);
  Fr v;
#pragma unroll
  for (int i = 0; i < Fr::N; i++) v.v[i] = zk_u32(r + 12 + 4 * i);
  if (row < nc) {
    const ZkeyCsr& x = m ? b : a;
    const uint32_t pos = x.row_ptr[row] + atomicSub(counts + (size_t)m * domain_size + row, 1u) - 1;
    x.col[pos] = col;
    reinterpret_cast<Fr*>(x.val)[pos] = v;
  } else {
    const uint32_t s = row - nc;
    if (m == 1 || col != s || v != Fr::one()) atomicMin(pub_err, 2 * s + m);
  }
}
// public-input row s (s <= npub): A holds exactly one entry and B none
static __global__ void zkey_pub_rows_kernel(const uint32_t* counts, uint32_t domain_size, uint32_t nc, uint32_t npub,
                                     uint32_t* pub_err) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s > npub) return;
  if (counts[nc + s] != 1) atomicMin(pub_err, 2 * s);
  if (counts[(size_t)domain_size + nc + s] != 0) atomicMin(pub_err, 2 * s + 1);
}

// Exclusive prefix sum out[i] = sum_{j < i} in[j] over i <= n (in[n] read as 0, so out[n] is the total): per-block scans of
// 1024 elements, one block scanning the block totals with a running carry, and the fix-up.
__device__ __forceinline__ uint32_t zkey_block_scan(uint32_t v, uint32_t* total) {
  __shared__ uint32_t warp_tot[32];
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= (uint32_t)d) x += y;
  }
  if (lane == 31) warp_tot[wid] = x;
  __syncthreads();
  if (wid == 0) {
    uint32_t w = lane < (blockDim.x >> 5) ? warp_tot[lane] : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= (uint32_t)d) w += y;
    }
    warp_tot[lane] = w;   // inclusive over warps
  }
  __syncthreads();
  const uint32_t ex = x - v + (wid ? warp_tot[wid - 1] : 0);
  *total = warp_tot[(blockDim.x >> 5) - 1];
  __syncthreads();   // warp_tot is reused by the next call
  return ex;
}
static __global__ void __launch_bounds__(1024) zkey_scan_blocks(const uint32_t* in, uint32_t n, uint32_t* out, uint32_t* block_tot) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t tot;
  const uint32_t ex = zkey_block_scan(i < n ? in[i] : 0u, &tot);
  if (i <= n) out[i] = ex;
  if (threadIdx.x == 0) block_tot[blockIdx.x] = tot;
}
static __global__ void __launch_bounds__(1024) zkey_scan_tops(uint32_t* block_tot, uint32_t nblocks) {
  uint32_t carry = 0;
  for (uint32_t b0 = 0; b0 < nblocks; b0 += blockDim.x) {
    const uint32_t i = b0 + threadIdx.x;
    const uint32_t v = i < nblocks ? block_tot[i] : 0u;
    uint32_t tot;
    const uint32_t ex = zkey_block_scan(v, &tot);
    if (i < nblocks) block_tot[i] = carry + ex;
    carry += tot;
  }
}
static __global__ void __launch_bounds__(1024) zkey_scan_fix(uint32_t* out, uint32_t n, const uint32_t* block_tot) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= n) out[i] += block_tot[blockIdx.x];
}

template <class Fr>
cudaError_t zkey_coef_enqueue(cudaStream_t st, uint8_t* rec, uint32_t count, uint32_t rs, uint64_t off0, uint32_t domain_size,
                              uint32_t nvars, uint32_t* counts, uint32_t* row_end, unsigned long long* err) {
  if (!count) return cudaSuccess;
  zkey_coef_kernel<Fr><<<(count + 255) / 256, 256, 0, st>>>(rec, count, rs, off0, domain_size, nvars, counts, row_end, err);
  return cudaGetLastError();
}
// row_ptr of both matrices (nc + 1 entries each) from the counts of rows < nc, and the public-input-row check: seven
// launches.  block_tot: at least (nc + 1 + 1023) / 1024 words.
inline cudaError_t zkey_row_ptr_enqueue(cudaStream_t st, const uint32_t* counts, uint32_t nc, uint32_t npub, uint32_t domain_size,
                                        uint32_t* rp_a, uint32_t* rp_b, uint32_t* block_tot, uint32_t* pub_err,
                                        unsigned long long* launches) {
  const uint32_t nb = (nc + 1 + 1023) / 1024;
  for (int m = 0; m < 2; m++) {
    uint32_t* rp = m ? rp_b : rp_a;
    zkey_scan_blocks<<<nb, 1024, 0, st>>>(counts + (size_t)m * domain_size, nc, rp, block_tot);
    zkey_scan_tops<<<1, 1024, 0, st>>>(block_tot, nb);
    zkey_scan_fix<<<nb, 1024, 0, st>>>(rp, nc, block_tot);
  }
  zkey_pub_rows_kernel<<<(npub + 1 + 255) / 256, 256, 0, st>>>(counts, domain_size, nc, npub, pub_err);
  *launches += 7;
  return cudaGetLastError();
}
// every decoded record into the CSR arrays, one launch per `chunk` records
template <class Fr>
cudaError_t zkey_scatter_enqueue(cudaStream_t st, const uint8_t* rec, uint64_t ncoefs, uint32_t chunk, uint32_t rs, uint32_t nc,
                                 uint32_t domain_size, uint32_t* counts, ZkeyCsr a, ZkeyCsr b, uint32_t* pub_err,
                                 unsigned long long* launches) {
  for (uint64_t f = 0; f < ncoefs; f += chunk) {
    const uint32_t cnt = (uint32_t)(ncoefs - f < chunk ? ncoefs - f : chunk);
    zkey_scatter_kernel<Fr><<<(cnt + 255) / 256, 256, 0, st>>>(rec + f * rs, cnt, rs, nc, a, b, counts, domain_size, pub_err);
    *launches += 1;
  }
  return cudaGetLastError();
}
// the .zkey kernels of one curve: the coefficient decode and CSR build, and the Montgomery little-endian point decode.
// Instantiated for the curves snarkjs writes (BN254, BLS12-381) only.
#define G16_ZKEY_TEMPLATES(X, CP)                                                                                      \
  X cudaError_t zkey_coef_enqueue<Fp<CP::FrP>>(cudaStream_t, uint8_t*, uint32_t, uint32_t, uint64_t, uint32_t, uint32_t, \
                                               uint32_t*, uint32_t*, unsigned long long*);                              \
  X cudaError_t zkey_scatter_enqueue<Fp<CP::FrP>>(cudaStream_t, const uint8_t*, uint64_t, uint32_t, uint32_t, uint32_t, \
                                                  uint32_t, uint32_t*, ZkeyCsr, ZkeyCsr, uint32_t*, unsigned long long*); \
  X cudaError_t ser_decode_enqueue<CP, false, true>(cudaStream_t, const uint8_t*, uint64_t, uint32_t, uint32_t, uint64_t, \
                                                    SerDest, unsigned long long*);                                      \
  X cudaError_t ser_decode_enqueue<CP, true, true>(cudaStream_t, const uint8_t*, uint64_t, uint32_t, uint32_t, uint64_t,  \
                                                   SerDest, unsigned long long*);
#endif

// ---- the host walk ---------------------------------------------------------------------------------------------------
struct ZkeyLayout {
  uint64_t off[10] = {}, size[10] = {};   // body offset and size of sections 1 .. 9
  uint32_t nvars = 0, npub = 0, domain_size = 0, ncoefs = 0;
  uint32_t rs = 0;                        // bytes per coefficient record
  uint64_t coef_off = 0;                  // byte offset of the first record
  SerItem it[SER_ITEMS];                  // the points, as the members of ser.cuh's ProvingKey order, at their file offsets
};
// the point member (name, index) holding byte `off` of the file
inline std::string zkey_locate(const ZkeyLayout& z, uint64_t off) {
  for (int m = 0; m < SER_ITEMS; m++) {
    const SerItem& x = z.it[m];
    if (off >= x.off && off < x.off + x.len * x.psize) {
      if (!x.vec) return x.name;
      return std::string(x.name) + "[" + std::to_string((off - x.off) / x.psize) + "]";
    }
  }
  return "?";
}
inline uint64_t zk_u64(const uint8_t* p) {
  uint64_t w;
  memcpy(&w, p, 8);
  return w;
}
// little-endian bytes == the limbs of P's modulus
template <class P>
bool zkey_is_modulus(const uint8_t* p) {
  for (int i = 0; i < P::N; i++)
    if (zk_u32(p + 4 * i) != P::mod(i)) return false;
  return true;
}
// Walks the section table and decides every size and header field of the file for curve CP from the bytes alone.  Returns
// "" and fills z, or why the file is refused (the first problem in file order).
template <class CP>
std::string zkey_walk(const uint8_t* b, uint64_t len, ZkeyLayout& z) {
  using Fmt = SerFormat<CP>;
  constexpr uint32_t NQ = Fmt::NB, NR = 4 * CP::FrP::N, G1 = 2 * NQ, G2 = 4 * NQ;
  z = ZkeyLayout{};
  if (len < 12) return "truncated input: " + std::to_string(len) + " bytes, a .zkey header is 12";
  if (memcmp(b, "zkey", 4) != 0) return "not a .zkey file (magic is not \"zkey\")";
  if (zk_u32(b + 4) != 1) return "unsupported .zkey version " + std::to_string(zk_u32(b + 4)) + " (expected 1)";
  const uint32_t nsec = zk_u32(b + 8);
  uint64_t pos = 12;
  bool seen[10] = {};
  for (uint32_t k = 0; k < nsec; k++) {
    if (len - pos < 12)
      return "truncated input: section " + std::to_string(k) + " of " + std::to_string(nsec) + " has no complete header at byte " +
             std::to_string(pos);
    const uint32_t id = zk_u32(b + pos);
    const uint64_t size = zk_u64(b + pos + 4);
    pos += 12;
    if (size > len - pos)
      return "truncated input: section " + std::to_string(id) + " at byte " + std::to_string(pos) + " declares " +
             std::to_string(size) + " bytes, " + std::to_string(len - pos) + " remain";
    if (id == 0) return "section id 0 at byte " + std::to_string(pos - 12);
    if (id <= 9) {
      if (seen[id]) return "section " + std::to_string(id) + " appears twice";
      seen[id] = true;
      z.off[id] = pos;
      z.size[id] = size;
    }
    pos += size;
  }
  if (pos != len) return "trailing bytes after the last section (" + std::to_string(len - pos) + ")";
  for (int id = 1; id <= 9; id++)
    if (!seen[id]) return "section " + std::to_string(id) + " is missing";
  auto bad_size = [&](int id, const char* what, uint64_t want) {
    return "section " + std::to_string(id) + " (" + what + "): size " + std::to_string(z.size[id]) + ", expected " +
           std::to_string(want);
  };
  if (z.size[1] != 4) return bad_size(1, "protocol", 4);
  if (zk_u32(b + z.off[1]) != 1)
    return "section 1: protocol " + std::to_string(zk_u32(b + z.off[1])) + " is not Groth16 (1)";
  // section 2: the fixed fields are read only where the section holds them
  const uint8_t* h = b + z.off[2];
  const uint64_t s2 = z.size[2];
  if (s2 < 4) return bad_size(2, "header", 4ull + NQ + 4 + NR + 12 + 3ull * G1 + 3ull * G2);
  const uint32_t n8q = zk_u32(h);
  if (n8q != NQ)
    return "section 2: n8q = " + std::to_string(n8q) + ", the context's curve has " + std::to_string(NQ) + "-byte base field elements";
  const uint64_t want2 = 4ull + NQ + 4 + NR + 12 + 3ull * G1 + 3ull * G2;
  if (s2 != want2) return bad_size(2, "header", want2);
  if (!zkey_is_modulus<typename CP::FqP>(h + 4)) return "section 2: q is not the base field modulus of the context's curve";
  const uint32_t n8r = zk_u32(h + 4 + NQ);
  if (n8r != NR) return "section 2: n8r = " + std::to_string(n8r) + ", the context's curve has " + std::to_string(NR) + "-byte scalars";
  if (!zkey_is_modulus<typename CP::FrP>(h + 8 + NQ)) return "section 2: r is not the scalar field modulus of the context's curve";
  const uint8_t* f = h + 8 + NQ + NR;
  z.nvars = zk_u32(f);
  z.npub = zk_u32(f + 4);
  z.domain_size = zk_u32(f + 8);
  if ((uint64_t)z.nvars < (uint64_t)z.npub + 1)
    return "section 2: nVars = " + std::to_string(z.nvars) + " is below nPublic + 1 = " + std::to_string((uint64_t)z.npub + 1);
  if (z.domain_size == 0 || (z.domain_size & (z.domain_size - 1)))
    return "section 2: domainSize = " + std::to_string(z.domain_size) + " is not a power of two";
  const uint64_t nw = (uint64_t)z.nvars - z.npub - 1;
  if (z.size[3] != (z.npub + 1ull) * G1) return bad_size(3, "IC", (z.npub + 1ull) * G1);
  z.rs = 12 + NR;
  if (z.size[4] < 4) return bad_size(4, "coefficients", 4);
  z.ncoefs = zk_u32(b + z.off[4]);
  z.coef_off = z.off[4] + 4;
  if (z.size[4] != 4 + (uint64_t)z.ncoefs * z.rs) return bad_size(4, "coefficients", 4 + (uint64_t)z.ncoefs * z.rs);
  if (z.size[5] != (uint64_t)z.nvars * G1) return bad_size(5, "A", (uint64_t)z.nvars * G1);
  if (z.size[6] != (uint64_t)z.nvars * G1) return bad_size(6, "B1", (uint64_t)z.nvars * G1);
  if (z.size[7] != (uint64_t)z.nvars * G2) return bad_size(7, "B2", (uint64_t)z.nvars * G2);
  if (z.size[8] != nw * G1) return bad_size(8, "C", nw * G1);
  if (z.size[9] != (uint64_t)z.domain_size * G1) return bad_size(9, "H", (uint64_t)z.domain_size * G1);
  // the points, in ser.cuh's member order, under the .zkey names
  const uint64_t p = z.off[2] + 8 + NQ + NR + 12;
  struct { int m; const char* name; bool g2, vec; uint64_t len, off; } pts[SER_ITEMS] = {
      {SER_ALPHA_G1, "alpha1", false, false, 1, p},
      {SER_BETA_G2, "beta2", true, false, 1, p + 2 * G1},
      {SER_GAMMA_G2, "gamma2", true, false, 1, p + 2 * G1 + G2},
      {SER_DELTA_G2, "delta2", true, false, 1, p + 3 * G1 + 2 * G2},
      {SER_GAMMA_ABC, "IC", false, true, z.npub + 1ull, z.off[3]},
      {SER_BETA_G1, "beta1", false, false, 1, p + G1},
      {SER_DELTA_G1, "delta1", false, false, 1, p + 2 * G1 + 2 * G2},
      {SER_A, "A", false, true, z.nvars, z.off[5]},
      {SER_B_G1, "B1", false, true, z.nvars, z.off[6]},
      {SER_B_G2, "B2", true, true, z.nvars, z.off[7]},
      {SER_H, "H", false, true, z.domain_size, z.off[9]},
      {SER_L, "C", false, true, nw, z.off[8]}};
  for (const auto& x : pts) {
    SerItem& it = z.it[x.m];
    it.name = x.name;
    it.g2 = x.g2;
    it.vec = x.vec;
    it.len = x.len;
    it.off = x.off;
    it.psize = x.g2 ? G2 : G1;
  }
  return "";
}
// The circuit the coefficients describe: num_constraints from the largest constraint index + 1 (row_end; 0 = no record),
// and the CircomReduction domain it must have.  "" or why the coefficients do not describe a circuit of this file.
inline std::string zkey_derive(const ZkeyLayout& z, uint32_t row_end, uint32_t* nc_out) {
  if ((uint64_t)row_end < z.npub + 1ull)
    return "coefficients: the largest constraint index " + (row_end ? std::to_string(row_end - 1) : std::string("(none)")) +
           " leaves no room for the " + std::to_string(z.npub + 1ull) + " public-input rows of A";
  const uint32_t nc = row_end - 1 - z.npub;
  uint64_t n = 1;
  while (n < (uint64_t)nc + z.npub + 1) n <<= 1;
  if (n != z.domain_size)
    return "section 2: domainSize = " + std::to_string(z.domain_size) + " is not the domain of the circuit (" + std::to_string(n) +
           " for " + std::to_string(nc) + " constraints and " + std::to_string(z.npub + 1ull) + " inputs)";
  *nc_out = nc;
  return "";
}
// why the record at byte `off` was refused (code from zkey_coef_decode)
inline std::string zkey_coef_reason(const uint8_t* b, const ZkeyLayout& z, uint64_t off, uint32_t code) {
  const uint64_t i = (off - z.coef_off) / z.rs;
  const uint8_t* r = b + z.coef_off + i * z.rs;
  std::string s = "coefficient " + std::to_string(i) + ": ";
  switch (code) {
    case ZK_ERR_MATRIX: return s + "matrix " + std::to_string(zk_u32(r)) + " is neither A (0) nor B (1)";
    case ZK_ERR_CONSTRAINT:
      return s + "constraint " + std::to_string(zk_u32(r + 4)) + " >= domainSize " + std::to_string(z.domain_size);
    case ZK_ERR_SIGNAL: return s + "signal " + std::to_string(zk_u32(r + 8)) + " >= nVars " + std::to_string(z.nvars);
    case ZK_ERR_VALUE: return s + "value is not a canonical field element (>= r)";
    default: return s + "unknown error";
  }
}

}  // namespace g16
