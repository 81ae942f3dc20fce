// r1cs.cuh -- circom .r1cs circuits and .wtns witnesses (iden3 r1csfile / wtnsfile, as circom writes them and ark-circom's
// R1CSFile and read_witness read them): the host walk of the section table, header and term counts, and the device decode
// of every term into the resident CSR matrices A, B and C, and of every witness element into Montgomery limbs.
//
// .r1cs: "r1cs", version u32 = 1, nSections u32, then nSections records {type u32, size u64, size bytes} in any order.  All
// integers little-endian.  Sections 1 and 2 appear exactly once; 4 and 5 (custom gates, PLONK only) are refused; every
// other section (3: the wire-to-label map) is skipped.
//   1  header, exactly 32 + n8 bytes: n8 u32, prime (n8 bytes), nWires u32, nPubOut u32, nPubIn u32, nPrvIn u32,
//      nLabels u64, mConstraints u32
//   2  mConstraints constraints, each three linear combinations A, B, C; a combination is nTerms u32, then nTerms
//      {wire u32, coefficient (n8 bytes, canonical: standard form, below the prime)}.  Constraint: A.w * B.w - C.w = 0.
// The circuit (ark-circom's R1CS::from(R1CSFile)): num_inputs = 1 + nPubOut + nPubIn, num_witness = nWires - num_inputs,
// column = wire id (wire 0 is One).  Terms stay as the file has them, in file order: zero coefficients and a wire repeated
// within a combination stay separate entries, as ark-circom pushes them; every result is a field sum, so nothing differs
// from ark-relations' compacted matrices.
//
// .wtns: "wtns", version u32 = 2, nSections u32, the same records; sections 1 and 2 exactly once each, others skipped.
//   1  n8 u32, prime (n8 bytes), nWitness u32             2  nWitness canonical n8-byte values
#pragma once
#include <cstring>
#include <string>
#include <vector>
#include "ser.cuh"

namespace g16 {

// per-item result codes; r1cs_reason() gives the message of each
enum : uint32_t { R1_OK = 0, R1_ERR_WIRE = 1, R1_ERR_VALUE = 2 };
G16_HD uint32_t r1_u32(const uint8_t* p) {
  uint32_t w;
#ifdef __CUDA_ARCH__
  // terms are 4 + n8 bytes and follow 4-byte counts, so every field starts 4-byte aligned in the staging buffer
  w = *reinterpret_cast<const uint32_t*>(p);
#else
  memcpy(&w, p, 4);
#endif
  return w;
}
// One canonical element at p (4 Fr::N bytes): R1_OK with c R in val, or R1_ERR_VALUE when it is not below r.  The
// .r1cs coefficients and the .wtns elements both go through it.
template <class P>
G16_HD uint32_t r1cs_elem_decode(const uint8_t* p, Fp<P>& val) {
  Fp<P> v;
#pragma unroll
  for (int i = 0; i < P::N; i++) v.v[i] = r1_u32(p + 4 * i);
  if (!ser_lt_mod(v)) return R1_ERR_VALUE;
  val = Fp<P>::to_mont(v);
  return R1_OK;
}
// One term at p (wire u32, coefficient): checks wire < nwires, then the coefficient.
template <class P>
G16_HD uint32_t r1cs_term_decode(const uint8_t* p, uint32_t nwires, uint32_t& wire, Fp<P>& val) {
  wire = r1_u32(p);
  if (wire >= nwires) return R1_ERR_WIRE;
  return r1cs_elem_decode(p + 4, val);
}

#ifdef __CUDACC__
// The resident CSR arrays the terms land in, one per matrix (A, B, C).
struct R1csCsr {
  const uint32_t* row_ptr[3];
  uint32_t* col[3];
  void* val[3];
};
// One thread per term t0 + t of a chunk.  tp: the per-constraint term prefix (tp[i] = terms of constraints < i); the
// chunk's terms belong to constraints c_lo .. c_hi, so a binary search over that range gives the term's constraint i, its
// place among that constraint's terms, its matrix (A, then B, then C) and its position in the row.  Its bytes are at
// section offset 12 i + ts tp[i] + 4 (matrix + 1) + ts (place); the chunk's copy starts at section offset `base`.  An accepted
// term is written at row_ptr[i] + position: every term has its own slot, so no atomics and the CSR is the file's order.  A
// refused one lands in *err as (file offset << 8 | code), the smallest winning.
template <class Fr>
__global__ void __launch_bounds__(256) r1cs_term_kernel(const uint8_t* chunk, uint64_t base, uint64_t sec_off, uint64_t t0,
                                                        uint32_t count, uint32_t c_lo, uint32_t c_hi, const uint64_t* tp,
                                                        uint32_t ts, uint32_t nwires, R1csCsr csr, unsigned long long* err) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= count) return;
  const uint64_t g = t0 + t;
  uint32_t lo = c_lo, hi = c_hi;   // the largest i in [lo, hi] with tp[i] <= g
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo + 1) / 2;
    if (tp[mid] <= g) lo = mid; else hi = mid - 1;
  }
  const uint32_t i = lo;
  const uint64_t within = g - tp[i];   // place among the constraint's terms
  // the matrix by constant indices only (a dynamic index into csr would put the struct in local memory)
  const uint32_t a0 = csr.row_ptr[0][i], na = csr.row_ptr[0][i + 1] - a0;
  const uint32_t b0 = csr.row_ptr[1][i], nb = csr.row_ptr[1][i + 1] - b0;
  const uint32_t m = within < na ? 0 : within < (uint64_t)na + nb ? 1 : 2;
  const uint32_t pos = m == 0 ? a0 + (uint32_t)within : m == 1 ? b0 + (uint32_t)(within - na) : csr.row_ptr[2][i] + (uint32_t)(within - na - nb);
  const uint64_t off = 12ull * i + (uint64_t)ts * tp[i] + 4ull * (m + 1) + (uint64_t)ts * within;
  uint32_t wire;
  Fr v;
  const uint32_t code = r1cs_term_decode(chunk + (off - base), nwires, wire, v);
  if (code) {
    atomicMin(err, ((sec_off + off) << 8) | code);
    return;
  }
  (m == 0 ? csr.col[0] : m == 1 ? csr.col[1] : csr.col[2])[pos] = wire;
  reinterpret_cast<Fr*>(m == 0 ? csr.val[0] : m == 1 ? csr.val[1] : csr.val[2])[pos] = v;
}
// One thread per element e0 + e of a .wtns chunk (n8 bytes each, the chunk's copy at `chunk`), written to out[e0 + e] as
// c R; a refused one lands in *err as (file offset << 8 | code).
template <class Fr>
__global__ void __launch_bounds__(256) wtns_elem_kernel(const uint8_t* chunk, uint64_t off0, uint64_t e0, uint32_t count,
                                                        Fr* out, unsigned long long* err) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= count) return;
  constexpr uint32_t NB = 4 * Fr::N;
  Fr v;
  const uint32_t code = r1cs_elem_decode(chunk + (uint64_t)e * NB, v);
  if (code) atomicMin(err, ((off0 + (uint64_t)e * NB) << 8) | code);
  else out[e0 + e] = v;
}

template <class Fr>
cudaError_t r1cs_term_enqueue(cudaStream_t st, const uint8_t* chunk, uint64_t base, uint64_t sec_off, uint64_t t0, uint32_t count,
                              uint32_t c_lo, uint32_t c_hi, const uint64_t* tp, uint32_t ts, uint32_t nwires, R1csCsr csr,
                              unsigned long long* err) {
  if (!count) return cudaSuccess;
  r1cs_term_kernel<Fr><<<(count + 255) / 256, 256, 0, st>>>(chunk, base, sec_off, t0, count, c_lo, c_hi, tp, ts, nwires, csr, err);
  return cudaGetLastError();
}
template <class Fr>
cudaError_t wtns_elem_enqueue(cudaStream_t st, const uint8_t* chunk, uint64_t off0, uint64_t e0, uint32_t count, void* out,
                              unsigned long long* err) {
  if (!count) return cudaSuccess;
  wtns_elem_kernel<Fr><<<(count + 255) / 256, 256, 0, st>>>(chunk, off0, e0, count, reinterpret_cast<Fr*>(out), err);
  return cudaGetLastError();
}
// the .r1cs / .wtns kernels of one curve (all four: circom writes any prime field)
#define G16_R1CS_TEMPLATES(X, CP)                                                                                       \
  X cudaError_t r1cs_term_enqueue<Fp<CP::FrP>>(cudaStream_t, const uint8_t*, uint64_t, uint64_t, uint64_t, uint32_t,     \
                                               uint32_t, uint32_t, const uint64_t*, uint32_t, uint32_t, R1csCsr,          \
                                               unsigned long long*);                                                     \
  X cudaError_t wtns_elem_enqueue<Fp<CP::FrP>>(cudaStream_t, const uint8_t*, uint64_t, uint64_t, uint32_t, void*,         \
                                               unsigned long long*);
#endif

// ---- the host walks ----------------------------------------------------------------------------------------------------
inline uint64_t r1_u64(const uint8_t* p) {
  uint64_t w;
  memcpy(&w, p, 8);
  return w;
}
// little-endian bytes == the limbs of P's modulus
template <class P>
bool r1_is_modulus(const uint8_t* p) {
  for (int i = 0; i < P::N; i++)
    if (r1_u32(p + 4 * i) != P::mod(i)) return false;
  return true;
}
struct BinSection {
  uint64_t off = 0, size = 0;
};
// The section table of an iden3 binary file (magic, version, nSections, {type, size, body}): the bodies of sections 1 and 2,
// each found exactly once; other types are skipped, except refuse_lo .. refuse_hi (the .r1cs custom-gate sections; 0 =
// none), which are refused.  "" or why the table is refused.
inline std::string bin_sections(const uint8_t* b, uint64_t len, const char* magic, uint32_t version, BinSection sec[3],
                                uint32_t refuse_lo = 0, uint32_t refuse_hi = 0) {
  const std::string ext = std::string(".") + magic;
  if (!b && len) return "null input";
  if (len < 12) return "truncated input: " + std::to_string(len) + " bytes, a " + ext + " header is 12";
  if (memcmp(b, magic, 4) != 0) return "not a " + ext + " file (magic is not \"" + magic + "\")";
  if (r1_u32(b + 4) != version)
    return "unsupported " + ext + " version " + std::to_string(r1_u32(b + 4)) + " (expected " + std::to_string(version) + ")";
  const uint32_t nsec = r1_u32(b + 8);
  uint64_t pos = 12;
  bool seen[3] = {};
  for (uint32_t k = 0; k < nsec; k++) {
    if (len - pos < 12)
      return "truncated input: section " + std::to_string(k) + " of " + std::to_string(nsec) + " has no complete header at byte " +
             std::to_string(pos);
    const uint32_t id = r1_u32(b + pos);
    const uint64_t size = r1_u64(b + pos + 4);
    pos += 12;
    if (size > len - pos)
      return "truncated input: section " + std::to_string(id) + " at byte " + std::to_string(pos) + " declares " +
             std::to_string(size) + " bytes, " + std::to_string(len - pos) + " remain";
    if (refuse_lo && id >= refuse_lo && id <= refuse_hi)
      return "section " + std::to_string(id) + ": custom gates are not R1CS";
    if (id == 1 || id == 2) {
      if (seen[id]) return "section " + std::to_string(id) + " appears twice";
      seen[id] = true;
      sec[id] = BinSection{pos, size};
    }
    pos += size;
  }
  if (pos != len) return "trailing bytes after the last section (" + std::to_string(len - pos) + ")";
  for (int id = 1; id <= 2; id++)
    if (!seen[id]) return "section " + std::to_string(id) + " is missing";
  return "";
}

struct R1csLayout {
  uint64_t sec2_off = 0, sec2_size = 0;   // the constraint section's body
  uint32_t n8 = 0, nwires = 0, npubout = 0, npubin = 0, nprvin = 0, m = 0;
  uint64_t nlabels = 0;
  uint32_t num_inputs = 0, num_witness = 0;
  uint32_t ts = 0;                         // bytes per term, 4 + n8
  std::vector<uint32_t> rp[3];             // row_ptr of A, B, C (m + 1 entries each)
  std::vector<uint64_t> tp;                // terms of constraints < i (m + 1 entries); tp[m] = every term
};
// section offset of term k (0-based among constraint i's terms, A then B then C) of constraint i
inline uint64_t r1cs_term_off(const R1csLayout& z, uint32_t i, uint64_t k) {
  int m = 0;
  uint64_t r = k;
  for (; m < 2; m++) {
    const uint64_t nm = z.rp[m][i + 1] - z.rp[m][i];
    if (r < nm) break;
    r -= nm;
  }
  return 12ull * i + (uint64_t)z.ts * z.tp[i] + 4ull * (m + 1) + (uint64_t)z.ts * k;
}
// Walks the section table, the header and the term counts of every constraint for the scalar field P, and builds the
// three row_ptr arrays and the term prefix.  Returns "" and fills z, or why the file is refused (the first problem found).
template <class P>
std::string r1cs_walk(const uint8_t* b, uint64_t len, R1csLayout& z) {
  constexpr uint32_t NR = 4 * P::N;
  z = R1csLayout{};
  BinSection sec[3];
  std::string why = bin_sections(b, len, "r1cs", 1, sec, 4, 5);
  if (!why.empty()) return why;
  const uint8_t* h = b + sec[1].off;
  if (sec[1].size < 4) return "section 1 (header): size " + std::to_string(sec[1].size) + ", expected " + std::to_string(32 + NR);
  z.n8 = r1_u32(h);
  if (z.n8 != NR)
    return "section 1: n8 = " + std::to_string(z.n8) + ", the context's curve has " + std::to_string(NR) + "-byte scalars";
  if (sec[1].size != 32 + NR)
    return "section 1 (header): size " + std::to_string(sec[1].size) + ", expected " + std::to_string(32 + NR);
  if (!r1_is_modulus<P>(h + 4)) return "section 1: prime is not the scalar field modulus of this curve";
  const uint8_t* f = h + 4 + NR;
  z.nwires = r1_u32(f);
  z.npubout = r1_u32(f + 4);
  z.npubin = r1_u32(f + 8);
  z.nprvin = r1_u32(f + 12);
  z.nlabels = r1_u64(f + 16);
  z.m = r1_u32(f + 24);
  const uint64_t ni = 1ull + z.npubout + z.npubin;
  if ((uint64_t)z.nwires < ni + z.nprvin)
    return "section 1: nWires = " + std::to_string(z.nwires) + " is below 1 + nPubOut + nPubIn + nPrvIn = " +
           std::to_string(ni + z.nprvin);
  z.num_inputs = (uint32_t)ni;
  z.num_witness = (uint32_t)(z.nwires - ni);
  z.ts = 4 + NR;
  z.sec2_off = sec[2].off;
  z.sec2_size = sec[2].size;
  const uint64_t S = sec[2].size;
  // every constraint takes at least its three counts: bounds what is allocated below by the file's size
  if (12ull * z.m > S)
    return "section 2 holds " + std::to_string(S) + " bytes, its " + std::to_string(z.m) + " constraints need at least " +
           std::to_string(12ull * z.m);
  for (auto& v : z.rp) v.assign((size_t)z.m + 1, 0);
  z.tp.assign((size_t)z.m + 1, 0);
  const uint8_t* s = b + sec[2].off;
  uint64_t pos = 0, nnz[3] = {0, 0, 0};
  static const char* names = "ABC";
  for (uint32_t i = 0; i < z.m; i++) {
    for (int m = 0; m < 3; m++) {
      if (S - pos < 4)
        return "section 2 holds " + std::to_string(S) + " bytes, its constraints need more: constraint " + std::to_string(i) +
               "'s " + names[m] + " term count lies past its end";
      const uint32_t n = r1_u32(s + pos);
      pos += 4;
      if ((uint64_t)n * z.ts > S - pos)
        return "section 2 holds " + std::to_string(S) + " bytes, its constraints need more: constraint " + std::to_string(i) +
               "'s " + std::to_string(n) + " " + names[m] + " terms run past its end";
      pos += (uint64_t)n * z.ts;
      nnz[m] += n;
      if (nnz[m] >= (1ull << 32))
        return std::string("matrix ") + names[m] + " holds 2^32 or more entries (row_ptr is 32-bit)";
      z.rp[m][i + 1] = (uint32_t)nnz[m];
    }
    z.tp[i + 1] = nnz[0] + nnz[1] + nnz[2];
  }
  const uint64_t need = 12ull * z.m + (uint64_t)z.ts * z.tp[z.m];
  if (need != S) return "section 2 holds " + std::to_string(S) + " bytes, its constraints need " + std::to_string(need);
  return "";
}
// why the term at file offset `off` was refused (code from r1cs_term_decode)
inline std::string r1cs_reason(const uint8_t* b, const R1csLayout& z, uint64_t off, uint32_t code) {
  const uint64_t rel = off - z.sec2_off;
  if (z.m == 0) return "byte " + std::to_string(off) + ": unknown error";
  // the constraint: the last i whose start 12 i + ts tp[i] is <= rel
  uint32_t lo = 0, hi = z.m - 1;
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo + 1) / 2;
    if (12ull * mid + (uint64_t)z.ts * z.tp[mid] <= rel) lo = mid; else hi = mid - 1;
  }
  const uint32_t i = lo;
  uint64_t k = 0;
  while (r1cs_term_off(z, i, k) != rel) k++;   // at most the constraint's terms
  int m = 0;
  for (; m < 2; m++) {
    const uint64_t nm = z.rp[m][i + 1] - z.rp[m][i];
    if (k < nm) break;
    k -= nm;
  }
  std::string s = "constraint " + std::to_string(i) + ", " + "ABC"[m] + " term " + std::to_string(k) + " (byte " +
                  std::to_string(off) + "): ";
  switch (code) {
    case R1_ERR_WIRE: return s + "wire " + std::to_string(r1_u32(b + off)) + " >= nWires " + std::to_string(z.nwires);
    case R1_ERR_VALUE: return s + "coefficient is not below r";
    default: return s + "unknown error";
  }
}

struct WtnsLayout {
  uint64_t off = 0;   // file offset of element 0
  uint32_t n = 0;     // nWitness
  uint32_t n8 = 0;
};
template <class P>
std::string wtns_walk(const uint8_t* b, uint64_t len, WtnsLayout& w) {
  constexpr uint32_t NR = 4 * P::N;
  w = WtnsLayout{};
  BinSection sec[3];
  std::string why = bin_sections(b, len, "wtns", 2, sec);
  if (!why.empty()) return why;
  const uint8_t* h = b + sec[1].off;
  if (sec[1].size < 4) return "section 1 (header): size " + std::to_string(sec[1].size) + ", expected " + std::to_string(8 + NR);
  w.n8 = r1_u32(h);
  if (w.n8 != NR)
    return "section 1: n8 = " + std::to_string(w.n8) + ", the context's curve has " + std::to_string(NR) + "-byte scalars";
  if (sec[1].size != 8 + NR)
    return "section 1 (header): size " + std::to_string(sec[1].size) + ", expected " + std::to_string(8 + NR);
  if (!r1_is_modulus<P>(h + 4)) return "section 1: prime is not the scalar field modulus of this curve";
  w.n = r1_u32(h + 4 + NR);
  w.off = sec[2].off;
  if (sec[2].size != (uint64_t)w.n * NR)
    return "section 2 holds " + std::to_string(sec[2].size) + " bytes, " + std::to_string(w.n) + " elements need " +
           std::to_string((uint64_t)w.n * NR);
  return "";
}
inline std::string wtns_reason(const WtnsLayout& w, uint64_t off, uint32_t code) {
  const uint64_t e = (off - w.off) / w.n8;
  return "witness[" + std::to_string(e) + "] (byte " + std::to_string(off) + "): " + (code == R1_ERR_VALUE ? "not below r" : "unknown error");
}

}  // namespace g16
