// ptau.cuh -- snarkjs .ptau powers-of-tau transcripts (iden3 binary container, as snarkjs `powersoftau` writes them): the
// host walk of the section table and the header, where each member and each level of Lagrange points lies, and the layout
// of the prepared file g16_ptau_prepare writes.  Nothing is decoded: the points are affine, Montgomery form and
// little-endian, which is this ABI's limb layout (as in a .zkey), so they are copied as they are and checked by whichever
// call reads them.
//
// "ptau", version u32 = 1, nSections u32, then {id u32, size u64, body} records in any order; integers little-endian.  n8 is
// the base-field byte size; a G1 point is x || y (n8 bytes each), a G2 point x.c0 || x.c1 || y.c0 || y.c1 (BW6-761: x || y
// over Fq); the identity is all-zero bytes.
//   1   header, exactly 12 + n8 bytes: n8 u32, q (n8 bytes), power u32, ceremonyPower u32
//   2   tauG1 = [tau^i]G1, 2^(power+1) - 1 points      3   tauG2 = [tau^i]G2, 2^power points
//   4   alphaTauG1, 2^power points                      5   betaTauG1, 2^power points
//   6   betaG2, one point                               7   contributions (skipped)
//   12..15  prepared files only (snarkjs `powersoftau prepare phase2`): the Lagrange points of sections 2..5.  Level k
//       holds the 2^k points (1/2^k) sum_{j<2^k} omega_k^(-ij) X_j over the first 2^k points X_j of the source section;
//       levels are concatenated from k = 0 up, so level k starts at point 2^k - 1.  Sections 13..15 hold levels 0 .. power
//       (2^(power+1) - 1 points); section 12 also holds level power + 1, formed from the 2^(power+1) - 1 points of
//       section 2 with the missing last power taken as the identity (2^(power+2) - 1 points).  The odd entries of that
//       level are the CircomReduction H query at delta = 1; those of an interior level k + 1 <= power, taken over all
//       2^(k+1) powers, are that query plus (omega_2n^(2i+1) / 2n) [tau^(2n-1)] (n = 2^k), which the key setup takes off.
// Sections 1..6 appear exactly once; 12..15 all four or none, each at most once; any other id is skipped.  The curve is
// decided by the prime: n8 and q must be the context's base field.  When power + 1 exceeds the scalar field's two-adicity
// (BN254 at power 28) level power + 1 cannot exist and what snarkjs writes in section 12 there is unconfirmed: sections
// 12..15 are then not interpreted, and the file reads as unprepared (its powers still serve).
#pragma once
#include <algorithm>
#include <string>
#include <utility>
#include <vector>
#include "r1cs.cuh"

namespace g16 {

// the members of sections 2..5, and of their Lagrange sections 12..15, in the order of g16_srs_desc
enum { PTAU_TAU_G1 = 0, PTAU_TAU_G2, PTAU_ALPHA, PTAU_BETA, PTAU_MEMBERS };
// sizes stay far inside 64 bits up to here (2^(power+2) points of at most 192 bytes)
constexpr uint32_t PTAU_MAX_POWER = 48;

struct PtauLayout {
  uint32_t n8 = 0, power = 0, ceremony_power = 0;
  bool prepared = false;                      // sections 12..15 present and interpreted
  uint32_t g1_bytes = 0, g2_bytes = 0;
  uint64_t off[PTAU_MEMBERS] = {}, len[PTAU_MEMBERS] = {};   // sections 2..5: file offset of point 0, points
  uint64_t beta_g2_off = 0;                   // section 6
  uint64_t lag_off[PTAU_MEMBERS] = {};        // sections 12..15: file offset of point 0 (prepared only)
  uint32_t bytes(int m) const { return m == PTAU_TAU_G2 ? g2_bytes : g1_bytes; }
};
// first point of level k in sections 12..15
inline uint64_t ptau_level_start(uint32_t k) { return (1ull << k) - 1; }

// The first part of ptau_walk: the section table and section 1 alone.  Fills sec (ids 1..15), z.n8, z.power and
// z.ceremony_power; no other section's size is compared yet.
template <class CP>
std::string ptau_walk_header(const uint8_t* b, uint64_t len, PtauLayout& z, BinSection* sec) {
  using FqP = typename CP::FqP;
  constexpr uint32_t N8 = 4 * FqP::N;
  z = PtauLayout{};
  const uint64_t need = bin_id(1) | bin_id(2) | bin_id(3) | bin_id(4) | bin_id(5) | bin_id(6);
  const uint64_t lag = bin_id(12) | bin_id(13) | bin_id(14) | bin_id(15);
  std::string why = bin_sections(b, len, "ptau", 1, need | lag, need, sec);
  if (!why.empty()) return why;
  const uint8_t* h = b + sec[1].off;
  const std::string hsize = "section 1 (header): size " + std::to_string(sec[1].size) + ", expected " + std::to_string(12 + N8);
  if (sec[1].size < 4) return hsize;
  z.n8 = r1_u32(h);
  if (z.n8 != N8)
    return "section 1: n8 = " + std::to_string(z.n8) + ", the context's curve has " + std::to_string(N8) + "-byte base field elements";
  if (sec[1].size != 12 + N8) return hsize;
  if (!r1_is_modulus<FqP>(h + 4)) return "section 1: q is not the base field modulus of this curve";
  z.power = r1_u32(h + 4 + N8);
  z.ceremony_power = r1_u32(h + 8 + N8);
  if (z.power > PTAU_MAX_POWER)
    return "section 1: power " + std::to_string(z.power) + " is above " + std::to_string(PTAU_MAX_POWER);
  return "";
}
// Walks the section table and the header for the curve CP.  Returns "" and fills z, or why the file is refused (the first
// problem found).
template <class CP>
std::string ptau_walk(const uint8_t* b, uint64_t len, PtauLayout& z) {
  constexpr uint32_t N8 = 4 * CP::FqP::N;
  BinSection sec[16];
  std::string why = ptau_walk_header<CP>(b, len, z, sec);
  if (!why.empty()) return why;
  z.g1_bytes = 2 * N8;
  z.g2_bytes = (uint32_t)sizeof(Affine<typename CP::G2F>);
  const uint64_t np = 1ull << z.power;
  auto sized = [&](uint32_t id, uint64_t pts, uint32_t bytes, const char* what) -> std::string {
    if (sec[id].size == pts * bytes) return "";
    return "section " + std::to_string(id) + " holds " + std::to_string(sec[id].size) + " bytes, " + what + " " +
           std::to_string(pts * bytes);
  };
  const uint64_t pts[PTAU_MEMBERS] = {2 * np - 1, np, np, np};
  for (int m = 0; m < PTAU_MEMBERS; m++) {
    if (!(why = sized(2 + m, pts[m], z.bytes(m), m == PTAU_TAU_G1 ? "2^(power+1) - 1 points need" : "2^power points need")).empty())
      return why;
    z.off[m] = sec[2 + m].off;
    z.len[m] = pts[m];
  }
  if (!(why = sized(6, 1, z.g2_bytes, "one G2 point needs")).empty()) return why;
  z.beta_g2_off = sec[6].off;
  std::string present;
  int nlag = 0;
  for (uint32_t id = 12; id <= 15; id++)
    if (sec[id].found) { present += (nlag++ ? ", " : "") + std::to_string(id); }
  if (nlag != 0 && nlag != PTAU_MEMBERS)
    return "sections 12-15 (Lagrange points) appear all four or none: only " + present + " present";
  if (nlag == 0 || z.power + 1 > (uint32_t)CP::FrP::TWO_ADICITY) return "";
  for (int m = 0; m < PTAU_MEMBERS; m++) {
    const bool h1 = m == PTAU_TAU_G1;
    if (!(why = sized(12 + m, h1 ? 4 * np - 1 : 2 * np - 1, z.bytes(m), h1 ? "2^(power+2) - 1 points need" : "2^(power+1) - 1 points need")).empty())
      return why;
    z.lag_off[m] = sec[12 + m].off;
  }
  z.prepared = true;
  return "";
}

// ---- prepared files (g16_ptau_prepare) ----------------------------------------------------------------------------------
// The top level of member m: power + 1 for tauG1, power for the others.
inline uint32_t ptau_top_level(int m, uint32_t power) { return power + (m == PTAU_TAU_G1); }
// Levels 1 .. PTAU_SMALL_LEVELS of a member are transformed concurrently, each on its own stream and in its own slice of
// the work buffers (level k at point 2^k - 1): together they hold 2^PTAU_SMALL_LEVELS - 1 butterflies, fewer than one wave
// of the stage kernel on an H100 for either group.  The larger levels reuse the start of the buffers one at a time.
constexpr uint32_t PTAU_SMALL_LEVELS = 14;
// Points of each work buffer (XYZZ and affine staging) for a member whose top level is `top`.  Saturates far above any
// device's memory (ptau_top_level <= PTAU_MAX_POWER + 1).
inline uint64_t ptau_work_points(uint32_t top) {
  return std::max<uint64_t>(1ull << top, ptau_level_start(std::min(top, PTAU_SMALL_LEVELS) + 1));
}
// The file g16_ptau_prepare writes: "ptau", version 1, nSections; the kept sections (every section of the input but
// 12..15, byte for byte in input order: `kept` of them, `kept_bytes` with their 12-byte heads); then sections 12, 13, 14
// and 15, each holding levels 0 .. ptau_top_level of its member.
struct PtauPrepared {
  uint32_t nsec = 0;
  uint64_t size = 0;
  uint64_t lag_off[PTAU_MEMBERS] = {};   // body offset of sections 12..15
  uint64_t lag_pts[PTAU_MEMBERS] = {};   // their points: 2^(top + 1) - 1
};
inline PtauPrepared ptau_prepared_layout(uint32_t kept, uint64_t kept_bytes, uint32_t power, uint32_t g1_bytes, uint32_t g2_bytes) {
  PtauPrepared p;
  p.nsec = kept + PTAU_MEMBERS;
  uint64_t pos = 12 + kept_bytes;
  for (int m = 0; m < PTAU_MEMBERS; m++) {
    p.lag_pts[m] = (2ull << ptau_top_level(m, power)) - 1;
    p.lag_off[m] = pos + 12;
    pos += 12 + p.lag_pts[m] * (m == PTAU_TAU_G2 ? g2_bytes : g1_bytes);
  }
  p.size = pos;
  return p;
}
// The kept sections of a file ptau_walk accepted: {offset of the section's head, its bytes with the head}, in file order.
inline std::vector<std::pair<uint64_t, uint64_t>> ptau_kept_sections(const uint8_t* b) {
  std::vector<std::pair<uint64_t, uint64_t>> out;
  const uint32_t nsec = r1_u32(b + 8);
  uint64_t pos = 12;
  for (uint32_t k = 0; k < nsec; k++) {
    const uint32_t id = r1_u32(b + pos);
    const uint64_t rec = 12 + r1_u64(b + pos + 4);
    if (id < 12 || id > 15) out.push_back({pos, rec});
    pos += rec;
  }
  return out;
}

}  // namespace g16
