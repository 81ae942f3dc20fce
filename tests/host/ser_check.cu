// Host-only check (built by nvcc, runs without a GPU) of the proving-key wire format code of groth16_b200/csrc/ser.cuh:
//   1. the chunk planner and the placement rule: for chunk sizes 1, 2, 7, 1000, odd vector lengths and world 1 .. 3, every
//      point is visited once, at its byte offset, and every MSM pair has exactly one owner, in the slot g16_pk_load uses;
//   2. ser_decode / ser_encode, the per-point functions the kernels run, on cases read from stdin (tests/test_ser_host.py
//      writes them and compares the answers with groth16_b200.serialize.ArkCodec):
//        D <curve> <g2> <flags> <hex bytes>                 ->  "ERR <code>" | "INF" | "PT <hex canonical coordinates>"
//        E <curve> <g2> <flags> INF | <hex coordinates>     ->  "BYTES <hex>"
//      curve: 0 BLS12-381, 1 BN254, 2 BLS12-377; coordinates x y (G1) or x0 x1 y0 y1 (G2).
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>
#include "../../groth16_b200/csrc/ser.cuh"
using namespace g16;

static int bad = 0, cases = 0;
#define CHECK(cond, ...)            \
  do {                              \
    cases++;                        \
    if (!(cond)) {                  \
      bad++;                        \
      fprintf(stderr, __VA_ARGS__); \
      fprintf(stderr, "\n");        \
    }                               \
  } while (0)

static void check_planner() {
  const uint64_t lens[][5] = {{3, 5, 5, 7, 2}, {1, 1, 1, 1, 0}, {9, 1001, 1001, 1999, 17}, {0, 2, 2, 2, 0}};
  for (auto& L : lens)
    for (int nb : {32, 48})
      for (bool compress : {true, false}) {
        // build the stream skeleton with these lengths: gamma_abc = L[0], a = b1 = b2 = L[1..3]... and h, l
        SerItem it[SER_ITEMS];
        ser_items(it);
        it[SER_GAMMA_ABC].len = L[0];
        it[SER_A].len = L[1]; it[SER_B_G1].len = L[1]; it[SER_B_G2].len = L[2];
        it[SER_H].len = L[3]; it[SER_L].len = L[4];
        const uint64_t total = ser_size(it, nb, compress);
        std::vector<uint8_t> bytes(total, 0);
        for (int m = 0; m < SER_ITEMS; m++)
          if (it[m].vec)
            for (int k = 0; k < 8; k++) bytes[it[m].off - 8 + k] = (uint8_t)(it[m].len >> (8 * k));
        SerItem w[SER_ITEMS];
        CHECK(ser_walk(bytes.data(), total, nb, compress, w).empty(), "walk rejected a well-formed skeleton");
        for (int m = 0; m < SER_ITEMS; m++)
          CHECK(w[m].len == it[m].len && w[m].off == it[m].off && w[m].psize == it[m].psize, "walk: member %d", m);
        CHECK(!ser_walk(bytes.data(), total - 1, nb, compress, w).empty(), "walk accepted a truncated stream");
        std::vector<uint8_t> more(bytes);
        more.push_back(0);
        CHECK(ser_walk(more.data(), total + 1, nb, compress, w) == "trailing bytes after the proving key", "trailing bytes");
        for (uint32_t chunk : {1u, 2u, 7u, 1000u}) {
          const std::vector<SerChunk> plan = ser_plan(it, chunk);
          std::vector<std::vector<int>> seen(SER_ITEMS);
          for (int m = 0; m < SER_ITEMS; m++) seen[m].assign(it[m].len, 0);
          for (const SerChunk& c : plan) {
            CHECK(c.count >= 1 && c.count <= chunk, "chunk size");
            for (uint32_t t = 0; t < c.count; t++) {
              const uint64_t i = c.first + t;
              CHECK(i < it[c.member].len, "index past the member");
              if (i >= it[c.member].len) continue;
              seen[c.member][i]++;
              CHECK(c.off + (uint64_t)t * it[c.member].psize == it[c.member].off + i * it[c.member].psize, "offset");
              CHECK(ser_locate(it, c.off + (uint64_t)t * it[c.member].psize) ==
                        std::string(it[c.member].name) + "[" + std::to_string(i) + "]", "locate");
            }
          }
          for (int m = 0; m < SER_ITEMS; m++)
            for (uint64_t i = 0; i < it[m].len; i++) CHECK(seen[m][i] == 1, "member %d point %llu visited %d times", m, (unsigned long long)i, seen[m][i]);
          // ownership: a / b queries skip element 0; pairs truncated to a circuit one shorter than the key
          for (int m : {(int)SER_A, (int)SER_B_G2, (int)SER_H, (int)SER_L})
            for (uint32_t world = 1; world <= 3; world++) {
              const uint64_t skip = (m == SER_A || m == SER_B_G2) ? 1 : 0;
              const uint64_t pairs = it[m].len > skip ? it[m].len - skip - (it[m].len - skip > 1 ? 1 : 0) : 0;
              std::vector<int> owners(pairs, 0);
              for (uint32_t rank = 0; rank < world; rank++) {
                const uint64_t cnt = pairs > rank ? (pairs - rank + world - 1) / world : 0;   // Engine::shard
                std::vector<int> slot_used(cnt, 0);
                for (const SerChunk& c : plan) {
                  if (c.member != m) continue;
                  for (uint32_t t = 0; t < c.count; t++) {
                    const uint64_t i = c.first + t;
                    const int64_t s = ser_slot(i, skip, pairs, rank, world);
                    if (s < 0) continue;
                    const uint64_t j = i - skip;
                    CHECK(j < pairs && j % world == rank && (uint64_t)s == (j - rank) / world && (uint64_t)s < cnt,
                          "slot of member %d point %llu rank %u world %u", m, (unsigned long long)i, rank, world);
                    if (j < pairs) owners[j]++;
                    if ((uint64_t)s < cnt) slot_used[s]++;
                  }
                }
                for (uint64_t s = 0; s < cnt; s++) CHECK(slot_used[s] == 1, "slot %llu filled %d times", (unsigned long long)s, slot_used[s]);
              }
              for (uint64_t j = 0; j < pairs; j++) CHECK(owners[j] == 1, "pair %llu has %d owners", (unsigned long long)j, owners[j]);
            }
        }
      }
  // an absurd prefix is refused before anything is sized from it
  std::vector<uint8_t> b(4096, 0);
  SerItem w[SER_ITEMS];
  const uint64_t at = 48 + 3 * 96;   // gamma_abc_g1's prefix, compressed 48-byte field
  b[at + 7] = 0x01;
  CHECK(ser_walk(b.data(), b.size(), 48, true, w).find("exceeds the limit") != std::string::npos, "absurd prefix");
}

// ---- per-point functions --------------------------------------------------------------------------------------------
template <class P>
static Fp<P> parse_fq(const std::string& hex) {
  Fp<P> r = Fp<P>::zero();
  int bit = 0;
  for (int k = (int)hex.size() - 1; k >= 0; k--, bit += 4) {
    const char ch = hex[k];
    const uint32_t d = ch <= '9' ? ch - '0' : (ch | 0x20) - 'a' + 10;
    if (bit < 32 * P::N) r.v[bit / 32] |= d << (bit % 32);
  }
  return r;
}
template <class P>
static std::string hex_fq(const Fp<P>& a) {
  std::string s;
  char buf[16];
  for (int i = P::N - 1; i >= 0; i--) { snprintf(buf, sizeof buf, "%08x", a.v[i]); s += buf; }
  return s;
}
static std::vector<uint8_t> parse_bytes(const std::string& hex) {
  std::vector<uint8_t> out(hex.size() / 2);
  for (size_t i = 0; i < out.size(); i++) out[i] = (uint8_t)std::stoul(hex.substr(2 * i, 2), nullptr, 16);
  return out;
}

template <class CP, bool G2>
static std::string run(char op, uint32_t flags, std::istringstream& in) {
  using P = typename CP::FqP;
  using Fq = Fp<P>;
  using A = Affine<SerField<CP, G2>>;
  constexpr int NC = G2 ? 2 : 1;
  if (op == 'D') {
    std::string hex;
    in >> hex;
    const std::vector<uint8_t> raw = parse_bytes(hex);
    if ((int)raw.size() != SerFormat<CP>::point_bytes(G2, flags & SER_COMPRESSED)) return "BADLEN";
    A p;
    const uint32_t code = ser_decode<CP, G2>(raw.data(), flags, p);
    if (code) return "ERR " + std::to_string(code);
    if (p.is_inf()) return "INF";
    Fq c[4];
    if constexpr (G2) { c[0] = p.x.c0; c[1] = p.x.c1; c[2] = p.y.c0; c[3] = p.y.c1; }
    else { c[0] = p.x; c[1] = p.y; }
    std::string s = "PT";
    for (int k = 0; k < 2 * NC; k++) s += " " + hex_fq(Fq::from_mont(c[k]));
    return s;
  }
  std::string first;
  in >> first;
  A p = A::inf();
  if (first != "INF") {
    Fq c[4];
    c[0] = Fq::to_mont(parse_fq<P>(first));
    for (int k = 1; k < 2 * NC; k++) { std::string h; in >> h; c[k] = Fq::to_mont(parse_fq<P>(h)); }
    if constexpr (G2) p = A{{c[0], c[1]}, {c[2], c[3]}};
    else p = A{c[0], c[1]};
  }
  std::vector<uint8_t> out(SerFormat<CP>::point_bytes(G2, flags & SER_COMPRESSED), 0xAA);
  ser_encode<CP, G2>(p, flags, out.data());
  std::string s = "BYTES ";
  char buf[4];
  for (uint8_t b : out) { snprintf(buf, sizeof buf, "%02x", b); s += buf; }
  return s;
}

template <class CP>
static std::string run_curve(char op, bool g2, uint32_t flags, std::istringstream& in) {
  return g2 ? run<CP, true>(op, flags, in) : run<CP, false>(op, flags, in);
}

int main() {
  check_planner();
  printf("planner: %d checks, %d mismatches\n", cases, bad);
  std::string line;
  int points = 0;
  while (std::getline(std::cin, line)) {
    if (line.empty()) continue;
    std::istringstream in(line);
    char op;
    int curve, g2;
    uint32_t flags;
    in >> op >> curve >> g2 >> flags;
    std::string r;
    switch (curve) {
      case 0: r = run_curve<BLS381_Params>(op, g2, flags, in); break;
      case 1: r = run_curve<BN254_Params>(op, g2, flags, in); break;
      default: r = run_curve<BLS377_Params>(op, g2, flags, in); break;
    }
    printf("%s\n", r.c_str());
    points++;
  }
  fprintf(stderr, "%d point cases\n", points);
  return bad ? 1 : 0;
}
