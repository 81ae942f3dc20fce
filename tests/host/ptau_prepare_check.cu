// Host-only driver (built by nvcc, runs without a GPU) of what g16_ptau_prepare decides on the host and of the lane map of
// its transform, for tests/test_ptau_prepare_host.py.  Every function called is the one the library calls (ptau.cuh,
// srs.cuh).  One request per line on stdin, one answer per line on stdout:
//   file <curve> <path>                      -> "ok size nsec | lag_off x4 | lag_pts x4 | kept record offsets" or
//                                               "err <message>" (the walk's refusal)
//   header <curve> <power> <kept> <bytes>    -> "size nsec | lag_off x4 | lag_pts x4" for `kept` kept sections of `bytes`
//   map <max_log_n>                          -> "map: <checks> checks, <bad> mismatches": for every n = 2^log_n up to
//       2^max_log_n and every stage, srs_butterfly_at covers each butterfly of the stage exactly once (each point once),
//       joins points h apart with twiddle k = i0 mod h, srs_twiddle_exp(k) = k N / 2h, and the 32 lanes of every warp
//       share one twiddle wherever the stage has at least 32 butterflies per twiddle (else each twiddle is shared by
//       all n / 2h lanes of its group); srs_bitrev is the bit reversal.
//   recode <curve> <max_log_n>               -> "recode: <checks> checks, <bad> mismatches": every twiddle of every domain
//       2^log_n <= 2^max_log_n, formed by srs_twiddle as the stage kernel forms it, recoded by srs_recode_w4 into signed
//       4-bit digits in [-7, 8] that reconstruct it (sum d_i 16^i, in big-integer arithmetic here).
// <curve> is bn254, bls12_381, bls12_377 or bw6_761.
#include <fstream>
#include <iostream>
#include <iterator>
#include <set>
#include <sstream>
#include <string>
#include <vector>
#include "../../groth16_b200/csrc/ptau.cuh"
#include "../../groth16_b200/csrc/ntt.cuh"
#include "../../groth16_b200/csrc/srs.cuh"
using namespace g16;

static std::string layout_line(const PtauPrepared& p) {
  std::string s = std::to_string(p.size) + " " + std::to_string(p.nsec) + " |";
  for (uint64_t v : p.lag_off) s += " " + std::to_string(v);
  s += " |";
  for (uint64_t v : p.lag_pts) s += " " + std::to_string(v);
  return s;
}

template <class CP>
static std::string file(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  const std::vector<uint8_t> b((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  PtauLayout z;
  const std::string why = ptau_walk<CP>(b.data(), b.size(), z);
  if (!why.empty()) return "err " + why;
  const auto kept = ptau_kept_sections(b.data());
  uint64_t bytes = 0;
  for (const auto& k : kept) bytes += k.second;
  std::string s = "ok " + layout_line(ptau_prepared_layout((uint32_t)kept.size(), bytes, z.power, z.g1_bytes, z.g2_bytes)) + " |";
  for (const auto& k : kept) s += " " + std::to_string(k.first);
  return s;
}

template <class CP>
static std::string header(uint32_t power, uint32_t kept, uint64_t bytes) {
  const uint32_t g1 = 8 * CP::FqP::N, g2 = (uint32_t)sizeof(Affine<typename CP::G2F>);
  return layout_line(ptau_prepared_layout(kept, bytes, power, g1, g2));
}

static std::string map(int max_log_n) {
  uint64_t checks = 0, bad = 0;
  auto expect = [&](bool c) { checks++; bad += !c; };
  for (int log_n = 1; log_n <= max_log_n; log_n++) {
    const uint32_t n = 1u << log_n;
    for (uint32_t i = 0; i < n; i++) {
      uint32_t r = 0;
      for (int b = 0; b < log_n; b++) r |= ((i >> b) & 1u) << (log_n - 1 - b);
      expect(srs_bitrev(i, log_n) == r);
    }
    const int tab_log = log_n + 1;   // any table of a larger domain serves
    for (int log_h = 0; log_h < log_n; log_h++) {
      const uint32_t h = 1u << log_h, groups = n / (2 * h);
      std::vector<uint8_t> seen(n, 0);
      std::vector<uint32_t> tw(n / 2);
      for (uint32_t t = 0; t < n / 2; t++) {
        uint32_t k, i0;
        srs_butterfly_at(t, log_n, log_h, k, i0);
        const uint32_t i1 = i0 + h;
        expect(i1 < n && (i0 & h) == 0 && k == (i0 & (h - 1)));
        if (i1 < n) { seen[i0]++; seen[i1]++; }
        expect(srs_twiddle_exp(k, log_h, tab_log) == (uint64_t)k * ((1ull << tab_log) / (2 * h)));
        tw[t] = k;
      }
      for (uint32_t i = 0; i < n; i++) expect(seen[i] == 1);
      for (uint32_t w = 0; w < n / 2; w += 32) {   // one warp: lanes t = w .. w + 31
        std::set<uint32_t> ks;
        const uint32_t lanes = std::min<uint32_t>(32, n / 2 - w);
        for (uint32_t l = 0; l < lanes; l++) ks.insert(tw[w + l]);
        expect(ks.size() == (groups >= 32 ? 1u : (lanes + groups - 1) / groups));
      }
    }
  }
  return "map: " + std::to_string(checks) + " checks, " + std::to_string(bad) + " mismatches";
}

template <class CP>
static std::string recode(int max_log_n) {
  using Fr = Fp<typename CP::FrP>;
  constexpr int NL = Fr::N;
  uint64_t checks = 0, bad = 0;
  for (int log_n = 1; log_n <= max_log_n; log_n++) {
    Fr tab[64];
    tab[0] = Fr::inv(fr_domain_root<Fr>(log_n));
    for (int b = 1; b < 64; b++) tab[b] = Fr::sqr(tab[b - 1]);
    for (int log_h = 0; log_h < log_n; log_h++)
      for (uint32_t k = 1; k < (1u << log_h); k++) {
        const Fr w = srs_twiddle(tab, srs_twiddle_exp(k, log_h, log_n));
        int8_t d[8 * NL + 1];
        const int nd = srs_recode_w4(w.v, NL, d);
        int64_t acc[NL + 1] = {};   // sum d_i 16^i by Horner, in signed 32-bit limbs with carries
        bool range = nd == 8 * NL + 1;
        for (int i = nd - 1; i >= 0; i--) {
          range &= d[i] >= -7 && d[i] <= 8;
          int64_t c = d[i];
          for (int l = 0; l <= NL; l++) {
            const int64_t v = acc[l] * 16 + c;
            acc[l] = v & 0xffffffffll;
            c = v >> 32;   // arithmetic shift: floor division
          }
        }
        bool same = range;
        for (int l = 0; l < NL; l++) same &= (uint32_t)acc[l] == w.v[l];
        same &= acc[NL] == 0;
        checks++;
        bad += !same;
      }
  }
  return "recode: " + std::to_string(checks) + " checks, " + std::to_string(bad) + " mismatches";
}

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op, curve;
    in >> op;
    std::string out;
    if (op == "recode") {
      int m;
      in >> curve >> m;
      if (curve == "bn254") out = recode<BN254_Params>(m);
      else if (curve == "bls12_381") out = recode<BLS381_Params>(m);
      else if (curve == "bls12_377") out = recode<BLS377_Params>(m);
      else out = recode<BW6_Params>(m);
    } else if (op == "map") {
      int m;
      in >> m;
      out = map(m);
    } else if (op == "file") {
      std::string path;
      in >> curve >> path;
      if (curve == "bn254") out = file<BN254_Params>(path);
      else if (curve == "bls12_381") out = file<BLS381_Params>(path);
      else if (curve == "bls12_377") out = file<BLS377_Params>(path);
      else out = file<BW6_Params>(path);
    } else {
      uint32_t power, kept;
      uint64_t bytes;
      in >> curve >> power >> kept >> bytes;
      if (curve == "bn254") out = header<BN254_Params>(power, kept, bytes);
      else if (curve == "bls12_381") out = header<BLS381_Params>(power, kept, bytes);
      else if (curve == "bls12_377") out = header<BLS377_Params>(power, kept, bytes);
      else out = header<BW6_Params>(power, kept, bytes);
    }
    std::cout << out << "\n" << std::flush;
  }
  return 0;
}
