// Host-only driver (built by nvcc, runs without a GPU) of the .r1cs / .wtns code of groth16_b200/csrc/r1cs.cuh, for
// tests/test_r1cs_host.py, which compares every answer with tests/r1cs_ref.py.  One request per line on stdin, one answer
// per line on stdout:
//   walk <curve> <path>                 -> "ok ni nw m ts | rpA | rpB | rpC | tp" (space-separated) or "err <message>"
//   term <curve> <nwires> <hex term>    -> "<code> <wire> <hex of c R, little-endian>"
//   elem <curve> <hex element>          -> "<code> <hex of c R>"
//   wtns <curve> <path>                 -> "ok n off" or "err <message>"
// <curve> is bn254, bls12_381, bls12_377 or bw6_761.
#include <cstdio>
#include <fstream>
#include <iostream>
#include <iterator>
#include <sstream>
#include <string>
#include <vector>
#include "../../groth16_b200/csrc/r1cs.cuh"
using namespace g16;

static std::vector<uint8_t> unhex(const std::string& h) {
  std::vector<uint8_t> out(h.size() / 2);
  for (size_t i = 0; i < out.size(); i++) out[i] = (uint8_t)std::stoul(h.substr(2 * i, 2), nullptr, 16);
  return out;
}
static std::string hex(const void* p, size_t n) {
  static const char* d = "0123456789abcdef";
  std::string s;
  for (size_t i = 0; i < n; i++) {
    const uint8_t b = static_cast<const uint8_t*>(p)[i];
    s += d[b >> 4];
    s += d[b & 15];
  }
  return s;
}
static std::vector<uint8_t> slurp(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  return std::vector<uint8_t>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}
template <class V>
static std::string join(const V& v) {
  std::string s;
  for (auto x : v) s += " " + std::to_string(x);
  return s;
}

template <class CP>
static std::string run(const std::string& op, std::istringstream& in) {
  using P = typename CP::FrP;
  if (op == "walk") {
    std::string path;
    in >> path;
    const std::vector<uint8_t> b = slurp(path);
    R1csLayout z;
    const std::string why = r1cs_walk<P>(b.data(), b.size(), z);
    if (!why.empty()) return "err " + why;
    return "ok " + std::to_string(z.num_inputs) + " " + std::to_string(z.num_witness) + " " + std::to_string(z.m) + " " +
           std::to_string(z.ts) + " |" + join(z.rp[0]) + " |" + join(z.rp[1]) + " |" + join(z.rp[2]) + " |" + join(z.tp);
  }
  if (op == "term") {
    uint32_t nw;
    std::string h;
    in >> nw >> h;
    const std::vector<uint8_t> t = unhex(h);
    uint32_t wire = 0;
    Fp<P> v = Fp<P>::zero();
    const uint32_t code = r1cs_term_decode(t.data(), nw, wire, v);
    return std::to_string(code) + " " + std::to_string(wire) + " " + hex(v.v, sizeof(v.v));
  }
  if (op == "elem") {
    std::string h;
    in >> h;
    const std::vector<uint8_t> t = unhex(h);
    Fp<P> v = Fp<P>::zero();
    const uint32_t code = r1cs_elem_decode(t.data(), v);
    return std::to_string(code) + " " + hex(v.v, sizeof(v.v));
  }
  if (op == "wtns") {
    std::string path;
    in >> path;
    const std::vector<uint8_t> b = slurp(path);
    WtnsLayout w;
    const std::string why = wtns_walk<P>(b.data(), b.size(), w);
    if (!why.empty()) return "err " + why;
    return "ok " + std::to_string(w.n) + " " + std::to_string(w.off);
  }
  return "err unknown request";
}

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op, curve;
    in >> op >> curve;
    std::string out;
    if (curve == "bn254") out = run<BN254_Params>(op, in);
    else if (curve == "bls12_381") out = run<BLS381_Params>(op, in);
    else if (curve == "bls12_377") out = run<BLS377_Params>(op, in);
    else out = run<BW6_Params>(op, in);
    std::cout << out << "\n" << std::flush;
  }
  return 0;
}
