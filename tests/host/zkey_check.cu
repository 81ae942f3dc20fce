// Host-only driver (built by nvcc, runs without a GPU) of the .zkey code of groth16_b200/csrc/zkey.cuh and the Montgomery
// little-endian point decode of ser.cuh, for tests/test_zkey_host.py, which compares every answer with tests/zkey_ref.py.
// One request per line on stdin, one answer per line on stdout:
//   walk <curve> <path>                   -> "ok nvars npub domain_size ncoefs coef_off" or "err <message>"
//   coef <curve> <domain_size> <nvars> <hex record>  -> "<code> <hex of c R, little-endian>"
//   point <curve> <g2> <validate> <hex>   -> "<code> <hex of the decoded affine limbs>"
// <curve> is bn254 or bls12_381.
#include <cstdio>
#include <fstream>
#include <iostream>
#include <iterator>
#include <sstream>
#include <string>
#include <vector>
#include "../../groth16_b200/csrc/zkey.cuh"
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

template <class CP>
static std::string run(const std::string& op, std::istringstream& in) {
  if (op == "walk") {
    std::string path;
    in >> path;
    std::ifstream f(path, std::ios::binary);
    std::vector<uint8_t> b((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    ZkeyLayout z;
    const std::string why = zkey_walk<CP>(b.data(), b.size(), z);
    if (!why.empty()) return "err " + why;
    return "ok " + std::to_string(z.nvars) + " " + std::to_string(z.npub) + " " + std::to_string(z.domain_size) + " " +
           std::to_string(z.ncoefs) + " " + std::to_string(z.coef_off);
  }
  if (op == "coef") {
    uint32_t ds, nv;
    std::string h;
    in >> ds >> nv >> h;
    const std::vector<uint8_t> rec = unhex(h);
    ZkeyCoef c;
    Fp<typename CP::FrP> v = Fp<typename CP::FrP>::zero();
    const uint32_t code = zkey_coef_decode(rec.data(), ds, nv, c, v);
    return std::to_string(code) + " " + hex(v.v, sizeof(v.v));
  }
  if (op == "point") {
    int g2, validate;
    std::string h;
    in >> g2 >> validate >> h;
    const std::vector<uint8_t> raw = unhex(h);
    const uint32_t fl = validate ? SER_VALIDATE : 0;
    if (g2) {
      Affine<SerField<CP, true>> p{};
      const uint32_t code = ser_decode_mont<CP, true>(raw.data(), fl, p);
      return std::to_string(code) + " " + hex(&p, sizeof(p));
    }
    Affine<SerField<CP, false>> p{};
    const uint32_t code = ser_decode_mont<CP, false>(raw.data(), fl, p);
    return std::to_string(code) + " " + hex(&p, sizeof(p));
  }
  return "err unknown request";
}

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op, curve;
    in >> op >> curve;
    const std::string out = curve == "bn254" ? run<BN254_Params>(op, in) : run<BLS381_Params>(op, in);
    std::cout << out << "\n" << std::flush;
  }
  return 0;
}
