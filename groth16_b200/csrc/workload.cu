// workload.cu -- host-side generator of the synthetic R1CS that bench.py and the full-size tests prove (SURVEY.md section
// 8d: "do not use DummyCircuit as the only workload").  No GPU involved; it lives in the library only because the
// Python loop it replaces needs a minute at 2^24 constraints and the oracle (test infrastructure) must not be imported
// by the product path.  Nothing in the reference corresponds to it: arkworks users bring their own circuits.
//
// Constraint i (i < nc = 2^log_n - 2):  (z_p + k_i) * z_q = z_new,  p, q uniform over the variables that exist when the
// constraint is written, k_i a 124-bit constant, two uniformly random seed witnesses.  The last product is the single public
// input, so that num_constraints + num_instance_variables == 2^log_n exactly (the sizing trick of benches/bench.rs:19-20).
// Satisfiable by construction; a, b queries dense; witness values uniform-looking in [0, r).
#include <cstring>
#include <string>
#include <vector>
#include "../../include/g16b200.h"
#include "fp.cuh"

// The same file also builds, with a plain host compiler, as the stand-alone groth16_b200/libg16workload.so
// (-DG16_WORKLOAD_STANDALONE; Makefile): bench.py's `--impl reference` arm and anything else that only needs a circuit can then
// generate it without loading the CUDA library at all.
namespace g16 {
#ifdef G16_WORKLOAD_STANDALONE
static thread_local std::string g_workload_err;
static int fail(int code, const std::string& msg) { g_workload_err = msg; return code; }
#else
int fail(int code, const std::string& msg);
#endif

static inline uint64_t splitmix(uint64_t& s) {
  s += 0x9E3779B97F4A7C15ull;
  uint64_t z = s;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

template <class FrP>
static int synth(uint32_t log_n, uint64_t seed, uint32_t* a_col, uint64_t* a_val, uint32_t* b_col, uint32_t* c_col, uint64_t* z_out) {
  using Fr = Fp<FrP>;
  constexpr int W = Fr::N / 2;   // u64 limbs per Fr
  const uint64_t nc = (1ull << log_n) - 2;
  const uint32_t ninst = 2;
  uint64_t st = seed * 0x2545F4914F6CDD1Dull + 0x1234567ull;
  auto rand_fr = [&]() {   // uniform below 2^(BITS-1) < r: plenty for a workload
    Fr x;
    for (int i = 0; i < Fr::N; i += 2) { const uint64_t w = splitmix(st); x.v[i] = (uint32_t)w; x.v[i + 1] = (uint32_t)(w >> 32); }
    const int top = FrP::BITS - 1 - 32 * (Fr::N - 1);   // bits kept in the top limb
    x.v[Fr::N - 1] &= (top >= 32) ? 0xffffffffu : ((1u << top) - 1);
    return Fr::to_mont(x);
  };
  std::vector<Fr> vals(nc + 2);
  std::vector<uint32_t> cols(nc + 2);
  vals[0] = rand_fr();
  vals[1] = rand_fr();
  cols[0] = ninst;
  cols[1] = ninst + 1;
  const Fr one = Fr::one();
  uint32_t n_w = 2;
  for (uint64_t i = 0; i < nc; i++) {
    const uint64_t avail = i + 2;
    const uint64_t p = splitmix(st) % avail, q = splitmix(st) % avail;
    Fr k = Fr::zero();
    const uint64_t lo = splitmix(st) & ((1ull << 62) - 1), hi = splitmix(st) & ((1ull << 62) - 1);
    k.v[0] = (uint32_t)lo; k.v[1] = (uint32_t)(lo >> 32) | (uint32_t)(hi << 30); k.v[2] = (uint32_t)(hi >> 2); k.v[3] = (uint32_t)(hi >> 34);
    const Fr km = Fr::to_mont(k);
    vals[i + 2] = Fr::mul(Fr::add(vals[p], km), vals[q]);
    cols[i + 2] = (i == nc - 1) ? 1u : ninst + n_w++;
    a_col[2 * i] = cols[p];
    a_col[2 * i + 1] = 0;   // the constant One carries k_i
    memcpy(a_val + 2 * W * i, one.v, sizeof(Fr));
    memcpy(a_val + 2 * W * i + W, km.v, sizeof(Fr));
    b_col[i] = cols[q];
    c_col[i] = cols[i + 2];
  }
  // full assignment: One, the public input, then the witnesses in column order
  memcpy(z_out, one.v, sizeof(Fr));
  for (uint64_t j = 0; j < nc + 2; j++) memcpy(z_out + W * (uint64_t)cols[j], vals[j].v, sizeof(Fr));
  return G16_OK;
}
}  // namespace g16

#ifdef G16_WORKLOAD_STANDALONE
extern "C" const char* g16_workload_last_error() { return g16::g_workload_err.c_str(); }
#endif
extern "C" int g16_synthetic_r1cs(int curve, uint32_t log_n, uint64_t seed, uint32_t* a_col, uint64_t* a_val, uint32_t* b_col,
                                  uint32_t* c_col, uint64_t* full_assignment) {
  using namespace g16;
  if (!a_col || !a_val || !b_col || !c_col || !full_assignment) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
  if (log_n < 3 || log_n > 28) return fail(G16_ERR_BAD_ARGUMENT, "log_n out of range (3..28)");
  switch (curve) {
    case G16_CURVE_BLS12_381: return synth<BLS381_FrP>(log_n, seed, a_col, a_val, b_col, c_col, full_assignment);
    case G16_CURVE_BN254: return synth<BN254_FrP>(log_n, seed, a_col, a_val, b_col, c_col, full_assignment);
    case G16_CURVE_BLS12_377: return synth<BLS377_FrP>(log_n, seed, a_col, a_val, b_col, c_col, full_assignment);
    case G16_CURVE_BW6_761: return synth<BW6_FrP>(log_n, seed, a_col, a_val, b_col, c_col, full_assignment);
    default: return fail(G16_ERR_BAD_ARGUMENT, "unknown curve id");
  }
}
