// k_ntt_bls377.cu -- NTT / witness-map kernels over the scalar field of BLS377
#include "ntt.cuh"
namespace g16 {
G16_NTT_TEMPLATES(template, Fp<BLS377_FrP>)
}  // namespace g16
