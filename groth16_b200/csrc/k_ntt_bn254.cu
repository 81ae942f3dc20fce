// k_ntt_bn254.cu -- NTT / witness-map kernels over the scalar field of BN254
#include "ntt.cuh"
namespace g16 {
G16_NTT_TEMPLATES(template, Fp<BN254_FrP>)
}  // namespace g16
