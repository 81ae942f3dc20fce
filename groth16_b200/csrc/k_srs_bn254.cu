// k_srs_bn254.cu -- transcript-setup kernels (srs.cuh) of BN254
#include "srs.cuh"
namespace g16 {
G16_SRS_TEMPLATES(template, BN254_Params)
G16_SRS_POINT_TEMPLATES(template, BN254_Params::G2F, Fp<BN254_FrP>)
}  // namespace g16
