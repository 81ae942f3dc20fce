// k_msm_g2_bn254.cu -- MSM / fixed-base kernels over G2 (Fq2) of BN254
#include "msm.cuh"
namespace g16 {
using Fq2_bn254 = BN254_Params::G2F;
G16_MSM_TEMPLATES(template, Fq2_bn254, Fp<BN254_FrP>)
}  // namespace g16
