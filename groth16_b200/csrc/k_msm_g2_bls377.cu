// k_msm_g2_bls377.cu -- MSM / fixed-base kernels over G2 (Fq2) of BLS377
#include "msm.cuh"
namespace g16 {
using Fq2_bls377 = BLS377_Params::G2F;
G16_MSM_TEMPLATES(template, Fq2_bls377, Fp<BLS377_FrP>)
}  // namespace g16
