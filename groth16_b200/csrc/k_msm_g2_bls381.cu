// k_msm_g2_bls381.cu -- MSM / fixed-base kernels over G2 (Fq2) of BLS381
#include "msm.cuh"
namespace g16 {
using Fq2_bls381 = BLS381_Params::G2F;
G16_MSM_TEMPLATES(template, Fq2_bls381, Fp<BLS381_FrP>)
}  // namespace g16
