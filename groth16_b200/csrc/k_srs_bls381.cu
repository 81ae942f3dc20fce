// k_srs_bls381.cu -- transcript-setup kernels (srs.cuh) of BLS12-381
#include "srs.cuh"
namespace g16 {
G16_SRS_TEMPLATES(template, BLS381_Params)
G16_SRS_POINT_TEMPLATES(template, BLS381_Params::G2F, Fp<BLS381_FrP>)
}  // namespace g16
