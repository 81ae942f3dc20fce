// k_srs_bls377.cu -- transcript-setup kernels (srs.cuh) of BLS12-377
#include "srs.cuh"
namespace g16 {
G16_SRS_TEMPLATES(template, BLS377_Params)
G16_SRS_POINT_TEMPLATES(template, BLS377_Params::G2F, Fp<BLS377_FrP>)
}  // namespace g16
