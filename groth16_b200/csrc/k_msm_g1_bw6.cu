// k_msm_g1_bw6.cu -- MSM / fixed-base kernels over G1 and G2 of BW6-761: both curves are over Fq, and the XYZZ and
// batched-affine formulas never read the coefficient b, so one instantiation serves both groups
#include "msm.cuh"
namespace g16 {
G16_MSM_TEMPLATES(template, Fp<BW6_FqP>, Fp<BW6_FrP>)
}  // namespace g16
