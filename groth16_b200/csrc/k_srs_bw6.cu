// k_srs_bw6.cu -- transcript-setup kernels (srs.cuh) of BW6-761
#include "srs.cuh"
namespace g16 {
G16_SRS_TEMPLATES(template, BW6_Params)
// BW6-761's G2 is over Fq: its G2 points use the G1 instances above
}  // namespace g16
