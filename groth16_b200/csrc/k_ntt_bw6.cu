// k_ntt_bw6.cu -- NTT / witness-map kernels over the scalar field of BW6-761 (BLS12-377's base field)
#include "ntt.cuh"
namespace g16 {
G16_NTT_TEMPLATES(template, Fp<BW6_FrP>)
}  // namespace g16
