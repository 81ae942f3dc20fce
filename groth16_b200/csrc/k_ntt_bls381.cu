// k_ntt_bls381.cu -- NTT / witness-map kernels over the scalar field of BLS381
#include "ntt.cuh"
namespace g16 {
G16_NTT_TEMPLATES(template, Fp<BLS381_FrP>)
}  // namespace g16
