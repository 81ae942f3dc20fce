// k_ser_bls381.cu -- proving-key decode / encode kernels (ser.cuh), .zkey kernels (zkey.cuh) and .r1cs / .wtns kernels (r1cs.cuh) of BLS381
#include "ser.cuh"
#include "r1cs.cuh"
#include "zkey.cuh"
namespace g16 {
G16_SER_TEMPLATES(template, BLS381_Params)
G16_R1CS_TEMPLATES(template, BLS381_Params)
G16_ZKEY_TEMPLATES(template, BLS381_Params)
}  // namespace g16
