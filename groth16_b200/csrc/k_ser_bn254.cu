// k_ser_bn254.cu -- proving-key decode / encode kernels (ser.cuh), .zkey kernels (zkey.cuh) and .r1cs / .wtns kernels (r1cs.cuh) of BN254
#include "ser.cuh"
#include "r1cs.cuh"
#include "zkey.cuh"
namespace g16 {
G16_SER_TEMPLATES(template, BN254_Params)
G16_R1CS_TEMPLATES(template, BN254_Params)
G16_ZKEY_TEMPLATES(template, BN254_Params)
}  // namespace g16
