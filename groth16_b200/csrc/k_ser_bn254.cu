// k_ser_bn254.cu -- proving-key decode / encode kernels (ser.cuh) of BN254
#include "ser.cuh"
namespace g16 {
G16_SER_TEMPLATES(template, BN254_Params)
}  // namespace g16
