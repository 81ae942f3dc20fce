// k_ser_bw6.cu -- proving-key decode / encode kernels (ser.cuh) and .r1cs / .wtns kernels (r1cs.cuh) of BW6-761
#include "ser.cuh"
#include "r1cs.cuh"
namespace g16 {
G16_SER_TEMPLATES(template, BW6_Params)
G16_R1CS_TEMPLATES(template, BW6_Params)
}  // namespace g16
