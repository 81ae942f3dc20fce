// k_ser_bls377.cu -- proving-key decode / encode kernels (ser.cuh) and .r1cs / .wtns kernels (r1cs.cuh) of BLS377
#include "ser.cuh"
#include "r1cs.cuh"
namespace g16 {
G16_SER_TEMPLATES(template, BLS377_Params)
G16_R1CS_TEMPLATES(template, BLS377_Params)
}  // namespace g16
