// k_ser_bls377.cu -- proving-key decode / encode kernels (ser.cuh) of BLS377
#include "ser.cuh"
namespace g16 {
G16_SER_TEMPLATES(template, BLS377_Params)
}  // namespace g16
