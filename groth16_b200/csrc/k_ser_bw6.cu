// k_ser_bw6.cu -- proving-key decode / encode kernels (ser.cuh) of BW6-761
#include "ser.cuh"
namespace g16 {
G16_SER_TEMPLATES(template, BW6_Params)
}  // namespace g16
