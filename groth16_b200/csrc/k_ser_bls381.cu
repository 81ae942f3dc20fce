// k_ser_bls381.cu -- proving-key decode / encode kernels (ser.cuh) of BLS381
#include "ser.cuh"
namespace g16 {
G16_SER_TEMPLATES(template, BLS381_Params)
}  // namespace g16
