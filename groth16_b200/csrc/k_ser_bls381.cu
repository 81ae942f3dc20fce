// k_ser_bls381.cu -- proving-key decode / encode kernels (ser.cuh) and .zkey kernels (zkey.cuh) of BLS381
#include "ser.cuh"
#include "zkey.cuh"
namespace g16 {
G16_SER_TEMPLATES(template, BLS381_Params)
G16_ZKEY_TEMPLATES(template, BLS381_Params)
}  // namespace g16
