// engine_bn254.cu -- host orchestration (Engine<BN254_Params>) ; its kernels live in k_*_bn254.cu
#include "engine.cuh"
namespace g16 {
G16_CURVE_KERNELS(extern template, BN254_Params)
G16_R1CS_TEMPLATES(extern template, BN254_Params)
G16_ZKEY_TEMPLATES(extern template, BN254_Params)
IEngine* make_engine_bn254(int device, int* rc) { return make_engine<BN254_Params>(device, rc); }
}  // namespace g16
