// engine_bls377.cu -- host orchestration (Engine<BLS377_Params>) ; its kernels live in k_*_bls377.cu
#include "engine.cuh"
namespace g16 {
G16_CURVE_KERNELS(extern template, BLS377_Params)
G16_R1CS_TEMPLATES(extern template, BLS377_Params)
IEngine* make_engine_bls377(int device, int* rc) { return make_engine<BLS377_Params>(device, rc); }
}  // namespace g16
