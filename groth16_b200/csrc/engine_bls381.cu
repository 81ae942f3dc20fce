// engine_bls381.cu -- host orchestration (Engine<BLS381_Params>) ; its kernels live in k_*_bls381.cu
#include "engine.cuh"
namespace g16 {
G16_CURVE_KERNELS(extern template, BLS381_Params)
G16_R1CS_TEMPLATES(extern template, BLS381_Params)
G16_ZKEY_TEMPLATES(extern template, BLS381_Params)
IEngine* make_engine_bls381(int device, int* rc) { return make_engine<BLS381_Params>(device, rc); }
}  // namespace g16
