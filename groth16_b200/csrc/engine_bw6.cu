// engine_bw6.cu -- host orchestration (Engine<BW6_Params>) ; its kernels live in k_*_bw6.cu.  G2 is over Fq, so G1 and
// G2 share one set of MSM instances (k_msm_g1_bw6.cu) and G16_CURVE_KERNELS, which lists both, is not used here.
#include "engine.cuh"
namespace g16 {
static_assert(std::is_same<BW6_Params::G2F, Fp<BW6_FqP>>::value, "BW6-761's G2 is over Fq");
G16_NTT_TEMPLATES(extern template, Fp<BW6_FrP>)
G16_MSM_TEMPLATES(extern template, Fp<BW6_FqP>, Fp<BW6_FrP>)
G16_SER_TEMPLATES(extern template, BW6_Params)
G16_SRS_TEMPLATES(extern template, BW6_Params)
G16_R1CS_TEMPLATES(extern template, BW6_Params)
IEngine* make_engine_bw6(int device, int* rc) { return make_engine<BW6_Params>(device, rc); }
}  // namespace g16
