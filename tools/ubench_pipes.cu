// tools/ubench_pipes.cu -- which execution pipes bound 384-bit modular arithmetic on an H100 (sm_90a)?
// Measures, with all SMs full of warps and long independent dependency chains per thread:
//   imad_wide   mad.wide.u32 (IMAD.WIDE.U32)            the instruction the Montgomery products are made of
//   imad_lo     mad.lo.u32   (IMAD)                      32-bit multiply-add
//   dfma        fma.rz.f64   (DFMA)                      the alternative multiplier: 52-bit limbs in doubles
//   iadd3       add.u32 chains                           carry-propagation side work (ALU pipe)
//   mix_*       two of them interleaved in one thread    do the pipes overlap (separate issue ports) or serialise?
//   fq_mul_*    the library's BLS12-381 Fq product, alone and in loop bodies of growing code size (fq_mul_body)
// Output: one JSON line per test: {"test":..., "lane_ops_per_clk_per_sm":..., "gops":...}.  Used to decide whether a
// floating-point limb representation is worth building, and how large a hot loop may grow (DESIGN.md sections 3 and 6);
// not part of the product.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 --expt-relaxed-constexpr tools/ubench_pipes.cu -o tools/ubench_pipes
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>
#include "../groth16_b200/csrc/fp.cuh"

constexpr int ITER = 4096, CH = 8;

template <int MODE>
__global__ void __launch_bounds__(256) k(uint64_t* out, uint32_t seed, double dseed) {
  uint64_t a[CH];
  uint32_t c[CH];
  double d[CH];
  const uint32_t x = seed + threadIdx.x, y = seed * 3 + blockIdx.x;
  const double fx = dseed + threadIdx.x, fy = dseed * 0.5;
#pragma unroll
  for (int i = 0; i < CH; i++) { a[i] = i + x; c[i] = i * 7 + y; d[i] = fx + i; }
#pragma unroll 1
  for (int it = 0; it < ITER; it++) {
#pragma unroll
    for (int i = 0; i < CH; i++) {
      if (MODE == 0 || MODE == 4 || MODE == 5) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(a[i]) : "r"(x), "r"(c[i]));
      if (MODE == 1) asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(c[i]) : "r"(x), "r"(y));
      if (MODE == 2 || MODE == 4 || MODE == 6) asm volatile("fma.rz.f64 %0, %1, %2, %0;" : "+d"(d[i]) : "d"(fx), "d"(fy));
      if (MODE == 3 || MODE == 5 || MODE == 6) asm volatile("add.u32 %0, %0, %1;" : "+r"(c[i]) : "r"(y));
    }
  }
  uint64_t s = 0;
#pragma unroll
  for (int i = 0; i < CH; i++) s += a[i] + c[i] + (uint64_t)d[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// The library's 384-bit Montgomery product in isolation: CHAINS independent dependent-product chains per thread, resident
// warps per SM set by the dynamic shared memory request.  Upper bound of what any kernel built on fp.cuh can reach.
template <int CHAINS>
__global__ void __launch_bounds__(128) mulchain(uint32_t* out, int iters) {
  using F = g16::Fp<g16::BLS381_FqP>;
  F x[CHAINS], y = F::r2();
  for (int c = 0; c < CHAINS; c++) { x[c] = F::one(); x[c].v[0] += threadIdx.x + c; }
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int c = 0; c < CHAINS; c++) x[c] = F::mont_mul(x[c], y);   // the inlined body (F::mul is a call on the device)
  }
  uint32_t s = 0;
  for (int c = 0; c < CHAINS; c++) s += x[c].v[3];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
// Code-size sweep: one dependent product chain whose loop body is K fully inlined copies of the product (about 7 KB of
// SASS each), or, with CALL, K calls of the one out-of-line body the library's base-field products use.  The arithmetic is
// the same for every K; only the size of the straight-line body each warp runs through changes, so a drop in rate with K
// is instruction fetch (the SM's instruction caches are smaller than the larger bodies; NVIDIA does not publish sizes).
template <int K, bool CALL>
__global__ void __launch_bounds__(128) mulbody(uint32_t* out, int iters) {
  using F = g16::Fp<g16::BLS381_FqP>;
  F x = F::one(), y = F::r2();
  x.v[0] += threadIdx.x;
#pragma unroll 1
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int k = 0; k < K; k++) {
      if constexpr (CALL) x = F::mont_mul_call(x, y);
      else x = F::mont_mul(x, y);
    }
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = x.v[3];
}

// Milliseconds of the second of two launches of kern<<<sms * warps_per_sm / 4, 128>>>(out, iters), with exactly
// warps_per_sm / 4 blocks resident per SM (forced by the dynamic shared memory request).
static float time_resident(void (*kern)(uint32_t*, int), int warps_per_sm, int sms, int iters, int* blocks_out) {
  const int blocks_per_sm = warps_per_sm / 4;
  const int smem = (227 * 1024) / blocks_per_sm - 1024;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  const int blocks = sms * blocks_per_sm;
  uint32_t* out;
  cudaMalloc(&out, (size_t)blocks * 128 * 4);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  kern<<<blocks, 128, smem>>>(out, iters);
  cudaDeviceSynchronize();
  cudaEventRecord(e0);
  kern<<<blocks, 128, smem>>>(out, iters);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  cudaFree(out);
  *blocks_out = blocks;
  return ms;
}

template <int K, bool CALL>
static void run_body(int warps_per_sm, int sms, double mhz) {
  const int iters = 4096 / K;   // 4096 products per thread for every K
  int blocks = 0;
  const float ms = time_resident(mulbody<K, CALL>, warps_per_sm, sms, iters, &blocks);
  const double muls = (double)blocks * 128 * iters * K / (ms * 1e-3);
  cudaFuncAttributes fa;
  cudaFuncGetAttributes(&fa, mulbody<K, CALL>);
  printf("{\"test\": \"fq_mul_body\", \"copies\": %d, \"call\": %s, \"warps_per_sm\": %d, \"regs\": %d, \"local_bytes\": %zu, \"ms\": %.4f, "
         "\"muls_per_s\": %.4e, \"imad_wide_lanes_per_clk_per_sm\": %.2f, \"err\": \"%s\"}\n",
         K, CALL ? "true" : "false", warps_per_sm, fa.numRegs, fa.localSizeBytes, ms, muls, muls * 288 / (mhz * 1e6) / sms,
         cudaGetErrorString(cudaGetLastError()));
}

template <int CHAINS>
static void run_mul(int warps_per_sm, int sms, double mhz) {
  const int iters = 2000;
  int blocks = 0;
  const float ms = time_resident(mulchain<CHAINS>, warps_per_sm, sms, iters, &blocks);
  const double muls = (double)blocks * 128 * iters * CHAINS / (ms * 1e-3);
  printf("{\"test\": \"fq_mul_bls381\", \"chains_per_thread\": %d, \"warps_per_sm\": %d, \"ms\": %.4f, \"muls_per_s\": %.4e, \"imad_wide_per_s\": %.4e, "
         "\"imad_wide_lanes_per_clk_per_sm\": %.2f, \"err\": \"%s\"}\n",
         CHAINS, warps_per_sm, ms, muls, muls * 288, muls * 288 / (mhz * 1e6) / sms, cudaGetErrorString(cudaGetLastError()));
}

template <int MODE>
static void run(const char* name, int ops_per_slot, int sms, double mhz) {
  const int blocks = sms * 8;
  uint64_t* out;
  cudaMalloc(&out, (size_t)blocks * 256 * 8);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  k<MODE><<<blocks, 256>>>(out, 12345, 1.0000001);
  cudaDeviceSynchronize();
  cudaEventRecord(e0);
  k<MODE><<<blocks, 256>>>(out, 12345, 1.0000001);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  const double slots = (double)blocks * 256 * ITER * CH;   // (instruction group) executions, lane level
  const double per_s = slots / (ms * 1e-3);
  printf("{\"test\": \"%s\", \"ms\": %.4f, \"groups_per_s\": %.4e, \"lane_groups_per_clk_per_sm\": %.2f, \"instr_per_group\": %d}\n", name, ms, per_s,
         per_s / (mhz * 1e6) / sms, ops_per_slot);
  cudaFree(out);
}

int main() {
  cudaDeviceProp p;
  cudaGetDeviceProperties(&p, 0);
  int khz = 0;
  cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
  const double mhz = khz / 1000.0;
  printf("{\"device\": \"%s\", \"sms\": %d, \"clock_mhz_attr\": %.0f}\n", p.name, p.multiProcessorCount, mhz);
  run<0>("imad_wide", 1, p.multiProcessorCount, mhz);
  run<1>("imad_lo", 1, p.multiProcessorCount, mhz);
  run<2>("dfma", 1, p.multiProcessorCount, mhz);
  run<3>("iadd", 1, p.multiProcessorCount, mhz);
  run<4>("mix_imadwide_dfma", 2, p.multiProcessorCount, mhz);
  run<5>("mix_imadwide_iadd", 2, p.multiProcessorCount, mhz);
  run<6>("mix_dfma_iadd", 2, p.multiProcessorCount, mhz);
  for (int w : {4, 8, 12, 16, 24, 32, 48}) run_mul<1>(w, p.multiProcessorCount, mhz);
  for (int w : {4, 8, 12, 16, 24}) run_mul<2>(w, p.multiProcessorCount, mhz);
  for (int w : {8, 12}) {
    const int sms = p.multiProcessorCount;
    run_body<1, false>(w, sms, mhz);
    run_body<2, false>(w, sms, mhz);
    run_body<4, false>(w, sms, mhz);
    run_body<8, false>(w, sms, mhz);
    run_body<16, false>(w, sms, mhz);
    run_body<32, false>(w, sms, mhz);
    run_body<32, true>(w, sms, mhz);
  }
  return 0;
}
