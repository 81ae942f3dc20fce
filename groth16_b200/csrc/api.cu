// api.cu -- extern "C" surface of libg16b200.so (include/g16b200.h): argument checks, curve dispatch, error string.
#include <dlfcn.h>
#include <string>
#include "engine.cuh"

namespace g16 {
std::string& last_error_ref() {
  static thread_local std::string e;
  return e;
}
int fail(int code, const std::string& msg);   // out-of-line copy for translation units that do not include engine.cuh
NcclApi& nccl_api() {
  static NcclApi api;
  return api;
}
bool NcclApi::load() {
  if (handle) return true;
  // 1. a libnccl the host process has already loaded (torch ships its own), 2. G16_NCCL_LIB, 3. the system library
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  void* h = nullptr;
  for (const char* n : names)
    if ((h = dlopen(n, RTLD_NOW | RTLD_NOLOAD))) break;
  if (!h)
    if (const char* e = getenv("G16_NCCL_LIB")) h = dlopen(e, RTLD_NOW | RTLD_GLOBAL);
  if (!h)
    for (const char* n : names)
      if ((h = dlopen(n, RTLD_NOW | RTLD_GLOBAL))) break;
  if (!h) {
    const char* why = dlerror();   // one call: dlerror() clears the message it returns
    err = std::string("dlopen(libnccl.so.2): ") + (why ? why : "not found");
    return false;
  }
  auto sym = [&](const char* n) { return dlsym(h, n); };
  GetUniqueId = reinterpret_cast<int (*)(NcclUniqueId*)>(sym("ncclGetUniqueId"));
  CommInitRank = reinterpret_cast<int (*)(void**, int, NcclUniqueId, int)>(sym("ncclCommInitRank"));
  AllGather = reinterpret_cast<int (*)(const void*, void*, size_t, int, void*, cudaStream_t)>(sym("ncclAllGather"));
  CommDestroy = reinterpret_cast<int (*)(void*)>(sym("ncclCommDestroy"));
  Send = reinterpret_cast<int (*)(const void*, size_t, int, int, void*, cudaStream_t)>(sym("ncclSend"));
  Recv = reinterpret_cast<int (*)(void*, size_t, int, int, void*, cudaStream_t)>(sym("ncclRecv"));
  Broadcast = reinterpret_cast<int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t)>(sym("ncclBroadcast"));
  GroupStart = reinterpret_cast<int (*)()>(sym("ncclGroupStart"));
  GroupEnd = reinterpret_cast<int (*)()>(sym("ncclGroupEnd"));
  GetErrorString = reinterpret_cast<const char* (*)(int)>(sym("ncclGetErrorString"));
  if (!GetUniqueId || !CommInitRank || !AllGather || !CommDestroy || !GetErrorString || !Send || !Recv || !Broadcast || !GroupStart || !GroupEnd) { err = "libnccl lacks an expected symbol"; return false; }
  handle = h;
  return true;
}
int fail(int code, const std::string& msg) {
  last_error_ref() = msg;
  return code;
}
IEngine* make_engine_bls381(int device, int* rc);
IEngine* make_engine_bn254(int device, int* rc);
IEngine* make_engine_bls377(int device, int* rc);
}  // namespace g16

struct g16_ctx {
  g16::IEngine* eng;
};

using namespace g16;

extern "C" {

int g16_ctx_create(int curve, int device, g16_ctx** out) {
  if (!out) return fail(G16_ERR_BAD_ARGUMENT, "null out pointer");
  *out = nullptr;
  // A proof uses 6 streams per slot (witness map + five MSMs), two slots, plus the exchange stream.  With the default of 8
  // hardware work queues several of them share a queue and serialise behind each other: the H MSM would start only
  // when the L MSM has finished.  The variable is read when the CUDA
  // context is created, so this only helps when we get here before the host process touches the device; the Python package
  // and bench.py also set it at import.  An explicit setting by the user is respected.
  setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0);
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0)
    return fail(G16_ERR_CUDA, std::string("no CUDA device available (") + cudaGetErrorString(ce) + "); libg16b200 has no CPU fallback");
  if (device < 0 || device >= ndev) return fail(G16_ERR_BAD_ARGUMENT, "device index out of range");
  int rc = G16_OK;
  IEngine* e = nullptr;
  switch (curve) {
    case G16_CURVE_BLS12_381: e = make_engine_bls381(device, &rc); break;
    case G16_CURVE_BN254: e = make_engine_bn254(device, &rc); break;
    case G16_CURVE_BLS12_377: e = make_engine_bls377(device, &rc); break;
    default: return fail(G16_ERR_BAD_ARGUMENT, "unknown curve id");
  }
  if (!e) return rc ? rc : G16_ERR_CUDA;
  *out = new g16_ctx{e};
  return G16_OK;
}
void g16_ctx_destroy(g16_ctx* ctx) {
  if (!ctx) return;
  delete ctx->eng;
  delete ctx;
}
const char* g16_last_error(void) { return last_error_ref().c_str(); }

#define CTX_OR_FAIL(ctx) \
  if (!(ctx) || !(ctx)->eng) return fail(G16_ERR_BAD_ARGUMENT, "null context")

int g16_fq_limbs(const g16_ctx* ctx) { return (ctx && ctx->eng) ? ctx->eng->fq_limbs() : 0; }
int g16_partial_limbs(const g16_ctx* ctx) { return (ctx && ctx->eng) ? ctx->eng->partial_limbs() : 0; }
uint32_t g16_domain_log(const g16_ctx* ctx) { return (ctx && ctx->eng) ? ctx->eng->domain_log() : 0; }

int g16_ntt(g16_ctx* ctx, uint32_t log_n, int inverse, int coset, uint64_t* inout) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->ntt(log_n, inverse, coset, inout);
}
int g16_witness_map_evals(g16_ctx* ctx, uint32_t log_n, const uint64_t* a, const uint64_t* b, const uint64_t* c, uint64_t* h_out) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->witness_map_evals(log_n, a, b, c, h_out);
}
int g16_msm_g1(g16_ctx* ctx, const uint64_t* bases, const uint64_t* scalars, uint64_t n, uint64_t* out_xyz) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->msm_g1(bases, scalars, n, out_xyz);
}
int g16_msm_g2(g16_ctx* ctx, const uint64_t* bases, const uint64_t* scalars, uint64_t n, uint64_t* out_xyz) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->msm_g2(bases, scalars, n, out_xyz);
}
int g16_circuit_load(g16_ctx* ctx, uint32_t num_inputs, uint32_t num_constraints, uint32_t num_witness, const g16_csr* a,
                     const g16_csr* b, const g16_csr* c) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->circuit_load(num_inputs, num_constraints, num_witness, a, b, c);
}
int g16_pk_load(g16_ctx* ctx, const g16_pk_desc* pk, uint32_t rank, uint32_t world) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->pk_load(pk, rank, world);
}
int g16_setup(g16_ctx* ctx, const uint64_t* alpha, const uint64_t* beta, const uint64_t* gamma, const uint64_t* delta,
              const uint64_t* tau, const uint64_t* g1, const uint64_t* g2) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->setup(alpha, beta, gamma, delta, tau, g1, g2);
}
int g16_pk_export(g16_ctx* ctx, const g16_pk_export_desc* out) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->pk_export(out);
}
int g16_prove(g16_ctx* ctx, const uint64_t* r, const uint64_t* s, const uint64_t* full_assignment, uint32_t flags, uint64_t* proof_out) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->prove(r, s, full_assignment, flags, proof_out);
}
int g16_prove_partial(g16_ctx* ctx, const uint64_t* r, const uint64_t* full_assignment, uint32_t flags, uint64_t* partial_out) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->prove_partial(r, full_assignment, flags, partial_out);
}
int g16_prove_assemble(g16_ctx* ctx, const uint64_t* r, const uint64_t* s, const uint64_t* partials, uint32_t nparts, uint64_t* proof_out) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->prove_assemble(r, s, partials, nparts, proof_out);
}
int g16_prove_assemble_prepare(g16_ctx* ctx, const uint64_t* r, const uint64_t* s) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->assemble_prepare(r, s);
}
int g16_prove_submit(g16_ctx* ctx, int slot, const uint64_t* r, const uint64_t* s, const uint64_t* full_assignment, uint32_t flags) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->prove_submit(slot, r, s, full_assignment, flags);
}
int g16_prove_wait(g16_ctx* ctx, int slot, uint64_t* proof_out) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->prove_wait(slot, proof_out);
}
int g16_prove_partial_submit(g16_ctx* ctx, int slot, const uint64_t* r, const uint64_t* full_assignment, uint32_t flags) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->partial_submit(slot, r, full_assignment, flags);
}
int g16_prove_partial_wait(g16_ctx* ctx, int slot, uint64_t* partial_out) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->partial_wait(slot, partial_out);
}
int g16_witness_map(g16_ctx* ctx, const uint64_t* full_assignment, uint32_t flags, uint64_t* h_out) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->witness_map(full_assignment, flags, h_out);
}
int g16_get_timings(const g16_ctx* ctx, g16_timings* out) {
  CTX_OR_FAIL(ctx);
  if (!out) return fail(G16_ERR_BAD_ARGUMENT, "null out");
  *out = ctx->eng->tm;
  return G16_OK;
}

int g16_comm_unique_id(uint8_t* out128) {
  if (!out128) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
  NcclApi& api = nccl_api();
  if (!api.load()) return fail(G16_ERR_CUDA, "NCCL is not available: " + api.err);
  for (int k = 0; k < 2; k++) {   // one id per communicator: point all-gather, witness-map exchange
    NcclUniqueId id;
    const int rc = api.GetUniqueId(&id);
    if (rc != 0) return fail(G16_ERR_CUDA, std::string("ncclGetUniqueId: ") + api.GetErrorString(rc));
    memcpy(out128 + 128 * k, id.internal, 128);
  }
  return G16_OK;
}
int g16_comm_init(g16_ctx* ctx, const uint8_t* id128, uint32_t rank, uint32_t world) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->comm_init(id128, rank, world);
}
int g16_prove_sharded_submit(g16_ctx* ctx, int slot, const uint64_t* r, const uint64_t* s, const uint64_t* full_assignment, uint32_t flags) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->sharded_submit(slot, r, s, full_assignment, flags);
}
int g16_prove_sharded_wait(g16_ctx* ctx, int slot, uint64_t* proof_out) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->sharded_wait(slot, proof_out);
}
int g16_prove_sharded(g16_ctx* ctx, const uint64_t* r, const uint64_t* s, const uint64_t* full_assignment, uint32_t flags, uint64_t* proof_out) {
  CTX_OR_FAIL(ctx);
  const int rc = ctx->eng->sharded_submit(0, r, s, full_assignment, flags);
  if (rc) return rc;
  return ctx->eng->sharded_wait(0, proof_out);
}
int g16_get_config(const g16_ctx* ctx, g16_config* out) {
  CTX_OR_FAIL(ctx);
  return ctx->eng->get_config(out);
}
int g16_set_option(g16_ctx* ctx, const char* key, int64_t value) {
  CTX_OR_FAIL(ctx);
  if (!key) return fail(G16_ERR_BAD_ARGUMENT, "null key");
  return ctx->eng->set_option(key, (long long)value);
}

}  // extern "C"
