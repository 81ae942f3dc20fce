// engine.cuh -- per-curve host orchestration of the proving hot path behind the C ABI (include/g16b200.h).
//
// Mirrors, function by function, what /root/reference does between `create_proof_with_reduction_and_matrices`
// (prover.rs:26-51) and `Proof{a,b,c}` (prover.rs:127-131); the heavy steps are the CUDA kernels of ntt.cuh and
// msm.cuh, the O(1) tail (scalar multiplications by r and s, sums, into_affine; batch.cuh) runs on the host with the
// same field code.
#pragma once
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>       // header-only NVTX v3: no-ops unless a profiler injects itself
#include <nvtx3/nvToolsExtCudaRt.h>
#include <algorithm>
#include <array>
#include <cctype>
#include <cerrno>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstdio>
#include <condition_variable>
#include <deque>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>
#include "../../include/g16b200.h"
#include "batch.cuh"
#include "ec.cuh"
#include "msm.cuh"
#include "ntt.cuh"
#include "ser.cuh"
#include "srs.cuh"
#include "zkey.cuh"
#include "r1cs.cuh"
#include "ptau.cuh"

namespace g16 {

std::string& last_error_ref();
int fail(int code, const std::string& msg);   // api.cu
#define G16_CUDA(x)                                                                                       \
  do {                                                                                                    \
    cudaError_t _e = (x);                                                                                 \
    if (_e != cudaSuccess)                                                                                \
      return fail(G16_ERR_CUDA, std::string(#x) + ": " + cudaGetErrorString(_e) + " @" + __FILE__ + ":" + \
                                    std::to_string(__LINE__));                                            \
  } while (0)

// NVTX ranges named after the reference's own `start_timer!` spans (prover.rs:35,36,62,89,99,111,119; SURVEY.md section 5),
// so a Nsight timeline of this library reads like ark's `print-trace` output.  Host ranges bracket the enqueue of each
// stage; the CUDA streams carry the same names, which is where the asynchronous GPU work of the stage shows up.
struct NvtxSpan {
  explicit NvtxSpan(const char* name) { nvtxRangePushA(name); }
  ~NvtxSpan() { nvtxRangePop(); }
};
static constexpr const char* SPAN_PROVER = "Groth16::Prover";                 // prover.rs:35
static constexpr const char* SPAN_WITNESS_MAP = "R1CS to QAP witness map";    // prover.rs:36
static constexpr const char* SPAN_C = "Compute C";                            // prover.rs:62  (H and L MSMs, r*s*delta)
static constexpr const char* SPAN_A = "Compute A";                            // prover.rs:89
static constexpr const char* SPAN_B1 = "Compute B in G1";                     // prover.rs:99
static constexpr const char* SPAN_B2 = "Compute B in G2";                     // prover.rs:111
static constexpr const char* SPAN_FINISH_C = "Finish C";                      // prover.rs:119

// Persistent host workers of one context (one per MSM stream + one for the (r, s)-only scalar multiplications): a proof
// used to spawn and join six std::threads (VERDICT r1: visible as host-side contention with 8 replica processes per box).
class HostPool {
 public:
  struct Ticket {   // completion handle of one task
    std::mutex m;
    std::condition_variable cv;
    bool done = false;
    void wait() { std::unique_lock<std::mutex> l(m); cv.wait(l, [&] { return done; }); }
  };
  explicit HostPool(int n) {
    for (int i = 0; i < n; i++) th_.emplace_back([this] { run(); });
  }
  ~HostPool() {
    { std::lock_guard<std::mutex> l(m_); stop_ = true; }
    cv_.notify_all();
    for (auto& t : th_) t.join();
  }
  std::shared_ptr<Ticket> submit(std::function<void()> fn) {
    auto tk = std::make_shared<Ticket>();
    { std::lock_guard<std::mutex> l(m_); q_.emplace_back(std::move(fn), tk); }
    cv_.notify_one();
    return tk;
  }
 private:
  void run() {
    for (;;) {
      std::pair<std::function<void()>, std::shared_ptr<Ticket>> job;
      {
        std::unique_lock<std::mutex> l(m_);
        cv_.wait(l, [&] { return stop_ || !q_.empty(); });
        if (q_.empty()) return;
        job = std::move(q_.front());
        q_.pop_front();
      }
      job.first();
      { std::lock_guard<std::mutex> l(job.second->m); job.second->done = true; }
      job.second->cv.notify_all();
    }
  }
  std::vector<std::thread> th_;
  std::mutex m_;
  std::condition_variable cv_;
  std::deque<std::pair<std::function<void()>, std::shared_ptr<Ticket>>> q_;
  bool stop_ = false;
};

// ---- NCCL, resolved at run time --------------------------------------------------------------------------------------
// The final point exchange of a sharded proof is an NCCL all-gather issued by the library itself (north_star: "NCCL-over-
// NVLink only for the final partial-sum / G1/G2 point reduction").  libnccl is not linked: the process that hosts us
// (torch.distributed in bench.py and the tests, or a Rust/MPI launcher) has normally loaded its own copy already, and
// two different NCCL builds in one process are asking for trouble -- so the already-loaded library is looked up first.
struct NcclUniqueId { char internal[128]; };
struct NcclApi {
  void* handle = nullptr;
  int (*GetUniqueId)(NcclUniqueId*) = nullptr;
  int (*CommInitRank)(void**, int, NcclUniqueId, int) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*Send)(const void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*Recv)(void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*Broadcast)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  std::string err;
  bool load();
};
NcclApi& nccl_api();

struct IEngine {
  virtual ~IEngine() {}
  virtual int fq_limbs() const = 0;
  virtual int fr_limbs() const = 0;
  virtual int g2_limbs() const = 0;
  virtual int partial_limbs() const = 0;
  virtual int ntt(uint32_t log_n, int inverse, int coset, uint64_t* inout) = 0;
  virtual int witness_map_evals(uint32_t log_n, const uint64_t* a, const uint64_t* b, const uint64_t* c, uint64_t* h) = 0;
  virtual int msm_g1(const uint64_t* bases, const uint64_t* scalars, uint64_t n, uint64_t* out) = 0;
  virtual int msm_g2(const uint64_t* bases, const uint64_t* scalars, uint64_t n, uint64_t* out) = 0;
  virtual int circuit_load(int qap, uint32_t ni, uint32_t nc, uint32_t nw, const g16_csr* a, const g16_csr* b, const g16_csr* c) = 0;
  virtual int pk_load(const g16_pk_desc* pk, uint32_t rank, uint32_t world) = 0;
  virtual int setup(const uint64_t* alpha, const uint64_t* beta, const uint64_t* gamma, const uint64_t* delta,
                    const uint64_t* tau, const uint64_t* g1, const uint64_t* g2) = 0;
  virtual int pk_export(const g16_pk_export_desc* out) = 0;
  virtual int setup_from_srs(const g16_srs_desc* srs, uint32_t flags) = 0;
  virtual int setup_contribute(const uint64_t* delta) = 0;
  virtual int srs_from_secrets(const uint64_t* tau, const uint64_t* alpha, const uint64_t* beta, const uint64_t* g1,
                               const uint64_t* g2, const g16_srs_out* out) = 0;
  virtual int srs_contribute(const g16_srs_desc* in, const uint64_t* tau, const uint64_t* alpha, const uint64_t* beta,
                             uint32_t flags, uint64_t chunk_points, const g16_srs_out* out) = 0;
  virtual int srs_verify_pairs(const g16_srs_desc* srs, const uint64_t* g1, const uint64_t* g2, const uint64_t* rho,
                               uint32_t flags, uint64_t chunk_points, uint64_t* pairs_g1, uint64_t* pairs_g2) = 0;
  virtual int pk_verify_pairs(const g16_srs_desc* srs, const g16_pk_check_desc* pk, const uint64_t* rho, uint32_t flags,
                              uint64_t* pairs_g1, uint64_t* pairs_g2) = 0;
  virtual int pk_contribute(const g16_pk_delta_desc* in, const uint64_t* delta, uint32_t flags, uint64_t chunk_points,
                            const g16_pk_delta_out* out) = 0;
  virtual int contribution_chain_pairs(const uint64_t* start_g1, const uint64_t* end_g1, const g16_contribution_record* records,
                                       uint32_t count, uint32_t flags, uint64_t* pairs_g1, uint64_t* pairs_g2) = 0;
  virtual int pk_load_serialized(const uint8_t* bytes, uint64_t len, uint32_t flags, uint32_t rank, uint32_t world,
                                 const g16_pk_export_desc* vk_out) = 0;
  virtual int pk_export_serialized(uint32_t flags, uint8_t* out, uint64_t cap, uint64_t* len_out) = 0;
  virtual int zkey_load(const uint8_t* bytes, uint64_t len, uint32_t flags, uint32_t rank, uint32_t world,
                        const g16_pk_export_desc* vk_out, g16_zkey_info* info_out) = 0;
  virtual int r1cs_load(int qap, const uint8_t* bytes, uint64_t len, g16_r1cs_info* info_out) = 0;
  virtual int wtns_read(const uint8_t* bytes, uint64_t len, uint64_t* out, uint64_t cap, uint64_t* count_out) = 0;
  virtual int ptau_read(const uint8_t* bytes, uint64_t len, const g16_srs_out* srs_out, g16_lagrange_out* lag_out,
                        g16_ptau_info* info) = 0;
  virtual int setup_from_lagrange(const g16_srs_desc* srs, const g16_lagrange_desc* lag, const uint64_t* rho, uint32_t flags) = 0;
  virtual int ptau_prepare(const uint8_t* in, uint64_t in_len, uint32_t flags, uint8_t* out, uint64_t cap, uint64_t* len_out) = 0;
  virtual int prove(const uint64_t* r, const uint64_t* s, const uint64_t* z, uint32_t flags, uint64_t* proof) = 0;
  virtual int prove_partial(const uint64_t* r, const uint64_t* z, uint32_t flags, uint64_t* partial) = 0;
  virtual int prove_assemble(const uint64_t* r, const uint64_t* s, const uint64_t* partials, uint32_t nparts, uint64_t* proof) = 0;
  virtual int assemble_prepare(const uint64_t* r, const uint64_t* s) = 0;
  virtual int prove_submit(int slot, const uint64_t* r, const uint64_t* s, const uint64_t* z, uint32_t flags) = 0;
  virtual int prove_wait(int slot, uint64_t* proof) = 0;
  virtual int prove_batch(uint32_t count, const uint64_t* r, const uint64_t* s, const uint64_t* z, uint32_t group, uint32_t flags,
                          uint64_t* proofs) = 0;
  virtual int partial_submit(int slot, const uint64_t* r, const uint64_t* z, uint32_t flags) = 0;
  virtual int partial_wait(int slot, uint64_t* partial) = 0;
  virtual int witness_map(const uint64_t* z, uint32_t flags, uint64_t* h) = 0;
  virtual int check_witness(uint32_t count, const uint64_t* z, uint32_t flags, g16_witness_report* out) = 0;
  virtual uint32_t domain_log() const = 0;
  virtual int comm_init(const uint8_t* id128, uint32_t rank, uint32_t world) = 0;
  virtual int sharded_submit(int slot, const uint64_t* r, const uint64_t* s, const uint64_t* z, uint32_t flags) = 0;
  virtual int sharded_wait(int slot, uint64_t* proof) = 0;
  virtual int set_option(const char* key, long long value) = 0;
  virtual int get_option(const char* key, long long* value) const = 0;
  virtual int get_config(g16_config* out) const = 0;
  g16_timings tm{};
  // the resident circuit came from a full .zkey load: matrix C is resident empty, and the calls that read it refuse (api.cu)
  bool circuit_without_c = false;
};

// ------------------------------------------------------------------------------------------------
template <class CP>
struct Engine : IEngine {
  using Fr = Fp<typename CP::FrP>;
  using Fq = Fp<typename CP::FqP>;
  using Fq2 = typename CP::G2F;   // G2's coordinate field: Fq2, or Fq itself (BW6-761)
  using A1 = Affine<Fq>;
  using A2 = Affine<Fq2>;
  using P1 = XYZZ<Fq>;
  using P2 = XYZZ<Fq2>;
  static constexpr int NQ64 = Fq::N / 2;
  static constexpr int FR64 = Fr::N / 2;                  // u64 limbs of one ABI scalar
  static constexpr int G2_64 = (int)(sizeof(A2) / 8);     // u64 limbs of one ABI G2 affine point
  static constexpr int PROOF64 = 4 * NQ64 + G2_64;        // A (G1) || B (G2) || C (G1)
  static constexpr int FR_BITS = CP::FrP::BITS;
  enum { M_H = 0, M_L = 1, M_A = 2, M_B1 = 3, M_B2 = 4 };
  static const char* span_of(int m) {
    switch (m) {
      case M_H: return "Compute C: h_query MSM";
      case M_L: return "Compute C: l_query MSM";
      case M_A: return SPAN_A;
      case M_B1: return SPAN_B1;
      default: return SPAN_B2;
    }
  }

  int device = 0;
  // Everything one in-flight proof owns: streams, events, work vectors, MSM workspaces, timings.  Two slots allow a
  // software pipeline (g16_prove_submit / g16_prove_wait): the latency-bound tail of proof i overlaps the bulk of proof i+1.
  using Products = KeyProducts<Fq, Fq2>;
  // MSM results of this rank; sa = s * a and rb1 = r * b1 are formed by the finisher threads of the A / B-in-G1 MSMs as soon
  // as those MSMs are done (scaled == true), i.e. while the H MSM is still running, instead of after everything.
  struct Partials { P1 h, l, a, b1; P2 b2; P1 sa, rb1; bool scaled = false; };
  struct Slot {
    cudaStream_t st_main = nullptr, st_msm[5] = {};
    cudaEvent_t ev_start = nullptr, ev_z = nullptr, ev_h = nullptr, ev_m0[5] = {}, ev_m1[5] = {}, ev_a0[5] = {}, ev_a1[5] = {};
    cudaEvent_t ev_bsort = nullptr;   // B-in-G2's sorted entry list is complete (B-in-G1 borrows it)
    MsmSorted b_sorted;
    DevBuf d_z, d_a, d_b, d_c, d_t, d_h;
    MsmWorkspace<Fq> ws1[4];
    MsmWorkspace<Fq2> ws2;
    g16_timings tm{};
    // state of the submission in flight
    bool busy = false, serial = false, have_s = false;
    bool split_wm = false;   // this submission spreads the witness map over the ranks (sharded proof with a communicator)
    bool run[5] = {};
    MsmGeom geom[5] = {};
    Fr r, s;
    Products kp;
    std::shared_ptr<HostPool::Ticket> helper, helper2;   // key products in flight on the pool
    unsigned long long launches0 = 0;
    // batch proving (g16_prove_batch): the group this slot holds, and its fixed-base products
    uint32_t batch_first = 0, batch_count = 0;
    DevBuf d_tail;          // per proof: r, s, r s (Fr), then r d1, (r s) d1, s P_a, r P_b (G1 affine), s d2 (G2 affine)
    uint64_t* h_tail = nullptr;   // pinned copy of d_tail
    size_t h_tail_cap = 0;
    // G16_CHECK_WITNESS: the submission checks its assignments (r1cs_check); d_check -> h_check (pinned) after the witness
    // map, read where the results are collected
    bool check = false;
    DevBuf d_check;
    uint32_t* h_check = nullptr;
    size_t h_check_cap = 0;
  };
  static constexpr int NSLOTS = 2;
  Slot slots[NSLOTS];
  Slot& S0 = slots[0];   // slot used by the synchronous entry points
  std::unique_ptr<HostPool> pool;   // 5 MSM finishers + 2 helpers, alive for the context's lifetime
  NttDomain<Fr> dom;       // domain of the RESIDENT circuit (size 2^L); only circuit_load / the prover touch it
  NttDomain<Fr> dom_api;   // domain of the stand-alone g16_ntt / g16_witness_map_evals calls (any size): kept apart so that
                           // an NTT of another size between circuit_load and prove cannot leave the prover with the wrong
                           // twiddles (ADVICE r1: the two used to share `dom`)
  MsmCounters ctr;
  unsigned long long ntt_launches = 0;

  // resident circuit
  bool have_circuit = false;
  int qap = G16_QAP_LIBSNARK;   // its R1CS-to-QAP reduction: the witness map and the H query follow it
  uint32_t num_inputs = 0, num_constraints = 0, num_witness = 0;
  int L = 0;
  DevBuf csr_rp[3], csr_col[3], csr_val[3];
  std::vector<uint32_t> h_rp[3], h_col[3];   // host copies kept for g16_setup
  std::vector<Fr> h_val[3];

  // resident proving key (this rank's shard)
  bool have_pk = false;
  uint32_t rank = 0, world = 1;
  struct Shard {
    uint64_t pairs = 0;   // full MSM length
    uint64_t lo = 0, hi = 0;   // this rank owns pairs lo, lo + world, lo + 2 world, ... : hi - lo of them (lo = rank)
    MsmGeom geom{};
  };
  struct Query : Shard {
    DevBuf bases, mask;   // bases: geom.copies * (hi - lo) affine points, copy-major (copy j = 2^(c*ne*j) * P)
  } q[5];
  // Tuning options: defaults below (from sweeps of a full proof at 2^20, tools/sweep.py), overridden at context creation by
  // the environment and at run time by g16_set_option.  options() lists them.
  struct Tune {
    long long c = 0;          // window bits; 0 = pick from n
    long long ne = 1;         // effective windows with precomputed bases; 0 = no precomputation
    long long maxcopies = MSM_MAX_COPIES;
    long long ba_g1 = 4;      // batched-affine rounds before the XYZZ accumulation, G1 MSMs with >= 2^18 entries
    long long ba_g2 = 4;      // same for the G2 MSM (on an H100 a fifth round costs more than it saves)
    long long ba_m = 32;      // additions per thread and round
    long long ba_G = 16;      // thread products per inversion
    long long ba_gcd = 1;     // safegcd inversion
    long long k0_g1 = 0;      // sorted entries per accumulation thread (0 = automatic)
    long long k0_g2 = 0;
    long long acc_block = 128;
    // Smallest MSM (in bucket entries) that runs the rounds, and how many: a round halves a list whose buckets hold
    // `entries / buckets` slots on average and pads every bucket to 2^R slots, so R is the smallest value with
    // 11 * 2^R >= that average, capped by ba_g1 / ba_g2 (4 / 4 at
    // 2^20 pairs on one GPU, 3 on the 2.1 M-entry shards of an 8-way proof, 2 on its 1.0 M-entry A / B shards).
    long long ba_min_g1 = 1ll << 19;
    long long ba_min_g2 = 1ll << 19;
    long long ba_adaptive = 1;   // 0: exactly ba_g1 / ba_g2 rounds whatever the bucket occupancy (tests)
    long long share_b_sort = 1;  // let B-in-G2 borrow B-in-G1's sorted list when the keys allow it
    // 1 / 0 / -1 = automatic (sharded keys): hold the MSM accumulations back until the witness map is done.  Off: with
    // enough hardware work queues (CUDA_DEVICE_MAX_CONNECTIONS, see api.cu) the witness map is not held up, and delaying
    // the other accumulations then only idles the GPU
    long long wm_first = 0;
    long long wm_split = 1;      // sharded proofs with a communicator: spread the witness map over the ranks
    long long proof_slots = NSLOTS;   // slots the caller will use (1 halves the workspace the key must leave room for)
  } tune;
  // What a change of an option must redo.
  enum OptEffect {
    OPT_GEOM,        // re-derive the launch geometry of the resident key now
    OPT_NEXT_KEY,    // nothing: read at the next g16_pk_load / g16_setup
    OPT_B_SORT,      // re-decide whether B-in-G2 borrows B-in-G1's sorted list
    OPT_BA_MEMORY,   // re-decide which MSMs' round work lists fit in device memory
    OPT_NONE         // nothing: read by every proof
  };
  struct OptRange { long long lo, hi; };
  struct Option {
    const char* name;          // g16_set_option key; the environment variable is G16_<NAME IN UPPER CASE>
    long long Tune::*value;
    std::vector<OptRange> ok;  // accepted values: the union of these closed ranges
    OptEffect effect;
  };
  static const std::vector<Option>& options() {
    static const std::vector<Option> t = {
        {"msm_ne", &Tune::ne, {{0, 32}}, OPT_NEXT_KEY},
        {"msm_c", &Tune::c, {{0, 24}}, OPT_NEXT_KEY},
        {"msm_maxcopies", &Tune::maxcopies, {{1, MSM_MAX_COPIES}}, OPT_NEXT_KEY},
        {"msm_ba", &Tune::ba_g1, {{0, MSM_BA_MAX_ROUNDS}}, OPT_GEOM},
        {"msm_ba_g2", &Tune::ba_g2, {{0, MSM_BA_MAX_ROUNDS}}, OPT_GEOM},
        {"ba_m", &Tune::ba_m, {{1, 256}}, OPT_GEOM},
        {"ba_g", &Tune::ba_G, {{1, 4096}}, OPT_GEOM},
        {"ba_min_entries_g1", &Tune::ba_min_g1, {{0, LLONG_MAX}}, OPT_GEOM},
        {"ba_min_entries_g2", &Tune::ba_min_g2, {{0, LLONG_MAX}}, OPT_GEOM},
        {"acc_k0_g1", &Tune::k0_g1, {{0, 0}, {4, 1024}}, OPT_GEOM},
        {"acc_k0_g2", &Tune::k0_g2, {{0, 0}, {4, 1024}}, OPT_GEOM},
        {"acc_block", &Tune::acc_block, {{32, 32}, {64, 64}, {128, 128}}, OPT_GEOM},
        {"ba_inv_gcd", &Tune::ba_gcd, {{0, 1}}, OPT_GEOM},
        {"ba_adaptive", &Tune::ba_adaptive, {{0, 1}}, OPT_GEOM},
        {"share_b_sort", &Tune::share_b_sort, {{0, 1}}, OPT_B_SORT},
        {"wm_first", &Tune::wm_first, {{-1, 1}}, OPT_NONE},
        {"wm_split", &Tune::wm_split, {{0, 1}}, OPT_NONE},
        {"proof_slots", &Tune::proof_slots, {{1, NSLOTS}}, OPT_BA_MEMORY},
    };
    return t;
  }
  static const Option* find_option(const std::string& name) {
    for (const Option& o : options())
      if (name == o.name) return &o;
    return nullptr;
  }
  static bool accepts(const Option& o, long long v) {
    for (const OptRange& r : o.ok)
      if (v >= r.lo && v <= r.hi) return true;
    return false;
  }
  static std::string accepted(const Option& o) {   // e.g. "0, 4 .. 1024"
    std::string s;
    for (const OptRange& r : o.ok) {
      s += (s.empty() ? "" : ", ") + std::to_string(r.lo);
      if (r.hi > r.lo) s += " .. " + (r.hi == LLONG_MAX ? std::string() : std::to_string(r.hi));
    }
    return s;
  }
  MsmGeom pick_geom(uint64_t cnt) const {
    if (tune.ne <= 0) return msm_geom(cnt, FR_BITS, (int)tune.c, 0);
    // with all windows sharing one bucket set the bucket count is 2^(c-1) whatever the size: c = 16 from 2^16 pairs up
    // (also for the per-rank shards of a multi-GPU run), the size-based rule below that
    const int c = tune.c > 0 ? (int)tune.c : (cnt >= (1u << 16) ? 16 : 0);
    int ne = (int)tune.ne;
    MsmGeom g = msm_geom(cnt, FR_BITS, c, ne);
    while (g.copies > tune.maxcopies) g = msm_geom(cnt, FR_BITS, c, ++ne);
    return g;
  }
  // entries per level-0 thread, from the number of resident accumulation threads of this device
  int sm_count = 132;
  bool ba_allowed = true;   // cleared by pk_load / setup when the rounds' work lists would not fit in device memory
  uint32_t ba_allowed_mask = 0x1f;   // per MSM (bit m): the work lists of MSM m fit next to the key and the other MSMs' lists
  MsmGeom with_k0(MsmGeom g, bool g2, int m = -1) const {
    g.k0 = msm_pick_k0(g.max_entries, (uint64_t)sm_count * 128 * (g2 ? 2 : 3), g2 ? MSM_K0_AUTO_MIN_G2 : MSM_K0_AUTO_MIN_G1);
    // G2 additions are ~3x longer: 32 entries per thread (twice the thread count) shortens the last partial wave (-13 %)
    if (g2 && g.k0 > 32) g.k0 = 32;
    const int k = (int)(g2 ? tune.k0_g2 : tune.k0_g1);
    if (k >= 4 && k <= 1024) g.k0 = k;
    // batched-affine pre-reduction (msm_ba.cuh) for MSMs with at least 2^18 entries
    const int r = (int)(g2 ? tune.ba_g2 : tune.ba_g1);
    const bool allowed = ba_allowed && (m < 0 || ((ba_allowed_mask >> m) & 1));
    const uint64_t min_entries = (uint64_t)std::max(1ll << 18, g2 ? tune.ba_min_g2 : tune.ba_min_g1);
    int r_fit = 0;   // smallest R with 11 * 2^R >= average entries per bucket
    for (uint64_t per_bucket = g.max_entries / std::max<uint64_t>(1, g.nkeys); (11ull << r_fit) < per_bucket; r_fit++) {}
    if (!tune.ba_adaptive) r_fit = r;
    g.ba = (allowed && r > 0 && g.max_entries >= min_entries) ? std::min(std::min(r, r_fit), (int)MSM_BA_MAX_ROUNDS) : 0;
    g.ba_m = (int)tune.ba_m;
    g.ba_G = (int)tune.ba_G;
    g.ba_gcd = (int)tune.ba_gcd;
    g.acc_block = (int)tune.acc_block;
    return g;
  }
  bool share_b_sort = false;   // set when a key is made resident: b_g1_query and b_g2_query have the same identity pattern
  void refresh_geoms() {   // after a knob changed: same shards, new launch geometry
    for (int m = 0; m < 5; m++)
      if (q[m].hi > q[m].lo) q[m].geom = with_k0(q[m].geom, m == M_B2, m);
    // one padding for the list B1 lends to B2
    const int pad = std::max(q[M_B1].geom.ba, q[M_B2].geom.ba);
    q[M_B1].geom.ba_pad = share_b_sort ? pad : q[M_B1].geom.ba;
    q[M_B2].geom.ba_pad = share_b_sort ? pad : q[M_B2].geom.ba;
    for (int m : {M_H, M_L, M_A}) q[m].geom.ba_pad = q[m].geom.ba;
  }
  // B2 may borrow B1's sorted list iff both queries have the same shard, window geometry and identity mask
  int decide_b_sort_sharing() {
    share_b_sort = false;
    const Query &x = q[M_B1], &y = q[M_B2];
    const uint64_t cnt = x.hi - x.lo;
    if (tune.share_b_sort && cnt > 0 && cnt == y.hi - y.lo && x.lo == y.lo && x.geom.c == y.geom.c && x.geom.ne == y.geom.ne &&
        x.geom.copies == y.geom.copies) {
      std::vector<uint8_t> mx(cnt), my(cnt);
      G16_CUDA(cudaMemcpy(mx.data(), x.mask.p, cnt, cudaMemcpyDeviceToHost));
      G16_CUDA(cudaMemcpy(my.data(), y.mask.p, cnt, cudaMemcpyDeviceToHost));
      share_b_sort = mx == my;
    }
    return G16_OK;
  }
  // Work lists of the batched-affine rounds for all five MSMs of one proof slot; the rounds are switched off for this
  // key when two slots' worth would not fit next to the resident key (e.g. 2^24 constraints on one 80 GB GPU).
  void decide_ba_memory() {
    ba_allowed = true;
    ba_allowed_mask = 0x1f;
    refresh_geoms();
    size_t fr = 0, tot = 0;
    if (cudaMemGetInfo(&fr, &tot) != cudaSuccess) return;
    // The plain pipeline of every MSM (sorted index / key arrays, level-0 partial sums) is allocated whatever is decided
    // here: at 2^24 constraints it alone is ~16 GB per proof slot, so it is set aside before any work list is granted.
    uint64_t plain = 0;
    for (int m : {M_H, M_L, M_A, M_B1, M_B2}) {
      if (q[m].hi <= q[m].lo) continue;
      MsmGeom g = q[m].geom;
      g.ba = g.ba_pad = 0;
      MsmBaPlan bp;
      bp.make(g);
      plain += bp.len[0] * 8 + 2 * bp.l0_threads(g) * (4 + (m == M_B2 ? sizeof(XYZZ<Fq2>) : sizeof(XYZZ<Fq>)));
    }
    // greedy, G1 MSMs first (their lists are half the size of the G2 ones): keep the rounds for an MSM while the plain
    // pipelines and the lists of all MSMs granted so far fit `proof_slots` times into the free memory, with 10 GB to spare
    // for everything else (NTT domain and work vectors, CUDA context)
    const uint64_t margin = 10ull << 30;
    uint64_t used = 0;
    uint32_t mask = 0;
    for (int m : {M_H, M_L, M_A, M_B1, M_B2}) {
      if (q[m].hi <= q[m].lo) { mask |= 1u << m; continue; }
      MsmBaPlan bp;
      bp.make(q[m].geom);
      const uint64_t need = ((m == M_B2) ? bp.template extra_bytes<Fq2>() : bp.template extra_bytes<Fq>()) +
                            (bp.len[0] - q[m].geom.max_entries) * 8;   // bucket padding of the sorted arrays
      if ((uint64_t)tune.proof_slots * (plain + used + need) + margin <= fr) { used += need; mask |= 1u << m; }
    }
    ba_allowed_mask = mask;
    refresh_geoms();
  }
  int set_option(const char* key, long long v) override {
    if (any_busy()) return fail(G16_ERR_BAD_ARGUMENT, "a proof is in flight");
    const std::string k(key ? key : "");
    const Option* o = find_option(k);
    if (!o) return fail(G16_ERR_BAD_ARGUMENT, "unknown option: " + k);
    if (!accepts(*o, v))
      return fail(G16_ERR_BAD_ARGUMENT, "option " + k + " = " + std::to_string(v) + " is not one of " + accepted(*o));
    tune.*o->value = v;
    switch (o->effect) {
      case OPT_GEOM: refresh_geoms(); break;
      case OPT_B_SORT:
        if (have_pk) { int rc = decide_b_sort_sharing(); if (rc) return rc; }
        refresh_geoms();
        break;
      case OPT_BA_MEMORY: if (have_pk) decide_ba_memory(); break;
      case OPT_NEXT_KEY: case OPT_NONE: break;
    }
    return G16_OK;
  }
  // the value an option holds now, in the form g16_set_option accepts (set_option(k, get_option(k)) changes nothing)
  int get_option(const char* key, long long* out) const override {
    if (!out) return fail(G16_ERR_BAD_ARGUMENT, "null out");
    const std::string k(key ? key : "");
    const Option* o = find_option(k);
    if (!o) return fail(G16_ERR_BAD_ARGUMENT, "unknown option: " + k);
    *out = tune.*o->value;
    return G16_OK;
  }
  int get_config(g16_config* o) const override {
    if (!o) return fail(G16_ERR_BAD_ARGUMENT, "null");
    memset(o, 0, sizeof(*o));
    const MsmGeom& g1 = q[M_H].geom;
    const MsmGeom& g2 = q[M_B2].geom;
    o->c = g1.c; o->ne = g1.ne; o->copies = g1.copies;
    o->k0_g1 = g1.k0; o->k0_g2 = g2.k0;
    o->ba_rounds_g1 = g1.ba; o->ba_rounds_g2 = g2.ba;
    o->ba_m = (int32_t)tune.ba_m; o->ba_g = (int32_t)tune.ba_G; o->ba_inv_gcd = (int32_t)tune.ba_gcd; o->acc_block = (int32_t)tune.acc_block;
    o->sm_count = sm_count;
    o->world = (int32_t)world; o->rank = (int32_t)rank;
    return G16_OK;
  }
  template <class F>
  int finish_query(Query& x) {   // x.bases holds copy 0; build the other copies and the infinity mask
    const uint64_t cnt = x.hi - x.lo;
    G16_CUDA(x.mask.reserve(cnt + 16));
    G16_CUDA(msm_prepare_query<F>(S0.st_main, x.bases.template as<Affine<F>>(), (uint32_t)cnt, x.geom.copies, x.geom.c * x.geom.ne,
                                  x.mask.template as<uint8_t>()));
    return G16_OK;
  }
  A1 alpha_g1, beta_g1, delta_g1;
  A2 beta_g2, delta_g2;
  // the key points of the proof tail (batch.cuh): a_query[0] + alpha_g1, b_g1_query[0] + beta_g1, b_g2_query[0] + beta_g2
  A1 p_a, p_b;
  A2 p_2;
  // batch proving: fixed-base tables of d1, P_a, P_b (G1) and d2 (G2), built by the first g16_prove_batch under a key and
  // dropped whenever the circuit or key changes
  enum { TAB_D1 = 0, TAB_PA = 1, TAB_PB = 2, TAB_D2 = 3 };
  DevBuf tail_tab[4];
  bool tail_ready = false;
  // setup-only extras for pk_export
  A2 gamma_g2;
  DevBuf d_gamma_abc;
  bool from_setup = false;
  DevBuf full_a, full_b1, full_b2;  // setup keeps element 0 too, for export

  // ------------------------------------------------------------------
  int init(int dev) {
    device = dev;
    G16_CUDA(cudaSetDevice(dev));
    cudaDeviceProp prop;
    G16_CUDA(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9 || prop.minor != 0)
      return fail(G16_ERR_CUDA, "device is not sm_90 (this library ships sm_90a code only, for the H100)");
    sm_count = prop.multiProcessorCount;
    for (const Option& o : options()) {
      std::string var = "G16_";
      for (const char* p = o.name; *p; p++) var += (char)toupper(*p);
      const char* s = getenv(var.c_str());
      if (!s) continue;
      char* end = nullptr;
      errno = 0;
      const long long v = strtoll(s, &end, 10);
      if (end == s || *end || errno || !accepts(o, v))
        return fail(G16_ERR_BAD_ARGUMENT, var + "=\"" + s + "\" is not one of " + accepted(o));
      tune.*o.value = v;
    }
    pool.reset(new HostPool(7));
    // Stream priorities (greatest first): the witness map (H's MSM waits for it), then the G2 MSM (longest latency-bound
    // tail: its point additions cost ~3x a G1 addition), then H (starts last), then L / A / B-in-G1.  The heavy
    // accumulation kernels of the low-priority streams fill the machine while the high-priority tails trickle through.
    int prio_lo = 0, prio_hi = 0;
    G16_CUDA(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));   // lo = least priority (numerically greatest)
    auto level = [&](int k) { return std::min(prio_lo, prio_hi + k); };
    for (Slot& sl : slots) {
      G16_CUDA(cudaStreamCreateWithPriority(&sl.st_main, cudaStreamNonBlocking, level(0)));
      nvtxNameCudaStreamA(sl.st_main, SPAN_WITNESS_MAP);
      for (int i = 0; i < 5; i++) {
        const int pr = i == M_B2 ? level(1) : (i == M_H ? level(2) : prio_lo);
        G16_CUDA(cudaStreamCreateWithPriority(&sl.st_msm[i], cudaStreamNonBlocking, pr));
        nvtxNameCudaStreamA(sl.st_msm[i], span_of(i));
      }
      G16_CUDA(cudaEventCreate(&sl.ev_start));
      G16_CUDA(cudaEventCreate(&sl.ev_z));
      G16_CUDA(cudaEventCreate(&sl.ev_h));
      G16_CUDA(cudaEventCreateWithFlags(&sl.ev_bsort, cudaEventDisableTiming));
      for (int i = 0; i < 5; i++) {
        G16_CUDA(cudaEventCreate(&sl.ev_m0[i]));
        G16_CUDA(cudaEventCreate(&sl.ev_m1[i]));
        G16_CUDA(cudaEventCreate(&sl.ev_a0[i]));
        G16_CUDA(cudaEventCreate(&sl.ev_a1[i]));
      }
    }
    return G16_OK;
  }
  ~Engine() override {   // the DevBuf and MsmWorkspace members free themselves after this body, on this device
    cudaSetDevice(device);
    drop_key();   // waits for the pool tasks that read the key
    comm_release();
    pool.reset();
    cudaDeviceSynchronize();
    dom.release();
    dom_api.release();
    for (Slot& sl : slots) {
      if (sl.h_tail) cudaFreeHost(sl.h_tail);
      if (sl.h_check) cudaFreeHost(sl.h_check);
      if (sl.st_main) cudaStreamDestroy(sl.st_main);
      for (auto s : sl.st_msm) if (s) cudaStreamDestroy(s);
      auto kill = [](cudaEvent_t ev) { if (ev) cudaEventDestroy(ev); };
      kill(sl.ev_start); kill(sl.ev_z); kill(sl.ev_h); kill(sl.ev_bsort);
      for (int i = 0; i < 5; i++) { kill(sl.ev_m0[i]); kill(sl.ev_m1[i]); kill(sl.ev_a0[i]); kill(sl.ev_a1[i]); }
    }
    if (ev_batch) cudaEventDestroy(ev_batch);
  }
  int fq_limbs() const override { return NQ64; }
  int fr_limbs() const override { return FR64; }
  int g2_limbs() const override { return G2_64; }
  int partial_limbs() const override { return 4 * 2 * NQ64 + G2_64; }
  uint32_t domain_log() const override { return (uint32_t)L; }

  bool any_busy() const { return slots[0].busy || slots[1].busy; }
#define G16_NOT_BUSY() \
  if (any_busy()) return fail(G16_ERR_BAD_ARGUMENT, "a proof is in flight (g16_prove_wait / g16_prove_partial_wait it first)")

  // ---- small host helpers ----
  static Fr load_fr(const uint64_t* p) { Fr r; memcpy(r.v, p, sizeof(r.v)); return r; }
  static A1 load_a1(const uint64_t* p) { A1 r; memcpy(&r.x, p, sizeof(Fq)); memcpy(&r.y, p + NQ64, sizeof(Fq)); return r; }
  // x || y, each coordinate c0 || c1 over Fq2: exactly the packed image of A2
  static A2 load_a2(const uint64_t* p) { A2 r; memcpy(&r, p, sizeof(A2)); return r; }
  static void store_a1(uint64_t* p, const A1& a) { memcpy(p, &a.x, sizeof(Fq)); memcpy(p + NQ64, &a.y, sizeof(Fq)); }
  static void store_a2(uint64_t* p, const A2& a) { memcpy(p, &a, sizeof(A2)); }
  // Jacobian normalised to Z = 1 (identity: (1,1,0) like ark)
  template <class F, class PT>
  static void store_proj(uint64_t* p, const PT& pt) {
    Affine<F> a = pt.to_affine();
    F one = F::one(), zero = F::zero();
    const size_t w = sizeof(F) / 8;
    if (pt.is_inf()) { memcpy(p, &one, sizeof(F)); memcpy(p + w, &one, sizeof(F)); memcpy(p + 2 * w, &zero, sizeof(F)); }
    else { memcpy(p, &a.x, sizeof(F)); memcpy(p + w, &a.y, sizeof(F)); memcpy(p + 2 * w, &one, sizeof(F)); }
  }
  static void fr_to_canon(const Fr& m, uint32_t out[Fr::N]) {
    Fr c = Fr::from_mont(m);
    memcpy(out, c.v, sizeof(Fr));
  }
  static int check_log(uint32_t log_n) {
    if ((int)log_n > CP::FrP::TWO_ADICITY) return fail(G16_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "domain size exceeds the field's two-adicity (PolynomialDegreeTooLarge)");
    if (log_n > 28) return fail(G16_ERR_BAD_ARGUMENT, "log_n > 28 unsupported");
    return G16_OK;
  }

  // ---- domain + buffers ----
  int ensure_slot_buffers(Slot& sl, int Ln, uint32_t count = 1) {
    const size_t bytes = ((size_t)sizeof(Fr) << Ln) * count;
    G16_CUDA(sl.d_a.reserve(bytes)); G16_CUDA(sl.d_b.reserve(bytes)); G16_CUDA(sl.d_c.reserve(bytes));
    G16_CUDA(sl.d_t.reserve(bytes)); G16_CUDA(sl.d_h.reserve(bytes));
    return G16_OK;
  }
  int ensure_domain(NttDomain<Fr>& d, int Ln) {
    if (d.L != Ln) {
      G16_CUDA(cudaDeviceSynchronize());
      G16_CUDA(ntt_domain_build(d, Ln, S0.st_main, &ntt_launches));
      G16_CUDA(cudaStreamSynchronize(S0.st_main));
    }
    return ensure_slot_buffers(S0, Ln);
  }
  // the resident circuit's domain must be the one the prover / setup run with (plus, for CircomReduction, its table)
  int ensure_circuit_domain() {
    int rc = ensure_domain(dom, L);
    if (rc || qap != G16_QAP_CIRCOM || dom.odd_fwd_ninv) return rc;
    G16_CUDA(ntt_domain_build_odd(dom, S0.st_main, &ntt_launches));
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    return G16_OK;
  }
  // stand-alone transforms: the circuit's tables when the size matches, a separate domain otherwise
  NttDomain<Fr>* api_domain(int Ln, int* rc) {
    NttDomain<Fr>* d = (have_circuit && Ln == L) ? &dom : &dom_api;
    *rc = ensure_domain(*d, Ln);
    return d;
  }

  // one transform (ntt.cuh), counted in ntt_launches
  void ntt_any(cudaStream_t st, const NttDomain<Fr>& d, bool inverse, const Fr* src, Fr* work, Fr* dst, int load_mode, const Fr* ltab,
               const Fr* in_b, const Fr* in_c, const Fr& load_cst, int store_mode, const Fr* stab, const Fr& store_cst,
               uint32_t nvec = 1, const Fr* st_a = nullptr, const Fr* st_b = nullptr) {
    ntt_run<Fr>(st, d, inverse, src, work, dst, load_mode, ltab, in_b, in_c, load_cst, store_mode, stab, store_cst, &ntt_launches, nvec,
                st_a, st_b);
  }

  // ---- NTT API ----
  int ntt(uint32_t log_n, int inverse, int coset, uint64_t* inout) override {
    if (!inout) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    G16_NOT_BUSY();
    int rc = check_log(log_n);
    if (rc) return rc;
    G16_CUDA(cudaSetDevice(device));
    const NttDomain<Fr>& dom = *api_domain((int)log_n, &rc);   // shadows the circuit's domain on purpose
    if (rc) return rc;
    const size_t bytes = (size_t)sizeof(Fr) << log_n;
    Fr* x = S0.d_a.template as<Fr>();
    Fr* y = S0.d_t.template as<Fr>();
    G16_CUDA(cudaMemcpyAsync(x, inout, bytes, cudaMemcpyHostToDevice, S0.st_main));
    const Fr zero = Fr::zero();
    if (!inverse)
      ntt_any(S0.st_main, dom, false, x, x, y, coset ? NTT_LOAD_MUL_TABLE : NTT_LOAD_PLAIN, dom.coset_fwd, nullptr, nullptr, zero,
              NTT_STORE_PLAIN, nullptr, zero);
    else
      ntt_any(S0.st_main, dom, true, x, x, y, NTT_LOAD_PLAIN, nullptr, nullptr, nullptr, zero,
              coset ? NTT_STORE_MUL_TABLE : NTT_STORE_MUL_CONST, dom.coset_inv, dom.n_inv);
    G16_CUDA(cudaGetLastError());
    G16_CUDA(cudaMemcpyAsync(inout, y, bytes, cudaMemcpyDeviceToHost, S0.st_main));
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    return G16_OK;
  }

  // a, b, c (device, evaluations over the domain) -> S0.d_h (coefficients of h).  r1cs_to_qap.rs:201-232
  // count > 1: the witness maps of `count` proofs, vectors n apart in every buffer, one launch per pass for all of them
  void witness_map_device(Slot& sl, const NttDomain<Fr>& dom, uint32_t count = 1) {
    cudaStream_t st = sl.st_main;
    Fr* A = sl.d_a.template as<Fr>(); Fr* B = sl.d_b.template as<Fr>(); Fr* C = sl.d_c.template as<Fr>(); Fr* T = sl.d_t.template as<Fr>(); Fr* H = sl.d_h.template as<Fr>();
    const Fr zero = Fr::zero();
    for (Fr* X : {A, B, C}) {
      // domain.ifft_in_place (r1cs_to_qap.rs:201-202,220) followed by coset_domain.fft_in_place (:204-207,221): the inverse
      // transform's n^-1 and the coset pre-scaling g^i are one multiplication by the table n^-1 g^i at the second load
      ntt_any(st, dom, true, X, X, T, NTT_LOAD_PLAIN, nullptr, nullptr, nullptr, zero, NTT_STORE_PLAIN, nullptr, zero, count);
      ntt_any(st, dom, false, T, T, X, NTT_LOAD_MUL_TABLE, dom.coset_fwd_ninv, nullptr, nullptr, zero, NTT_STORE_PLAIN, nullptr, zero, count);
    }
    // (a*b - c) * Z^-1 fused into the load of coset_domain.ifft_in_place (r1cs_to_qap.rs:209,223-232)
    ntt_any(st, dom, true, A, T, H, NTT_LOAD_AB_MINUS_C, nullptr, B, C, dom.z_inv, NTT_STORE_MUL_TABLE, dom.coset_inv, zero, count);
  }

  // ark-circom's CircomReduction::witness_map_from_matrices on a, b (device row evaluations; c is not read) -> S0.d_h: the n
  // evaluations h[j] = A[j] B[j] - C[j] at the odd powers omega_2n^(2j+1), where X[j] is x's interpolant there and c = a o b.
  // Per vector: ifft, then the pre-scaling by omega_2n^i (one multiplication by n^-1 omega_2n^i at the forward load), then
  // fft.  6 transforms, no elementwise launch: c = a o b is formed by the load of c's iFFT -- first, while A and B still
  // hold the row evaluations -- and A*B - C by the last-pass store of c's forward transform.
  void witness_map_device_circom(Slot& sl, const NttDomain<Fr>& dom, uint32_t count = 1) {
    cudaStream_t st = sl.st_main;
    Fr* A = sl.d_a.template as<Fr>(); Fr* B = sl.d_b.template as<Fr>(); Fr* C = sl.d_c.template as<Fr>(); Fr* T = sl.d_t.template as<Fr>(); Fr* H = sl.d_h.template as<Fr>();
    const Fr zero = Fr::zero();
    ntt_any(st, dom, true, A, H, C, NTT_LOAD_AB, nullptr, B, nullptr, zero, NTT_STORE_PLAIN, nullptr, zero, count);
    for (Fr* X : {A, B}) {
      ntt_any(st, dom, true, X, X, T, NTT_LOAD_PLAIN, nullptr, nullptr, nullptr, zero, NTT_STORE_PLAIN, nullptr, zero, count);
      ntt_any(st, dom, false, T, T, X, NTT_LOAD_MUL_TABLE, dom.odd_fwd_ninv, nullptr, nullptr, zero, NTT_STORE_PLAIN, nullptr, zero, count);
    }
    ntt_any(st, dom, false, C, C, H, NTT_LOAD_MUL_TABLE, dom.odd_fwd_ninv, nullptr, nullptr, zero, NTT_STORE_AB_MINUS, nullptr, zero,
            count, A, B);
  }

  // The witness map of a SHARDED proof (SURVEY.md section 8e: the chains a, b, c are independent, r1cs_to_qap.rs:201-207,
  // 220-221): chain v (iFFT then coset FFT of one vector) runs on rank v mod world, the three results meet on rank
  // 3 mod world (ncclSend / ncclRecv of 32 B * n each over NVLink), which forms (a*b - c)/Z and the last coset iFFT
  // (r1cs_to_qap.rs:209,223-232), and h is broadcast to every rank for its share of the H MSM.  Per rank at most 3 of the 7
  // transforms instead of 7; everything is enqueued on the slot's main stream, no host synchronisation.
  int witness_map_split(Slot& sl) {
    NcclApi& api = nccl_api();
    cudaStream_t st = sl.st_main;
    Fr* V[3] = {sl.d_a.template as<Fr>(), sl.d_b.template as<Fr>(), sl.d_c.template as<Fr>()};
    Fr* T = sl.d_t.template as<Fr>();
    Fr* H = sl.d_h.template as<Fr>();
    const Fr zero = Fr::zero();
    const int w = (int)comm_world, me = (int)comm_rank, fin = 3 % w;
    const size_t bytes = (size_t)sizeof(Fr) << L;
    const bool circom = qap == G16_QAP_CIRCOM;
    const Fr* fwd_tab = circom ? dom.odd_fwd_ninv : dom.coset_fwd_ninv;
    // CircomReduction: chain c starts from a o b of this rank's own row evaluations, before chains a / b overwrite them
    if (circom && 2 % w == me) {
      ntt_any(st, dom, true, V[0], V[2], T, NTT_LOAD_AB, nullptr, V[1], nullptr, zero, NTT_STORE_PLAIN, nullptr, zero);
      ntt_any(st, dom, false, T, T, V[2], NTT_LOAD_MUL_TABLE, fwd_tab, nullptr, nullptr, zero, NTT_STORE_PLAIN, nullptr, zero);
    }
    for (int v = 0; v < 3; v++) {
      if (v % w != me || (circom && v == 2)) continue;
      ntt_any(st, dom, true, V[v], V[v], T, NTT_LOAD_PLAIN, nullptr, nullptr, nullptr, zero, NTT_STORE_PLAIN, nullptr, zero);
      ntt_any(st, dom, false, T, T, V[v], NTT_LOAD_MUL_TABLE, fwd_tab, nullptr, nullptr, zero, NTT_STORE_PLAIN, nullptr, zero);
    }
    int rc = api.GroupStart();
    for (int v = 0; v < 3 && rc == 0; v++) {
      const int src = v % w;
      if (src == fin) continue;
      if (me == src) rc = api.Send(V[v], bytes, /*ncclUint8*/ 1, fin, nccl_comm_wm, st);
      if (me == fin && rc == 0) rc = api.Recv(V[v], bytes, 1, src, nccl_comm_wm, st);
    }
    if (rc == 0) rc = api.GroupEnd(); else api.GroupEnd();
    if (rc != 0) return fail(G16_ERR_CUDA, std::string("witness-map exchange (ncclSend/Recv): ") + api.GetErrorString(rc));
    if (me == fin && circom) {
      ntt_ab_minus_c<Fr>(st, V[0], V[1], V[2], H, 1ull << L);
      ntt_launches++;
    } else if (me == fin) {
      ntt_any(st, dom, true, V[0], T, H, NTT_LOAD_AB_MINUS_C, nullptr, V[1], V[2], dom.z_inv, NTT_STORE_MUL_TABLE, dom.coset_inv, zero);
    }
    rc = api.Broadcast(H, H, bytes, 1, fin, nccl_comm_wm, st);
    if (rc != 0) return fail(G16_ERR_CUDA, std::string("witness-map broadcast (ncclBroadcast): ") + api.GetErrorString(rc));
    return G16_OK;
  }

  int witness_map_evals(uint32_t log_n, const uint64_t* a, const uint64_t* b, const uint64_t* c, uint64_t* h) override {
    if (!a || !b || !c || !h) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    G16_NOT_BUSY();
    int rc = check_log(log_n);
    if (rc) return rc;
    G16_CUDA(cudaSetDevice(device));
    const NttDomain<Fr>* d = api_domain((int)log_n, &rc);
    if (rc) return rc;
    const size_t bytes = (size_t)sizeof(Fr) << log_n;
    G16_CUDA(cudaMemcpyAsync(S0.d_a.p, a, bytes, cudaMemcpyHostToDevice, S0.st_main));
    G16_CUDA(cudaMemcpyAsync(S0.d_b.p, b, bytes, cudaMemcpyHostToDevice, S0.st_main));
    G16_CUDA(cudaMemcpyAsync(S0.d_c.p, c, bytes, cudaMemcpyHostToDevice, S0.st_main));
    witness_map_device(S0, *d);
    G16_CUDA(cudaGetLastError());
    G16_CUDA(cudaMemcpyAsync(h, S0.d_h.p, bytes, cudaMemcpyDeviceToHost, S0.st_main));
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    return G16_OK;
  }

  // ---- stand-alone MSM API (msm_bigint) ----
  template <class F, class WS>
  int msm_host(WS& ws, bool g2, const uint64_t* bases, const uint64_t* scalars, uint64_t n, uint64_t* out) {
    if (!out || (n && (!bases || !scalars))) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    if (n >= (1ull << 27)) return fail(G16_ERR_BAD_ARGUMENT, "n too large");
    G16_NOT_BUSY();
    G16_CUDA(cudaSetDevice(device));
    XYZZ<F> res = XYZZ<F>::inf();
    if (n) {
      DevBuf db, ds, dm;
      G16_CUDA(db.reserve(n * sizeof(Affine<F>)));
      G16_CUDA(ds.reserve(n * sizeof(Fr)));
      G16_CUDA(dm.reserve(n));
      G16_CUDA(cudaMemcpyAsync(db.p, bases, n * sizeof(Affine<F>), cudaMemcpyHostToDevice, S0.st_main));
      G16_CUDA(cudaMemcpyAsync(ds.p, scalars, n * sizeof(Fr), cudaMemcpyHostToDevice, S0.st_main));
      G16_CUDA(msm_prepare_query<F>(S0.st_main, db.template as<Affine<F>>(), (uint32_t)n, 1, 0, dm.template as<uint8_t>()));
      const MsmGeom g = with_k0(msm_geom(n, FR_BITS, (int)tune.c, 0), g2);   // caller-supplied bases: no precomputed copies
      G16_CUDA((msm_enqueue<F, Fr>(S0.st_main, ws, g, db.template as<Affine<F>>(), dm.template as<uint8_t>(), ds.template as<uint32_t>(), 1, false, &ctr, nullptr, nullptr, nullptr, nullptr, nullptr, 0)));
      G16_CUDA(cudaStreamSynchronize(S0.st_main));
      res = msm_finish<F>(ws, g);
    }
    store_proj<F>(out, res);
    return G16_OK;
  }
  int msm_g1(const uint64_t* bases, const uint64_t* scalars, uint64_t n, uint64_t* out) override { return msm_host<Fq>(S0.ws1[0], false, bases, scalars, n, out); }
  int msm_g2(const uint64_t* bases, const uint64_t* scalars, uint64_t n, uint64_t* out) override { return msm_host<Fq2>(S0.ws2, true, bases, scalars, n, out); }

  // ---- circuit ----
  int circuit_load(int qp, uint32_t ni, uint32_t nc, uint32_t nw, const g16_csr* a, const g16_csr* b, const g16_csr* c) override {
    if (qp != G16_QAP_LIBSNARK && qp != G16_QAP_CIRCOM) return fail(G16_ERR_BAD_ARGUMENT, "unknown R1CS-to-QAP reduction");
    if (!a || !b || !c || ni == 0) return fail(G16_ERR_BAD_ARGUMENT, "bad circuit description");
    G16_NOT_BUSY();
    uint64_t need = (uint64_t)nc + ni;
    int Ln = 0;
    while ((1ull << Ln) < need) Ln++;
    int rc = check_log((uint32_t)Ln);
    if (rc) return rc;
    // CircomReduction evaluates at the odd powers of omega_2n: the domain of size 2n must exist
    if (qp == G16_QAP_CIRCOM && Ln + 1 > CP::FrP::TWO_ADICITY)
      return fail(G16_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "CircomReduction needs a domain of twice the size, which exceeds the field's two-adicity (PolynomialDegreeTooLarge)");
    G16_CUDA(cudaSetDevice(device));
    const g16_csr* ms[3] = {a, b, c};
    const uint32_t nvars = ni + nw;
    for (const g16_csr* x : ms) {   // all three matrices pass before the resident circuit is touched
      if (!x->row_ptr) return fail(G16_ERR_BAD_ARGUMENT, "null row_ptr");
      if (x->row_ptr[0] != 0) return fail(G16_ERR_BAD_ARGUMENT, "row_ptr[0] must be 0");
      for (uint32_t i = 0; i < nc; i++)
        if (x->row_ptr[i + 1] < x->row_ptr[i]) return fail(G16_ERR_BAD_ARGUMENT, "row_ptr must be non-decreasing");
      const uint32_t nnz = x->row_ptr[nc];
      if (nnz && (!x->col || !x->val)) return fail(G16_ERR_BAD_ARGUMENT, "null col/val");
      for (uint32_t e = 0; e < nnz; e++) if (x->col[e] >= nvars) return fail(G16_ERR_BAD_ARGUMENT, "column index out of range");
    }
    drop_key();
    have_circuit = false;
    circuit_without_c = false;
    for (int m = 0; m < 3; m++) {
      const uint32_t nnz = ms[m]->row_ptr[nc];
      h_rp[m].assign(ms[m]->row_ptr, ms[m]->row_ptr + nc + 1);
      h_col[m].assign(ms[m]->col, ms[m]->col + nnz);
      h_val[m].resize(nnz);
      if (nnz) memcpy(h_val[m].data(), ms[m]->val, (size_t)nnz * sizeof(Fr));
      G16_CUDA(csr_rp[m].reserve((size_t)(nc + 1) * 4));
      G16_CUDA(csr_col[m].reserve((size_t)nnz * 4 + 4));
      G16_CUDA(csr_val[m].reserve((size_t)nnz * sizeof(Fr) + sizeof(Fr)));
      G16_CUDA(cudaMemcpy(csr_rp[m].p, ms[m]->row_ptr, (size_t)(nc + 1) * 4, cudaMemcpyHostToDevice));
      if (nnz) {
        G16_CUDA(cudaMemcpy(csr_col[m].p, ms[m]->col, (size_t)nnz * 4, cudaMemcpyHostToDevice));
        G16_CUDA(cudaMemcpy(csr_val[m].p, ms[m]->val, (size_t)nnz * sizeof(Fr), cudaMemcpyHostToDevice));
      }
    }
    num_inputs = ni; num_constraints = nc; num_witness = nw; L = Ln; qap = qp;
    G16_CUDA(S0.d_z.reserve((size_t)nvars * sizeof(Fr)));
    if ((rc = ensure_circuit_domain())) return rc;
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    have_circuit = true;
    return G16_OK;
  }

  // ---- proving key ----
  // A key is made resident in three steps, by g16_pk_load, g16_setup and g16_pk_load_serialized alike: begin_key checks
  // the query lengths and only then drops the old key and reserves the new bases, the loader fills copy 0 of every query
  // and sets the single points, commit_key finishes the queries and marks the key resident.  A failure between the two
  // leaves no key resident.
  //
  // The only place the resident key and everything derived from it are dropped.  Waits first for the pool tasks that read
  // the key points: the key products of g16_prove_assemble_prepare and of a slot's proof (also after a failed submit).
  void drop_key() {
    for (Slot& sl : slots)
      for (auto* h : {&sl.helper, &sl.helper2})
        if (*h) { (*h)->wait(); h->reset(); }
    if (asm_helper) { asm_helper->wait(); asm_helper.reset(); }
    have_pk = from_setup = tail_ready = asm_valid = share_b_sort = false;
  }
  Shard shard(uint64_t pairs, uint32_t rk, uint32_t wd, bool g2) const {
    // Interleaved (strided) split: rank k owns pairs k, k + world, ...  Contiguous ranges would be badly unbalanced
    // whenever the density of a query varies with the variable index (early variables of a circuit are used more often).
    const uint64_t cnt = pairs > rk ? (pairs - rk + wd - 1) / wd : 0;
    return Shard{pairs, rk, rk + cnt, with_k0(pick_geom(cnt), g2)};
  }
  // sorted entries carry (copy * n + index) in 31 bits and offsets are 32-bit
  static bool geom_fits(const Shard& x) {
    return (uint64_t)x.geom.copies * (x.hi - x.lo) < (1ull << 31) && x.geom.max_entries < (1ull << 32);
  }
  // len: the raw lengths of the H, L, A, B1 and B2 queries (element 0 of A, B1 and B2 included).  Returns with nothing
  // changed when the key cannot be made resident.
  int begin_key(uint32_t rk, uint32_t wd, const uint64_t len[5]) {
    if (len[M_A] < 1 || len[M_B1] < 1 || len[M_B2] < 1)
      return fail(G16_ERR_MALFORMED_KEY, "a/b queries must hold at least the constant-one base");
    // msm_bigint truncates to the shorter operand (SURVEY.md section 2a; relied upon at prover.rs:66)
    const uint64_t nz1 = nvars() - 1;   // |input_assignment ++ aux_assignment|, prover.rs:85
    const uint64_t pairs[5] = {std::min<uint64_t>(len[M_H], 1ull << L), std::min<uint64_t>(len[M_L], num_witness),
                               std::min(len[M_A] - 1, nz1), std::min(len[M_B1] - 1, nz1), std::min(len[M_B2] - 1, nz1)};
    Shard sh[5];
    for (int m = 0; m < 5; m++) {
      sh[m] = shard(pairs[m], rk, wd, m == M_B2);
      if (!geom_fits(sh[m])) return fail(G16_ERR_BAD_ARGUMENT, "query too large for one GPU: shard it (world > 1) or raise G16_MSM_NE");
    }
    drop_key();
    rank = rk; world = wd;
    for (int m = 0; m < 5; m++) {
      static_cast<Shard&>(q[m]) = sh[m];
      const size_t esz = m == M_B2 ? sizeof(A2) : sizeof(A1);
      G16_CUDA(q[m].bases.reserve((size_t)q[m].geom.copies * (q[m].hi - q[m].lo) * esz + 16));
    }
    return G16_OK;
  }
  // The only place a key becomes resident: copy 0 of every query's bases and alpha_g1, beta_g1, beta_g2 are in place.
  int commit_key(const A1& a_q0, const A1& b1_q0, const A2& b2_q0, bool setup_key) {
    int rc;
    for (int m = 0; m < 5; m++)
      if ((rc = (m == M_B2) ? finish_query<Fq2>(q[m]) : finish_query<Fq>(q[m]))) return rc;
    set_tail_points(a_q0, b1_q0, b2_q0);
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    if ((rc = decide_b_sort_sharing())) return rc;
    decide_ba_memory();
    have_pk = true;
    from_setup = setup_key;
    return G16_OK;
  }
  template <class F>
  int upload_query(Query& x, const uint64_t* host_full, uint64_t skip_first) {
    using AT = Affine<F>;
    const uint64_t cnt = x.hi - x.lo;
    if (cnt) {
      const size_t limbs = sizeof(AT) / 8;
      // gather every world-th point of the full host array
      G16_CUDA(cudaMemcpy2DAsync(x.bases.p, sizeof(AT), host_full + (skip_first + x.lo) * limbs, (size_t)world * sizeof(AT), sizeof(AT), cnt,
                                 cudaMemcpyHostToDevice, S0.st_main));
    }
    return G16_OK;
  }
  uint64_t nvars() const { return (uint64_t)num_inputs + num_witness; }
  // H query length of the resident circuit's keys: n - 1 points, n under CircomReduction
  uint64_t h_query_len() const { return qap == G16_QAP_CIRCOM ? 1ull << L : (1ull << L) - 1; }
  // a_q0, b1_q0, b2_q0: element 0 of a_query, b_g1_query, b_g2_query; alpha_g1, beta_g1, beta_g2 already set
  void set_tail_points(const A1& a_q0, const A1& b1_q0, const A2& b2_q0) {
    P1 pa = P1::from_affine(a_q0), pb = P1::from_affine(b1_q0);
    P2 p2 = P2::from_affine(b2_q0);
    pa.madd(alpha_g1);
    pb.madd(beta_g1);
    p2.madd(beta_g2);
    p_a = pa.to_affine();
    p_b = pb.to_affine();
    p_2 = p2.to_affine();
  }
  int pk_load(const g16_pk_desc* pk, uint32_t rk, uint32_t wd) override {
    if (!have_circuit) return fail(G16_ERR_BAD_ARGUMENT, "g16_circuit_load must precede g16_pk_load");
    if (!pk || wd == 0 || rk >= wd) return fail(G16_ERR_BAD_ARGUMENT, "bad pk / rank / world");
    G16_NOT_BUSY();
    if (!pk->a_query || !pk->b_g1_query || !pk->b_g2_query || !pk->alpha_g1 || !pk->beta_g1 || !pk->delta_g1 || !pk->beta_g2 || !pk->delta_g2)
      return fail(G16_ERR_BAD_ARGUMENT, "null pk member");
    if ((pk->h_len && !pk->h_query) || (pk->l_len && !pk->l_query)) return fail(G16_ERR_BAD_ARGUMENT, "null h/l query");
    G16_CUDA(cudaSetDevice(device));
    const uint64_t len[5] = {pk->h_len, pk->l_len, pk->a_len, pk->b_g1_len, pk->b_g2_len};
    int rc = begin_key(rk, wd, len);
    if (rc) return rc;
    if ((rc = upload_query<Fq>(q[M_H], pk->h_query, 0))) return rc;
    if ((rc = upload_query<Fq>(q[M_L], pk->l_query, 0))) return rc;
    if ((rc = upload_query<Fq>(q[M_A], pk->a_query, 1))) return rc;
    if ((rc = upload_query<Fq>(q[M_B1], pk->b_g1_query, 1))) return rc;
    if ((rc = upload_query<Fq2>(q[M_B2], pk->b_g2_query, 1))) return rc;
    alpha_g1 = load_a1(pk->alpha_g1); beta_g1 = load_a1(pk->beta_g1); delta_g1 = load_a1(pk->delta_g1);
    beta_g2 = load_a2(pk->beta_g2); delta_g2 = load_a2(pk->delta_g2);
    return commit_key(load_a1(pk->a_query), load_a1(pk->b_g1_query), load_a2(pk->b_g2_query), false);
  }

  // ---- setup (generator.rs:47-208) ----
  template <class F>
  int batch_mul(const Affine<F>& gen, const Fr* d_scalars, uint64_t cnt, Affine<F>* d_out, DevBuf& table) {
    G16_CUDA(table.reserve((size_t)fb_windows<Fr>() * 255 * sizeof(XYZZ<F>)));
    G16_CUDA((fb_batch_mul<F, Fr>(S0.st_main, gen, d_scalars, cnt, d_out, table.template as<XYZZ<F>>())));
    return G16_OK;
  }
  int setup(const uint64_t* alpha_, const uint64_t* beta_, const uint64_t* gamma_, const uint64_t* delta_,
            const uint64_t* tau_, const uint64_t* g1_, const uint64_t* g2_) override {
    if (!have_circuit) return fail(G16_ERR_BAD_ARGUMENT, "g16_circuit_load must precede g16_setup");
    if (!alpha_ || !beta_ || !gamma_ || !delta_ || !tau_ || !g1_ || !g2_) return fail(G16_ERR_BAD_ARGUMENT, "null argument");
    G16_NOT_BUSY();
    G16_CUDA(cudaSetDevice(device));
    const Fr alpha = load_fr(alpha_), beta = load_fr(beta_), gamma = load_fr(gamma_), delta = load_fr(delta_), tau = load_fr(tau_);
    const A1 g1 = load_a1(g1_);
    const A2 g2 = load_a2(g2_);
    if (gamma.is_zero() || delta.is_zero()) return fail(G16_ERR_BAD_ARGUMENT, "gamma/delta must be invertible (UnexpectedIdentity)");
    { int rc0 = ensure_circuit_domain(); if (rc0) return rc0; }   // dom.omega / dom.n_inv below are the circuit's
    const uint64_t n = 1ull << L;
    const uint32_t nc = num_constraints, ni = num_inputs;
    const uint64_t nv = nvars();
    // --- instance_map_with_evaluation (r1cs_to_qap.rs:128-170) on the host ---
    Fr tn = tau;
    for (int i = 0; i < L; i++) tn = Fr::sqr(tn);
    const Fr zt = Fr::sub(tn, Fr::one());                      // evaluate_vanishing_polynomial(t)
    if (zt.is_zero()) return fail(G16_ERR_BAD_ARGUMENT, "tau lies in the evaluation domain");
    const bool circom = qap == G16_QAP_CIRCOM;
    if (circom && Fr::sqr(tn) == Fr::one()) return fail(G16_ERR_BAD_ARGUMENT, "tau lies in the domain of size 2n (CircomReduction)");
    // Lagrange coefficients u_i = zt * w^i / (n (tau - w^i))   (evaluate_all_lagrange_coefficients)
    std::vector<Fr> u(n), den(n);
    {
      Fr w = Fr::one();
      for (uint64_t i = 0; i < n; i++) { den[i] = Fr::sub(tau, w); w = Fr::mul(w, dom.omega); }
      // batch inversion
      std::vector<Fr> pref(n);
      Fr acc = Fr::one();
      for (uint64_t i = 0; i < n; i++) { pref[i] = acc; acc = Fr::mul(acc, den[i]); }
      Fr ai = Fr::inv(acc);
      for (uint64_t i = n; i-- > 0;) { Fr t = Fr::mul(ai, pref[i]); ai = Fr::mul(ai, den[i]); den[i] = t; }
      const Fr zn = Fr::mul(zt, dom.n_inv);
      w = Fr::one();
      for (uint64_t i = 0; i < n; i++) { u[i] = Fr::mul(Fr::mul(zn, w), den[i]); w = Fr::mul(w, dom.omega); }
    }
    std::vector<Fr> qa(nv, Fr::zero()), qb(nv, Fr::zero()), qc(nv, Fr::zero());
    for (uint32_t i = 0; i < ni; i++) qa[i] = u[nc + i];                         // r1cs_to_qap.rs:150-155
    std::vector<Fr>* outs[3] = {&qa, &qb, &qc};
    for (int m = 0; m < 3; m++)
      for (uint32_t i = 0; i < nc; i++)
        for (uint32_t e = h_rp[m][i]; e < h_rp[m][i + 1]; e++) {
          Fr& dst = (*outs[m])[h_col[m][e]];
          dst = Fr::add(dst, Fr::mul(u[i], h_val[m][e]));                          // r1cs_to_qap.rs:157-167
        }
    const Fr gi = Fr::inv(gamma), di = Fr::inv(delta);
    const uint64_t hn = h_query_len();
    std::vector<Fr> gabc(ni), lq(num_witness), hs(hn);
    for (uint64_t i = 0; i < nv; i++) {
      const Fr t = Fr::add(Fr::add(Fr::mul(beta, qa[i]), Fr::mul(alpha, qb[i])), qc[i]);
      if (i < ni) gabc[i] = Fr::mul(t, gi);                                        // generator.rs:113-117
      else lq[i - ni] = Fr::mul(t, di);                                            // generator.rs:119-123
    }
    if (!circom) {
      Fr p = Fr::mul(zt, di);                                                      // h_query_scalars, r1cs_to_qap.rs:237-247
      for (uint64_t i = 0; i + 1 < n; i++) { hs[i] = p; p = Fr::mul(p, tau); }
    } else {
      circom_h_scalars(tau, tn, di, hs);
    }
    // --- fixed-base batch multiplications on the GPU (generator.rs:129-183) ---
    const uint64_t len[5] = {hn, num_witness, nv, nv, nv};
    int rc = begin_key(0, 1, len);
    if (rc) return rc;
    {   // the scalars and tables are freed before commit_key weighs the free memory
      DevBuf d_s, tab1, tab2;
      G16_CUDA(d_s.reserve(std::max<uint64_t>(nv, n) * sizeof(Fr)));
      auto up = [&](const std::vector<Fr>& v) -> cudaError_t {
        return v.empty() ? cudaSuccess : cudaMemcpyAsync(d_s.p, v.data(), v.size() * sizeof(Fr), cudaMemcpyHostToDevice, S0.st_main);
      };
      G16_CUDA(full_a.reserve(nv * sizeof(A1))); G16_CUDA(full_b1.reserve(nv * sizeof(A1))); G16_CUDA(full_b2.reserve(nv * sizeof(A2)));
      G16_CUDA(d_gamma_abc.reserve((size_t)ni * sizeof(A1)));
      // a_query / b_g1_query / b_g2_query
      G16_CUDA(up(qa)); if ((rc = batch_mul<Fq>(g1, d_s.template as<Fr>(), nv, full_a.template as<A1>(), tab1))) return rc;
      G16_CUDA(cudaStreamSynchronize(S0.st_main));
      G16_CUDA(up(qb)); if ((rc = batch_mul<Fq>(g1, d_s.template as<Fr>(), nv, full_b1.template as<A1>(), tab1))) return rc;
      if ((rc = batch_mul<Fq2>(g2, d_s.template as<Fr>(), nv, full_b2.template as<A2>(), tab2))) return rc;
      G16_CUDA(cudaStreamSynchronize(S0.st_main));
      G16_CUDA(up(hs)); if ((rc = batch_mul<Fq>(g1, d_s.template as<Fr>(), hn, q[M_H].bases.template as<A1>(), tab1))) return rc;
      G16_CUDA(cudaStreamSynchronize(S0.st_main));
      G16_CUDA(up(lq)); if ((rc = batch_mul<Fq>(g1, d_s.template as<Fr>(), num_witness, q[M_L].bases.template as<A1>(), tab1))) return rc;
      G16_CUDA(cudaStreamSynchronize(S0.st_main));
      G16_CUDA(up(gabc)); if ((rc = batch_mul<Fq>(g1, d_s.template as<Fr>(), ni, d_gamma_abc.template as<A1>(), tab1))) return rc;
      G16_CUDA(cudaStreamSynchronize(S0.st_main));
    }
    // single points on the host (generator.rs:147-151,182)
    uint32_t k[Fr::N];
    auto mul1 = [&](const Fr& s) { fr_to_canon(s, k); return P1::from_affine(g1).mul_u32(k, Fr::N).to_affine(); };
    auto mul2 = [&](const Fr& s) { fr_to_canon(s, k); return P2::from_affine(g2).mul_u32(k, Fr::N).to_affine(); };
    alpha_g1 = mul1(alpha); beta_g1 = mul1(beta); delta_g1 = mul1(delta);
    beta_g2 = mul2(beta); gamma_g2 = mul2(gamma); delta_g2 = mul2(delta);
    return commit_setup_key();
  }
  // The last step of every key this library derives itself (g16_setup, g16_setup_from_srs, g16_setup_contribute): full_a,
  // full_b1, full_b2, d_gamma_abc, copy 0 of the H and L bases and the single points are in place.  Copies the MSM views
  // query[1..] of A and B and commits the key.
  int commit_setup_key() {
    const uint64_t nv = nvars();
    auto view = [&](Query& x, const DevBuf& full, size_t esz) {
      return nv > 1 ? cudaMemcpyAsync(x.bases.p, (char*)full.p + esz, (nv - 1) * esz, cudaMemcpyDeviceToDevice, S0.st_main) : cudaSuccess;
    };
    G16_CUDA(view(q[M_A], full_a, sizeof(A1)));
    G16_CUDA(view(q[M_B1], full_b1, sizeof(A1)));
    G16_CUDA(view(q[M_B2], full_b2, sizeof(A2)));
    A1 a_q0, b1_q0;
    A2 b2_q0;
    G16_CUDA(cudaMemcpyAsync(&a_q0, full_a.p, sizeof(A1), cudaMemcpyDeviceToHost, S0.st_main));
    G16_CUDA(cudaMemcpyAsync(&b1_q0, full_b1.p, sizeof(A1), cudaMemcpyDeviceToHost, S0.st_main));
    G16_CUDA(cudaMemcpyAsync(&b2_q0, full_b2.p, sizeof(A2), cudaMemcpyDeviceToHost, S0.st_main));
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    return commit_key(a_q0, b1_q0, b2_q0, true);
  }

  // ---- proving keys from a powers-of-tau transcript (srs.cuh) ----
  enum { SRS_TAU_G1 = 0, SRS_TAU_G2, SRS_ALPHA, SRS_BETA, SRS_BETA_G2, SRS_MEMBERS };
  static const char* srs_member(int m) {
    static const char* t[SRS_MEMBERS] = {"tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1", "beta_g2"};
    return t[m];
  }
  // The Lagrange members of g16_setup_from_lagrange, uploaded after the transcript's: member SRS_MEMBERS + k of the error word
  enum { LAG_TAU_G1 = 0, LAG_TAU_G2, LAG_ALPHA, LAG_BETA, LAG_H, LAG_MEMBERS };
  static const char* lag_member(int k) {
    static const char* t[LAG_MEMBERS] = {"tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1", "tau_g1_h"};
    return t[k];
  }
  // Stage times of the last g16_setup_from_srs (host clock around work that ends in a stream synchronise), read by
  // tools/bench_srs_setup.py through g16_get_timings: h2d_ms = upload and point checks, witness_map_ms = the group inverse
  // transforms, msm_ms[0] = the H query, msm_ms[1] = the sparse sums, total_ms = the whole call.
  int setup_from_srs(const g16_srs_desc* srs, uint32_t flags) override { return setup_from_transcript(srs, nullptr, nullptr, flags); }
  // g16_setup_from_lagrange: setup_from_transcript with the Lagrange points taken from `lag` after the combination check;
  // witness_map_ms = that check.
  int setup_from_lagrange(const g16_srs_desc* srs, const g16_lagrange_desc* lag, const uint64_t* rho, uint32_t flags) override {
    if (!lag) return fail(G16_ERR_BAD_ARGUMENT, "null lag");
    if (!rho) return fail(G16_ERR_BAD_ARGUMENT, "null rho");
    return setup_from_transcript(srs, lag, rho, flags);
  }
  // The key of the resident circuit from a transcript: the Lagrange points [L_i], [alpha L_i], [beta L_i] (G1) and [L_i]
  // (G2) are the group inverse transforms of the transcript's first n powers (lag == nullptr), or lag's points once the
  // combination check accepted them; under CircomReduction lag's tau_g1_h is the H query.  Everything else is shared.
  int setup_from_transcript(const g16_srs_desc* srs, const g16_lagrange_desc* lag, const uint64_t* rho_, uint32_t flags) {
    const char* who = lag ? "g16_setup_from_lagrange" : "g16_setup_from_srs";
    if (!have_circuit) return fail(G16_ERR_BAD_ARGUMENT, std::string("g16_circuit_load must precede ") + who);
    if (!srs) return fail(G16_ERR_BAD_ARGUMENT, "null srs");
    if (flags & ~(uint32_t)G16_SER_VALIDATE) return fail(G16_ERR_BAD_ARGUMENT, std::string(who) + " takes 0 or G16_SER_VALIDATE");
    G16_NOT_BUSY();
    const uint64_t n = 1ull << L;
    const uint64_t* ptr[SRS_MEMBERS] = {srs->tau_g1, srs->tau_g2, srs->alpha_tau_g1, srs->beta_tau_g1, srs->beta_g2};
    const uint64_t have[SRS_MEMBERS] = {srs->tau_g1_len, srs->tau_g2_len, srs->alpha_tau_g1_len, srs->beta_tau_g1_len, 1};
    const bool circom = qap == G16_QAP_CIRCOM;
    // lag's H points over 2n powers (an interior level of a .ptau's section 12): their check and correction read tau^(2n-1)
    const bool h2n = lag && circom && lag->h_over_2n;
    const uint64_t need[SRS_MEMBERS] = {2 * n - 1 + h2n, n, n, n, 1};
    for (int m = 0; m < SRS_MEMBERS; m++) {
      if (!ptr[m]) return fail(G16_ERR_BAD_ARGUMENT, std::string("null srs member ") + srs_member(m));
      if (have[m] < need[m])
        return fail(G16_ERR_BAD_ARGUMENT, std::string(srs_member(m)) + " holds " + std::to_string(have[m]) +
                                              " points, the circuit (domain 2^" + std::to_string(L) + ") needs at least " +
                                              std::to_string(need[m]) + (h2n ? " (lag.h_over_2n)" : ""));
    }
    const uint64_t* lptr[LAG_MEMBERS] = {};
    Fr rho = Fr::zero();
    if (lag) {
      if (lag->log_n != (uint32_t)L)
        return fail(G16_ERR_BAD_ARGUMENT, "lag.log_n = " + std::to_string(lag->log_n) + ", the circuit's domain is 2^" + std::to_string(L));
      const uint64_t* p[LAG_MEMBERS] = {lag->tau_g1, lag->tau_g2, lag->alpha_tau_g1, lag->beta_tau_g1, lag->tau_g1_h};
      for (int k = 0; k < LAG_MEMBERS; k++) {
        if (k == LAG_H && !circom) continue;   // LibsnarkReduction's H comes from tau_g1
        if (!p[k]) return fail(G16_ERR_BAD_ARGUMENT, std::string("null lag member ") + lag_member(k));
        lptr[k] = p[k];
      }
      rho = load_fr(rho_);
      if (rho.is_zero()) return fail(G16_ERR_BAD_ARGUMENT, "the challenge rho must be non-zero");
    }
    G16_CUDA(cudaSetDevice(device));
    int rc = ensure_circuit_domain();   // dom.n_inv
    if (rc) return rc;
    const auto t0 = std::chrono::steady_clock::now();
    auto ms_since = [](std::chrono::steady_clock::time_point a) {
      return (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count();
    };
    tm = g16_timings{};
    const uint32_t nc = num_constraints, ni = num_inputs, nw = num_witness;
    const uint64_t nv = nvars(), hn = h_query_len();
    const uint64_t len[5] = {hn, nw, nv, nv, nv};
    if ((rc = begin_key(0, 1, len))) return rc;   // from here on a failure leaves no key resident
    G16_CUDA(full_a.reserve(nv * sizeof(A1))); G16_CUDA(full_b1.reserve(nv * sizeof(A1))); G16_CUDA(full_b2.reserve(nv * sizeof(A2)));
    G16_CUDA(d_gamma_abc.reserve((size_t)ni * sizeof(A1)));
    cudaStream_t st = S0.st_main;
    {   // transcript buffers and scratch are freed before commit_key weighs the free memory
      // --- upload and check the prefixes, then lag's members (n points each) ---
      DevBuf up[SRS_MEMBERS], lup[LAG_MEMBERS], err;
      G16_CUDA(err.reserve(8));
      G16_CUDA(cudaMemsetAsync(err.p, 0xff, 8, st));
      auto upload_check = [&](DevBuf& d, const uint64_t* src, uint64_t cnt, bool g2, uint32_t member) -> cudaError_t {
        const size_t bytes = cnt * (g2 ? sizeof(A2) : sizeof(A1));
        cudaError_t x = d.reserve(bytes);
        if (x == cudaSuccess) x = cudaMemcpyAsync(d.p, src, bytes, cudaMemcpyHostToDevice, st);
        if (x != cudaSuccess) return x;
        return g2 ? srs_check<CP, true>(st, d.p, (uint32_t)cnt, flags, member, err.template as<unsigned long long>())
                  : srs_check<CP, false>(st, d.p, (uint32_t)cnt, flags, member, err.template as<unsigned long long>());
      };
      for (int m = 0; m < SRS_MEMBERS; m++) G16_CUDA(upload_check(up[m], ptr[m], need[m], m == SRS_TAU_G2 || m == SRS_BETA_G2, m));
      for (int k = 0; k < LAG_MEMBERS; k++)
        if (lptr[k]) G16_CUDA(upload_check(lup[k], lptr[k], n, k == LAG_TAU_G2, SRS_MEMBERS + k));
      unsigned long long first_err = 0;
      G16_CUDA(cudaMemcpyAsync(&first_err, err.p, 8, cudaMemcpyDeviceToHost, st));
      G16_CUDA(cudaStreamSynchronize(st));
      if (first_err != ~0ull) {
        const int m = (int)(first_err >> 48);
        return fail(G16_ERR_INVALID_DATA, (m < SRS_MEMBERS ? std::string(srs_member(m)) : std::string("lagrange.") + lag_member(m - SRS_MEMBERS)) +
                                              "[" + std::to_string((first_err >> 8) & ((1ull << 40) - 1)) + "]: " +
                                              ser_reason(first_err & 0xff));
      }
      tm.h2d_ms = ms_since(t0);
      auto t1 = std::chrono::steady_clock::now();
      if (lag) {
        if ((rc = lagrange_check(up, lup, rho, h2n))) return rc;
        tm.witness_map_ms = ms_since(t1);
        t1 = std::chrono::steady_clock::now();
      }
      // --- H query: [tau^(n+i)] - [tau^i] (LibsnarkReduction), or the odd entries of the size-2n inverse transform of
      // [tau^i], i < 2n - 1: 1/(2n) times the size-n transform of omega_2n^-i ([tau^i] - [tau^(i+n)]) (CircomReduction),
      // which lag's tau_g1_h holds (with h2n: plus (omega_2n^(2i+1) / 2n) [tau^(2n-1)], taken off here) ---
      const A1* t1p = up[SRS_TAU_G1].template as<A1>();
      DevBuf hpts, dfr, dtw;
      // the transforms' scalars (srs_ifft): tw[b] = omega_n^-(2^b), tw[32] = n^-1
      Fr tw[33];
      tw[0] = Fr::inv(fr_domain_root<Fr>(L));
      for (int b = 1; b < 32; b++) tw[b] = Fr::sqr(tw[b - 1]);
      tw[32] = dom.n_inv;
      if (!lag) {
        G16_CUDA(dfr.reserve(n * sizeof(Fr)));
        G16_CUDA(dtw.reserve(sizeof(tw)));
        G16_CUDA(cudaMemcpyAsync(dtw.p, tw, sizeof(tw), cudaMemcpyHostToDevice, st));
      }
      const Fr* dtab = dtw.template as<Fr>();
      if (lptr[LAG_H] && !h2n) {
        G16_CUDA(cudaMemcpyAsync(q[M_H].bases.p, lup[LAG_H].p, n * sizeof(A1), cudaMemcpyDeviceToDevice, st));
      } else if (lptr[LAG_H]) {
        if ((rc = lagrange_h_correct(lup[LAG_H].template as<A1>(), t1p + (2 * n - 1)))) return rc;
      } else {
        G16_CUDA(hpts.reserve(n * sizeof(P1)));
        if (!circom) {
          G16_CUDA(srs_diff<Fq>(st, t1p, (uint32_t)(2 * n - 1), (uint32_t)n, 0, (uint32_t)(n - 1), hpts.template as<P1>()));
          G16_CUDA(srs_affine<Fq>(st, hpts.template as<P1>(), (uint32_t)hn, q[M_H].bases.template as<A1>()));
        } else {   // s_j = omega_2n^-j / 2n on [tau^j] - [tau^(j+n)], transformed straight into the H query's bases (hn = n)
          std::vector<Fr> s(n);
          const Fr w_inv = Fr::inv(fr_domain_root<Fr>(L + 1));
          Fr c = Fr::inv(fr_from_u64<Fr>(2 * n));
          for (uint64_t i = 0; i < n; i++) { s[i] = c; c = Fr::mul(c, w_inv); }
          G16_CUDA(cudaMemcpyAsync(dfr.p, s.data(), n * sizeof(Fr), cudaMemcpyHostToDevice, st));
          G16_CUDA((srs_ifft<Fq, Fr>(st, t1p, 2 * n - 1, n, L, dfr.template as<Fr>(), 1, dtab, L, hpts.template as<P1>(),
                                     q[M_H].bases.template as<A1>(), &ntt_launches)));
          G16_CUDA(cudaStreamSynchronize(st));   // s is read by the copy above
        }
      }
      G16_CUDA(cudaStreamSynchronize(st));
      hpts.release();
      tm.msm_ms[M_H] = ms_since(t1);
      // --- Lagrange points: [L_i], [alpha L_i], [beta L_i] in G1 (s1 = three blocks of n) and [L_i] in G2: lag's checked
      // points, or the inverse transforms of the first n powers (srs_ifft, n^-1 applied as each point is loaded) ---
      t1 = std::chrono::steady_clock::now();
      DevBuf s1, s2;
      G16_CUDA(s1.reserve(3 * n * sizeof(P1)));
      G16_CUDA(s2.reserve(n * sizeof(P2)));
      P1* s1p = s1.template as<P1>();
      P2* s2p = s2.template as<P2>();
      if (lag) {   // counted with the sparse sums: witness_map_ms is the check
        const int src1[3] = {LAG_TAU_G1, LAG_ALPHA, LAG_BETA};
        for (int b = 0; b < 3; b++) G16_CUDA(srs_load<Fq>(st, lup[src1[b]].template as<A1>(), (uint32_t)n, s1p + b * n));
        G16_CUDA(srs_load<Fq2>(st, lup[LAG_TAU_G2].template as<A2>(), (uint32_t)n, s2p));
        G16_CUDA(cudaStreamSynchronize(st));
      } else {
        const int src1[3] = {SRS_TAU_G1, SRS_ALPHA, SRS_BETA};
        for (int b = 0; b < 3; b++)
          G16_CUDA((srs_ifft<Fq, Fr>(st, up[src1[b]].template as<A1>(), n, 0, L, dtab + 32, 0, dtab, L, s1p + b * n, nullptr,
                                     &ntt_launches)));
        G16_CUDA((srs_ifft<Fq2, Fr>(st, up[SRS_TAU_G2].template as<A2>(), n, 0, L, dtab + 32, 0, dtab, L, s2p, nullptr,
                                    &ntt_launches)));
        G16_CUDA(cudaStreamSynchronize(st));
      }
      for (DevBuf& u : up) u.release();
      for (DevBuf& u : lup) u.release();
      if (!lag) {
        tm.witness_map_ms = ms_since(t1);
        t1 = std::chrono::steady_clock::now();
      }
      // --- sparse sums (r1cs_to_qap.rs:150-167, generator.rs:113-123 with gamma = delta = 1) over the CSC of the matrices:
      // G1 columns [a_query | b_g1_query | gamma_abc_g1 ++ l_query] (3 nv), G2 columns b_g2_query (nv) ---
      struct Csc {
        std::vector<uint64_t> cp;
        std::vector<uint32_t> idx;
        std::vector<Fr> coeff;
      } c1, c2;
      const Fr one = Fr::one();
      // (matrix, column offset, source offset) of every term; instance rows L_(nc + j) added with coefficient One
      auto build = [&](Csc& c, uint64_t cols, std::initializer_list<std::array<uint64_t, 3>> parts,
                       std::initializer_list<std::array<uint64_t, 2>> inst) {
        c.cp.assign(cols + 1, 0);
        for (const auto& p : parts)
          for (uint32_t col : h_col[p[0]]) c.cp[p[1] + col + 1]++;
        for (const auto& p : inst)
          for (uint32_t j = 0; j < ni; j++) c.cp[p[0] + j + 1]++;
        for (uint64_t j = 0; j < cols; j++) c.cp[j + 1] += c.cp[j];
        std::vector<uint64_t> at(c.cp.begin(), c.cp.end() - 1);
        c.idx.resize(c.cp[cols]);
        c.coeff.resize(c.cp[cols]);
        for (const auto& p : parts)
          for (uint32_t i = 0; i < nc; i++)
            for (uint32_t e = h_rp[p[0]][i]; e < h_rp[p[0]][i + 1]; e++) {
              const uint64_t k = at[p[1] + h_col[p[0]][e]]++;
              c.idx[k] = (uint32_t)(p[2] + i);
              c.coeff[k] = h_val[p[0]][e];
            }
        for (const auto& p : inst)
          for (uint32_t j = 0; j < ni; j++) {
            const uint64_t k = at[p[0] + j]++;
            c.idx[k] = (uint32_t)(p[1] + nc + j);
            c.coeff[k] = one;
          }
      };
      build(c1, 3 * nv, {{0, 0, 0}, {1, nv, 0}, {0, 2 * nv, 2 * n}, {1, 2 * nv, n}, {2, 2 * nv, 0}}, {{0, 0}, {2 * nv, 2 * n}});
      build(c2, nv, {{1, 0, 0}}, {});
      SrsSumPlan p1, p2;
      p1.make(c1.cp);
      p2.make(c2.cp);
      // level 1 writes at most entries / 16 + columns items and every later level fewer: the ping-pong buffer `tmp` holds the
      // largest level, `terms` (level 0's output) receives the levels after it
      size_t chunk_max = 1, tmp_bytes = sizeof(P2);
      for (const SrsSumPlan* p : {&p1, &p2})
        for (const auto& lv : p->levels) {
          chunk_max = std::max(chunk_max, lv.size());
          tmp_bytes = std::max(tmp_bytes, (lv.size() - 1) * (p == &p1 ? sizeof(P1) : sizeof(P2)));
        }
      DevBuf didx, dco, terms, tmp, dchunk, dlast, out1;
      const uint64_t e_max = std::max<uint64_t>(c1.idx.size(), c2.idx.size());
      G16_CUDA(didx.reserve(e_max * 4 + 4));
      G16_CUDA(dco.reserve(e_max * sizeof(Fr) + sizeof(Fr)));
      G16_CUDA(terms.reserve(std::max(c1.idx.size() * sizeof(P1), c2.idx.size() * sizeof(P2)) + sizeof(P2)));
      G16_CUDA(tmp.reserve(tmp_bytes));
      G16_CUDA(dchunk.reserve(chunk_max * 8));
      G16_CUDA(dlast.reserve((3 * nv + 1) * 8));
      G16_CUDA(out1.reserve(3 * nv * sizeof(A1)));
      auto upload = [&](const Csc& c) -> cudaError_t {
        cudaError_t e = cudaSuccess;
        if (c.idx.empty()) return e;
        if ((e = cudaMemcpyAsync(didx.p, c.idx.data(), c.idx.size() * 4, cudaMemcpyHostToDevice, st))) return e;
        return cudaMemcpyAsync(dco.p, c.coeff.data(), c.coeff.size() * sizeof(Fr), cudaMemcpyHostToDevice, st);
      };
      G16_CUDA(upload(c1));
      G16_CUDA((srs_sum<Fq, Fr>(st, s1p, didx.template as<uint32_t>(), dco.template as<Fr>(), (uint32_t)c1.idx.size(), p1,
                                terms.template as<P1>(), tmp.template as<P1>(), dchunk.template as<uint64_t>(),
                                dlast.template as<uint64_t>(), (uint32_t)(3 * nv), out1.template as<A1>())));
      G16_CUDA(cudaStreamSynchronize(st));
      G16_CUDA(upload(c2));
      G16_CUDA((srs_sum<Fq2, Fr>(st, s2p, didx.template as<uint32_t>(), dco.template as<Fr>(), (uint32_t)c2.idx.size(), p2,
                                 terms.template as<P2>(), tmp.template as<P2>(), dchunk.template as<uint64_t>(),
                                 dlast.template as<uint64_t>(), (uint32_t)nv, full_b2.template as<A2>())));
      const A1* o1 = out1.template as<A1>();
      G16_CUDA(cudaMemcpyAsync(full_a.p, o1, nv * sizeof(A1), cudaMemcpyDeviceToDevice, st));
      G16_CUDA(cudaMemcpyAsync(full_b1.p, o1 + nv, nv * sizeof(A1), cudaMemcpyDeviceToDevice, st));
      if (ni) G16_CUDA(cudaMemcpyAsync(d_gamma_abc.p, o1 + 2 * nv, ni * sizeof(A1), cudaMemcpyDeviceToDevice, st));
      if (nw) G16_CUDA(cudaMemcpyAsync(q[M_L].bases.p, o1 + 2 * nv + ni, nw * sizeof(A1), cudaMemcpyDeviceToDevice, st));
      G16_CUDA(cudaStreamSynchronize(st));
      tm.msm_ms[M_L] = ms_since(t1);
    }
    // single points (gamma = delta = 1)
    alpha_g1 = load_a1(srs->alpha_tau_g1);
    beta_g1 = load_a1(srs->beta_tau_g1);
    delta_g1 = load_a1(srs->tau_g1);
    beta_g2 = load_a2(srs->beta_g2);
    gamma_g2 = delta_g2 = load_a2(srs->tau_g2);
    rc = commit_setup_key();
    tm.total_ms = ms_since(t0);
    return rc;
  }
  // The combination check of g16_setup_from_lagrange over the uploaded and checked points (up: the transcript's prefixes,
  // lup: lag's members).  With z_i = rho^i (i < n) and z^ = iFFT_n(z), n^-1 included:
  //   sum_i z_i lag.X_i = sum_{j<n} z^_j X_j    for X = tau_g1, tau_g2, alpha_tau_g1, beta_tau_g1 (L_i(X) = (1/n) sum_j
  //                                             omega^-ij X_j, so sum_i z_i L_i(X) = sum_j z^_j X_j)
  //   sum_i z_i H_i = sum_{j<m} w_j tau_g1_j     with w_j = omega_2n^-j z^_(j mod n) / 2 (CircomReduction: H_i is entry
  //                                             2i + 1 of the size-2n inverse transform of tau_g1[0, m), m = 2n - 1, or
  //                                             2n with h2n; the weights srs_h_weights forms)
  // Both sides lie in one group, so no pairing: one MSM per side, ten in all (eight under LibsnarkReduction).  A side that
  // differs is G16_ERR_INVALID_DATA naming the member and level.
  int lagrange_check(DevBuf* up, DevBuf* lup, const Fr& rho, bool h2n) {
    cudaStream_t st = S0.st_main;
    const uint64_t n = 1ull << L, nh = 2 * n - 1 + h2n;
    const bool circom = qap == G16_QAP_CIRCOM;
    const unsigned long long nl0 = ntt_launches;
    Fr tab[64];   // rho^(2^k), then omega_2n^-(2^k)
    tab[0] = rho;
    tab[32] = Fr::inv(fr_domain_root<Fr>(L + 1));
    for (int k = 1; k < 32; k++) { tab[k] = Fr::sqr(tab[k - 1]); tab[32 + k] = Fr::sqr(tab[31 + k]); }
    DevBuf dtab, dpow, dwork, dzh, dh, dmask;
    G16_CUDA(dtab.reserve(sizeof(tab)));
    G16_CUDA(dpow.reserve(n * sizeof(Fr)));
    G16_CUDA(dwork.reserve(n * sizeof(Fr)));
    G16_CUDA(dzh.reserve(n * sizeof(Fr)));
    G16_CUDA(dmask.reserve(circom ? nh : n));
    G16_CUDA(cudaMemcpyAsync(dtab.p, tab, sizeof(tab), cudaMemcpyHostToDevice, st));
    tm.h2d_bytes += sizeof(tab);
    const Fr* dt = dtab.template as<Fr>();
    Fr *P = dpow.template as<Fr>(), *Zh = dzh.template as<Fr>(), *H = nullptr;
    G16_CUDA(srs_powers<Fr>(st, dt, Fr::one(), (uint32_t)n, P));
    const Fr zero = Fr::zero();
    ntt_any(st, dom, true, P, dwork.template as<Fr>(), Zh, NTT_LOAD_PLAIN, nullptr, nullptr, nullptr, zero, NTT_STORE_MUL_CONST,
            nullptr, dom.n_inv);
    if (circom) {
      G16_CUDA(dh.reserve(nh * sizeof(Fr)));
      H = dh.template as<Fr>();
      G16_CUDA(srs_h_weights<Fr>(st, dt + 32, Fr::inv(fr_from_u64<Fr>(2)), Zh, (uint32_t)n, (uint32_t)nh, H));
    }
    G16_CUDA(cudaGetLastError());
    G16_CUDA(cudaStreamSynchronize(st));
    dwork.release();
    tm.launches += 1 + circom + (ntt_launches - nl0);   // powers, H weights, the transform
    MsmWorkspace<Fq> ws1;
    MsmWorkspace<Fq2> ws2;
    MsmCounters mc;
    uint8_t* mk = dmask.template as<uint8_t>();
    auto same = [](const auto& a, const auto& b) {
      const auto x = a.to_affine(), y = b.to_affine();
      return memcmp(&x, &y, sizeof(x)) == 0;
    };
    int rc;
    for (int k = 0; k < LAG_MEMBERS; k++) {
      if (k == LAG_H && !circom) continue;
      bool ok;
      rc = G16_OK;
      if (k == LAG_TAU_G2) {
        P2 lhs = P2::inf(), rhs = P2::inf();
        if (!(rc = msm_device<Fq2>(ws2, mc, true, lup[k].template as<A2>(), P, n, mk, lhs)))
          rc = msm_device<Fq2>(ws2, mc, true, up[SRS_TAU_G2].template as<A2>(), Zh, n, mk, rhs);
        ok = same(lhs, rhs);
      } else {
        P1 lhs = P1::inf(), rhs = P1::inf();
        const int src = k == LAG_H ? (int)SRS_TAU_G1 : k;   // LAG_TAU_G1, LAG_ALPHA, LAG_BETA are their SRS_ members
        if (!(rc = msm_device<Fq>(ws1, mc, false, lup[k].template as<A1>(), P, n, mk, lhs)))
          rc = msm_device<Fq>(ws1, mc, false, up[src].template as<A1>(), k == LAG_H ? H : Zh, k == LAG_H ? nh : n, mk, rhs);
        ok = same(lhs, rhs);
      }
      if (rc || !ok) tm.launches += mc.launches;
      if (rc) return rc;
      if (!ok) {
        if (k == LAG_H)
          return fail(G16_ERR_INVALID_DATA, "lagrange tau_g1_h (level 2^" + std::to_string(L + 1) + "): not the odd entries of the "
                                            "inverse transform of tau_g1[0, " + std::to_string(nh) + ")");
        return fail(G16_ERR_INVALID_DATA, std::string("lagrange ") + lag_member(k) + " (level 2^" + std::to_string(L) +
                                              "): not the inverse transform of " + srs_member(k) + "[0, " + std::to_string(n) + ")");
      }
    }
    tm.launches += mc.launches;
    return G16_OK;
  }
  // The H query from lag's tau_g1_h taken over 2n powers (an interior level of a .ptau's section 12), into q[M_H]'s bases:
  // with H'_i = (1/2n) sum_{j<2n} omega_2n^-((2i+1)j) [tau^j] and omega_2n^(-(2i+1)(2n-1)) = omega_2n^(2i+1),
  //   H_i = H'_i - c_i T,  c_i = (omega_2n / 2n) omega_n^i,  T = tau_g1[2n - 1]  (entry 2n - 1 of the H query's source is 0).
  // On the device: T copied to n slots, each times its c_i (srs_contribute_kernel, scalars from omega_n^(2^k)), then
  // srs_diff H'_i - c_i T and srs_affine.  h and t are device arrays of checked points.
  int lagrange_h_correct(const A1* h, const A1* t) {
    cudaStream_t st = S0.st_main;
    const uint64_t n = 1ull << L;
    DevBuf y, hpts, dtab;
    G16_CUDA(y.reserve(2 * n * sizeof(A1)));
    G16_CUDA(hpts.reserve(n * sizeof(P1)));
    A1* yp = y.template as<A1>();
    G16_CUDA(cudaMemcpyAsync(yp, h, n * sizeof(A1), cudaMemcpyDeviceToDevice, st));
    G16_CUDA(cudaMemcpyAsync(yp + n, t, sizeof(A1), cudaMemcpyDeviceToDevice, st));
    for (uint64_t k = 1; k < n; k *= 2)   // slots [n, n + k) hold T: copy them to [n + k, n + 2k)
      G16_CUDA(cudaMemcpyAsync(yp + n + k, yp + n, std::min(k, n - k) * sizeof(A1), cudaMemcpyDeviceToDevice, st));
    Fr tab[32];   // omega_n^(2^k)
    tab[0] = fr_domain_root<Fr>(L);
    for (int k = 1; k < 32; k++) tab[k] = Fr::sqr(tab[k - 1]);
    G16_CUDA(dtab.reserve(sizeof(tab)));
    G16_CUDA(cudaMemcpyAsync(dtab.p, tab, sizeof(tab), cudaMemcpyHostToDevice, st));
    const Fr c0 = Fr::mul(fr_domain_root<Fr>(L + 1), Fr::inv(fr_from_u64<Fr>(2 * n)));
    G16_CUDA((g16::srs_contribute<Fq, Fr>(st, yp + n, (uint32_t)n, dtab.template as<Fr>(), c0)));
    G16_CUDA(srs_diff<Fq>(st, yp, (uint32_t)(2 * n), 0, (uint32_t)n, (uint32_t)n, hpts.template as<P1>()));
    G16_CUDA(srs_affine<Fq>(st, hpts.template as<P1>(), (uint32_t)n, q[M_H].bases.template as<A1>()));
    G16_CUDA(cudaStreamSynchronize(st));   // tab is read by the copy above
    tm.h2d_bytes += sizeof(tab);
    tm.launches += 3;
    return G16_OK;
  }
  // One phase-2 contribution: delta_g1, delta_g2 times delta; the H and L queries times delta^-1; the key re-committed.
  int setup_contribute(const uint64_t* delta_) override {
    if (!delta_) return fail(G16_ERR_BAD_ARGUMENT, "null delta");
    G16_NOT_BUSY();
    if (!have_pk || !from_setup || world != 1)
      return fail(G16_ERR_BAD_ARGUMENT, "g16_setup_contribute needs a resident key made by g16_setup or g16_setup_from_srs (world 1)");
    const Fr d = load_fr(delta_);
    if (d.is_zero()) return fail(G16_ERR_BAD_ARGUMENT, "delta must be invertible (UnexpectedIdentity)");
    G16_CUDA(cudaSetDevice(device));
    const Fr di = Fr::inv(d);
    const uint64_t nv = nvars(), hn = h_query_len(), nw = num_witness, cnt = hn + nw;
    cudaStream_t st = S0.st_main;
    {
      DevBuf aff, pts, ds;
      G16_CUDA(aff.reserve(cnt * sizeof(A1) + sizeof(A1)));
      G16_CUDA(pts.reserve(cnt * sizeof(P1) + sizeof(P1)));
      G16_CUDA(ds.reserve(sizeof(Fr)));
      A1* a = aff.template as<A1>();
      if (hn) G16_CUDA(cudaMemcpyAsync(a, q[M_H].bases.p, hn * sizeof(A1), cudaMemcpyDeviceToDevice, st));
      if (nw) G16_CUDA(cudaMemcpyAsync(a + hn, q[M_L].bases.p, nw * sizeof(A1), cudaMemcpyDeviceToDevice, st));
      G16_CUDA(cudaMemcpyAsync(ds.p, &di, sizeof(Fr), cudaMemcpyHostToDevice, st));
      G16_CUDA(srs_load<Fq>(st, a, (uint32_t)cnt, pts.template as<P1>()));
      G16_CUDA((srs_scale<Fq, Fr>(st, pts.template as<P1>(), (uint32_t)cnt, ds.template as<Fr>(), 0)));
      G16_CUDA(srs_affine<Fq>(st, pts.template as<P1>(), (uint32_t)cnt, a));
      G16_CUDA(cudaStreamSynchronize(st));
      const uint64_t len[5] = {hn, nw, nv, nv, nv};
      int rc = begin_key(0, 1, len);
      if (rc) return rc;
      if (hn) G16_CUDA(cudaMemcpyAsync(q[M_H].bases.p, a, hn * sizeof(A1), cudaMemcpyDeviceToDevice, st));
      if (nw) G16_CUDA(cudaMemcpyAsync(q[M_L].bases.p, a + hn, nw * sizeof(A1), cudaMemcpyDeviceToDevice, st));
      G16_CUDA(cudaStreamSynchronize(st));
    }
    uint32_t k[Fr::N];
    fr_to_canon(d, k);
    delta_g1 = P1::from_affine(delta_g1).mul_u32(k, Fr::N).to_affine();
    delta_g2 = P2::from_affine(delta_g2).mul_u32(k, Fr::N).to_affine();
    return commit_setup_key();
  }
  // g16_srs_from_secrets: member i of each vector is tau^i times [1]G1, [1]G2, [alpha]G1, [beta]G1
  int srs_from_secrets(const uint64_t* tau_, const uint64_t* alpha_, const uint64_t* beta_, const uint64_t* g1_,
                       const uint64_t* g2_, const g16_srs_out* out) override {
    if (!tau_ || !alpha_ || !beta_ || !g1_ || !g2_ || !out || !out->beta_g2) return fail(G16_ERR_BAD_ARGUMENT, "null argument");
    if ((out->tau_g1_len && !out->tau_g1) || (out->tau_g2_len && !out->tau_g2) || (out->alpha_tau_g1_len && !out->alpha_tau_g1) ||
        (out->beta_tau_g1_len && !out->beta_tau_g1))
      return fail(G16_ERR_BAD_ARGUMENT, "null srs output member");
    const uint64_t mx = std::max(std::max(out->tau_g1_len, out->tau_g2_len), std::max(out->alpha_tau_g1_len, out->beta_tau_g1_len));
    if (mx >= (1ull << 31)) return fail(G16_ERR_BAD_ARGUMENT, "srs member too long");
    G16_NOT_BUSY();
    G16_CUDA(cudaSetDevice(device));
    const Fr tau = load_fr(tau_);
    const A1 g1 = load_a1(g1_);
    const A2 g2 = load_a2(g2_);
    uint32_t k[Fr::N];
    auto mul1 = [&](const Fr& s) { fr_to_canon(s, k); return P1::from_affine(g1).mul_u32(k, Fr::N).to_affine(); };
    auto mul2 = [&](const Fr& s) { fr_to_canon(s, k); return P2::from_affine(g2).mul_u32(k, Fr::N).to_affine(); };
    std::vector<Fr> pw(mx);
    Fr p = Fr::one();
    for (uint64_t i = 0; i < mx; i++) { pw[i] = p; p = Fr::mul(p, tau); }
    DevBuf ds, dout, tab;
    G16_CUDA(ds.reserve(mx * sizeof(Fr) + sizeof(Fr)));
    G16_CUDA(dout.reserve(mx * sizeof(A2) + sizeof(A2)));
    if (mx) G16_CUDA(cudaMemcpyAsync(ds.p, pw.data(), mx * sizeof(Fr), cudaMemcpyHostToDevice, S0.st_main));
    auto run1 = [&](const A1& gen, uint64_t* dst, uint64_t cnt) -> int {
      if (!cnt) return G16_OK;
      int rc = batch_mul<Fq>(gen, ds.template as<Fr>(), cnt, dout.template as<A1>(), tab);
      if (rc) return rc;
      G16_CUDA(cudaMemcpyAsync(dst, dout.p, cnt * sizeof(A1), cudaMemcpyDeviceToHost, S0.st_main));
      G16_CUDA(cudaStreamSynchronize(S0.st_main));
      return G16_OK;
    };
    int rc;
    if ((rc = run1(g1, out->tau_g1, out->tau_g1_len))) return rc;
    if ((rc = run1(mul1(load_fr(alpha_)), out->alpha_tau_g1, out->alpha_tau_g1_len))) return rc;
    if ((rc = run1(mul1(load_fr(beta_)), out->beta_tau_g1, out->beta_tau_g1_len))) return rc;
    if (out->tau_g2_len) {
      if ((rc = batch_mul<Fq2>(g2, ds.template as<Fr>(), out->tau_g2_len, dout.template as<A2>(), tab))) return rc;
      G16_CUDA(cudaMemcpyAsync(out->tau_g2, dout.p, out->tau_g2_len * sizeof(A2), cudaMemcpyDeviceToHost, S0.st_main));
      G16_CUDA(cudaStreamSynchronize(S0.st_main));
    }
    store_a2(out->beta_g2, mul2(load_fr(beta_)));
    return G16_OK;
  }
  // g16_srs_contribute: one phase-1 contribution (tau, alpha, beta).  Point i of tau_g1 and tau_g2 times tau^i, of
  // alpha_tau_g1 times alpha tau^i, of beta_tau_g1 times beta tau^i; beta_g2 times beta.  Two passes over the members in
  // chunks of at most `cap` points through one device buffer: every point is uploaded and checked before anything is written
  // to `out`, then every chunk is uploaded again, transformed in place on the device (srs_contribute_kernel) and copied out.
  // Timings (host clock around work that ends in a stream synchronise): h2d_ms = the check pass, msm_ms[m] = the transform
  // of member m < 4, total_ms = the whole call.
  int srs_contribute(const g16_srs_desc* in, const uint64_t* tau_, const uint64_t* alpha_, const uint64_t* beta_, uint32_t flags,
                     uint64_t chunk_points, const g16_srs_out* out) override {
    if (!in || !out || !tau_ || !alpha_ || !beta_) return fail(G16_ERR_BAD_ARGUMENT, "null argument");
    if (flags & ~(uint32_t)G16_SER_VALIDATE) return fail(G16_ERR_BAD_ARGUMENT, "g16_srs_contribute takes 0 or G16_SER_VALIDATE");
    const uint64_t* src[SRS_MEMBERS] = {in->tau_g1, in->tau_g2, in->alpha_tau_g1, in->beta_tau_g1, in->beta_g2};
    uint64_t* dst[SRS_MEMBERS] = {out->tau_g1, out->tau_g2, out->alpha_tau_g1, out->beta_tau_g1, out->beta_g2};
    const uint64_t len[SRS_MEMBERS] = {in->tau_g1_len, in->tau_g2_len, in->alpha_tau_g1_len, in->beta_tau_g1_len, 1};
    const uint64_t olen[SRS_MEMBERS] = {out->tau_g1_len, out->tau_g2_len, out->alpha_tau_g1_len, out->beta_tau_g1_len, 1};
    const uint64_t esz[SRS_MEMBERS] = {sizeof(A1), sizeof(A2), sizeof(A1), sizeof(A1), sizeof(A2)};
    for (int m = 0; m < SRS_MEMBERS; m++) {
      const std::string name = srs_member(m);
      if (olen[m] != len[m])
        return fail(G16_ERR_BAD_ARGUMENT, "out " + name + " holds " + std::to_string(olen[m]) + " points, in " + name + " " +
                                              std::to_string(len[m]) + ": the lengths must be equal");
      if (len[m] >> 32)
        return fail(G16_ERR_BAD_ARGUMENT, name + " holds " + std::to_string(len[m]) + " points, at most 2^32 - 1 are allowed");
      if (len[m] && (!src[m] || !dst[m])) return fail(G16_ERR_BAD_ARGUMENT, "null srs member " + name);
    }
    // an output range may be its own input range (in place) and must overlap no other input or output range
    auto overlap = [&](const void* a, int ma, const void* b, int mb) {
      return srs_overlap((uintptr_t)a, len[ma] * esz[ma], (uintptr_t)b, len[mb] * esz[mb]);
    };
    for (int o = 0; o < SRS_MEMBERS; o++)
      for (int m = 0; m < SRS_MEMBERS; m++) {
        if (overlap(dst[o], o, src[m], m) && !(o == m && (const void*)dst[o] == (const void*)src[m]))
          return fail(G16_ERR_BAD_ARGUMENT, std::string("out ") + srs_member(o) + " overlaps in " + srs_member(m) +
                                                ": an output may only be the very same array as its own input");
        if (m > o && overlap(dst[o], o, dst[m], m))
          return fail(G16_ERR_BAD_ARGUMENT, std::string("out ") + srs_member(o) + " overlaps out " + srs_member(m));
      }
    const Fr tau = load_fr(tau_), alpha = load_fr(alpha_), beta = load_fr(beta_);
    if (tau.is_zero() || alpha.is_zero() || beta.is_zero())
      return fail(G16_ERR_BAD_ARGUMENT, "tau, alpha and beta must be non-zero (UnexpectedIdentity)");
    G16_NOT_BUSY();
    G16_CUDA(cudaSetDevice(device));
    const auto t0 = std::chrono::steady_clock::now();
    auto ms_since = [](std::chrono::steady_clock::time_point a) {
      return (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count();
    };
    tm = g16_timings{};
    cudaStream_t st = S0.st_main;
    const uint64_t big = std::max(sizeof(A1), sizeof(A2));
    size_t free_b = 0, total_b = 0;
    G16_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const uint64_t longest = *std::max_element(len, len + SRS_MEMBERS);
    const uint64_t cap = srs_chunk_cap(chunk_points, longest, free_b, big);
    DevBuf buf, err, dtab;
    G16_CUDA(buf.reserve(cap * big));
    G16_CUDA(err.reserve(8));
    auto part = [&](int m, uint64_t i0) { return i0 * esz[m]; };   // byte offset of point i0 of member m
    // --- check pass: every point, chunk by chunk; the first bad one by member, then index ---
    for (int m = 0; m < SRS_MEMBERS; m++) {
      const bool g2 = m == SRS_TAU_G2 || m == SRS_BETA_G2;
      for (uint64_t i0 = 0; i0 < len[m];) {
        const uint32_t cnt = srs_chunk_len(len[m], i0, cap);
        G16_CUDA(cudaMemcpyAsync(buf.p, (const char*)src[m] + part(m, i0), cnt * esz[m], cudaMemcpyHostToDevice, st));
        G16_CUDA(cudaMemsetAsync(err.p, 0xff, 8, st));
        unsigned long long* e = err.template as<unsigned long long>();
        G16_CUDA((g2 ? srs_check<CP, true>(st, buf.p, cnt, flags, m, e) : srs_check<CP, false>(st, buf.p, cnt, flags, m, e)));
        unsigned long long first_err = 0;
        G16_CUDA(cudaMemcpyAsync(&first_err, err.p, 8, cudaMemcpyDeviceToHost, st));
        G16_CUDA(cudaStreamSynchronize(st));
        tm.h2d_bytes += cnt * esz[m];
        tm.d2h_bytes += 8;
        tm.launches++;
        if (first_err != ~0ull)
          return fail(G16_ERR_INVALID_DATA, std::string(srs_member(m)) + "[" +
                                                std::to_string(i0 + ((first_err >> 8) & ((1ull << 40) - 1))) + "]: " +
                                                ser_reason(first_err & 0xff));
        i0 += cnt;
      }
    }
    tm.h2d_ms = ms_since(t0);
    // --- transform pass: chunk [i0, i0 + cnt) of member m times x tau^(i0 + j), x = 1, 1, alpha, beta ---
    Fr tab[32];
    tab[0] = tau;
    for (int k = 1; k < 32; k++) tab[k] = Fr::sqr(tab[k - 1]);
    G16_CUDA(dtab.reserve(sizeof(tab)));
    G16_CUDA(cudaMemcpyAsync(dtab.p, tab, sizeof(tab), cudaMemcpyHostToDevice, st));
    tm.h2d_bytes += sizeof(tab);
    const Fr x[4] = {Fr::one(), Fr::one(), alpha, beta};
    for (int m = 0; m < 4; m++) {
      const auto t1 = std::chrono::steady_clock::now();
      for (uint64_t i0 = 0; i0 < len[m];) {
        const uint32_t cnt = srs_chunk_len(len[m], i0, cap);
        const Fr c = srs_power(x[m], tab, i0);
        G16_CUDA(cudaMemcpyAsync(buf.p, (const char*)src[m] + part(m, i0), cnt * esz[m], cudaMemcpyHostToDevice, st));
        G16_CUDA((m == SRS_TAU_G2 ? g16::srs_contribute<Fq2, Fr>(st, buf.template as<A2>(), cnt, dtab.template as<Fr>(), c)
                                  : g16::srs_contribute<Fq, Fr>(st, buf.template as<A1>(), cnt, dtab.template as<Fr>(), c)));
        G16_CUDA(cudaMemcpyAsync((char*)dst[m] + part(m, i0), buf.p, cnt * esz[m], cudaMemcpyDeviceToHost, st));
        tm.h2d_bytes += cnt * esz[m];
        tm.d2h_bytes += cnt * esz[m];
        tm.launches++;
        i0 += cnt;
      }
      G16_CUDA(cudaStreamSynchronize(st));
      tm.msm_ms[m] = ms_since(t1);
    }
    // beta_g2 is one point: on the host, as g16_setup_contribute does for delta_g2
    uint32_t k[Fr::N];
    fr_to_canon(beta, k);
    store_a2(dst[SRS_BETA_G2], P2::from_affine(load_a2(src[SRS_BETA_G2])).mul_u32(k, Fr::N).to_affine());
    tm.total_ms = ms_since(t0);
    return G16_OK;
  }
  // The MSM geometry of one chunk of a transcript check: caller-supplied bases, as msm_host runs them
  MsmGeom srs_verify_geom(uint64_t cnt, bool g2) const { return with_k0(msm_geom(cnt, FR_BITS, (int)tune.c, 0), g2); }
  // One member of g16_srs_verify_pairs: sum = sum_i rho^i X_i over its len points, in chunks of at most cap points through
  // buf (points), dsc (scalars) and dmask (identity mask).  Each chunk is uploaded and checked (the identity refused, and
  // with gen the first point must be that generator) and its error word read before its scalars and MSM are enqueued, so a
  // refusal stops the call before a later chunk is read.  The chunk's MSM result is added to sum on the host.
  template <class F>
  int srs_verify_member(int m, bool g2, const uint64_t* src, uint64_t len, const uint64_t* gen, uint32_t flags, uint64_t cap,
                        DevBuf& buf, DevBuf& dsc, DevBuf& dmask, DevBuf& err, const Fr* dtab, const Fr* tab, XYZZ<F>& sum) {
    cudaStream_t st = S0.st_main;
    MsmWorkspace<F> ws;   // this call's own: the prover's workspaces keep their sizes
    MsmCounters mc;
    sum = XYZZ<F>::inf();
    for (uint64_t i0 = 0; i0 < len;) {
      const uint32_t cnt = srs_chunk_len(len, i0, cap);
      G16_CUDA(cudaMemcpyAsync(buf.p, src + i0 * (sizeof(Affine<F>) / 8), cnt * sizeof(Affine<F>), cudaMemcpyHostToDevice, st));
      G16_CUDA(cudaMemsetAsync(err.p, 0xff, 8, st));
      unsigned long long* e = err.template as<unsigned long long>();
      const uint32_t fl = flags | SRS_REFUSE_IDENTITY;
      G16_CUDA((g2 ? srs_check<CP, true>(st, buf.p, cnt, fl, m, e) : srs_check<CP, false>(st, buf.p, cnt, fl, m, e)));
      unsigned long long first_err = 0;
      G16_CUDA(cudaMemcpyAsync(&first_err, err.p, 8, cudaMemcpyDeviceToHost, st));
      G16_CUDA(cudaStreamSynchronize(st));
      tm.h2d_bytes += cnt * sizeof(Affine<F>);
      tm.d2h_bytes += 8;
      tm.launches++;
      const uint64_t bad_at = first_err == ~0ull ? ~0ull : i0 + ((first_err >> 8) & ((1ull << 40) - 1));
      // point 0 first: a failed check there is named as such, else a wrong generator comes before any later bad point
      if (bad_at != 0 && i0 == 0 && gen && memcmp(src, gen, sizeof(Affine<F>)))
        return fail(G16_ERR_INVALID_DATA, std::string(srs_member(m)) + "[0]: not the generator " + (g2 ? "g2" : "g1"));
      if (first_err != ~0ull)
        return fail(G16_ERR_INVALID_DATA, std::string(srs_member(m)) + "[" + std::to_string(bad_at) + "]: " +
                                              srs_reason(first_err & 0xff));
      // scalars rho^(i0 + j), then the chunk's MSM
      G16_CUDA(srs_powers<Fr>(st, dtab, srs_power(Fr::one(), tab, i0), cnt, dsc.template as<Fr>()));
      tm.launches++;
      int rc = msm_device<F>(ws, mc, g2, buf.template as<Affine<F>>(), dsc.template as<Fr>(), cnt, dmask.template as<uint8_t>(), sum);
      if (rc) return rc;
      i0 += cnt;
    }
    tm.launches += mc.launches;
    return G16_OK;
  }
  // acc += sum_{i<cnt} s_i P_i over device bases and device Montgomery scalars, on the main stream through a workspace the
  // calling entry point owns (the prover's keep their sizes): the identity mask into dmask (cnt bytes), then the prover's
  // MSM pipeline, in pieces of at most SRS_VERIFY_MSM_MAX pairs; the host waits for each.  Counts the mask launches and the
  // bytes msm_enqueue copies back in tm, the pipeline's launches in mc.
  template <class F>
  int msm_device(MsmWorkspace<F>& ws, MsmCounters& mc, bool g2, Affine<F>* bases, const Fr* sc, uint64_t cnt, uint8_t* dmask,
                 XYZZ<F>& acc) {
    cudaStream_t st = S0.st_main;
    for (uint64_t i0 = 0; i0 < cnt; i0 += SRS_VERIFY_MSM_MAX) {
      const uint32_t c = (uint32_t)std::min<uint64_t>(SRS_VERIFY_MSM_MAX, cnt - i0);
      G16_CUDA(msm_prepare_query<F>(st, bases + i0, c, 1, 0, dmask));
      const MsmGeom g = srs_verify_geom(c, g2);
      G16_CUDA((msm_enqueue<F, Fr>(st, ws, g, bases + i0, dmask, reinterpret_cast<const uint32_t*>(sc + i0), 1, true, &mc, nullptr,
                                   nullptr, nullptr, nullptr, nullptr, 0)));
      G16_CUDA(cudaStreamSynchronize(st));
      acc.add(msm_finish<F>(ws, g));
      tm.launches++;
      tm.d2h_bytes += 4 + ws.plan.leaf_pts * g.sets() * sizeof(XYZZ<F>);   // msm_enqueue's slot total and leaf arrays
    }
    return G16_OK;
  }
  // g16_srs_verify_pairs: the five pairing equations of a powers-of-tau transcript under the challenge rho, after every
  // point passed the checks (srs_verify_member).  For a member X of N points, S = sum_{i<N} rho^i X_i is one MSM per member;
  // lo = S - rho^(N-1) X_(N-1) and hi = rho^-1 (S - X_0) are formed on the host.  Nothing is written until every check passed.
  // Timings (host clock around work that ends in a stream synchronise): msm_ms[m] = member m's chunk loop, total_ms = the
  // whole call.
  int srs_verify_pairs(const g16_srs_desc* srs, const uint64_t* g1_, const uint64_t* g2_, const uint64_t* rho_, uint32_t flags,
                       uint64_t chunk_points, uint64_t* pairs_g1, uint64_t* pairs_g2) override {
    if (!srs || !g1_ || !g2_ || !rho_ || !pairs_g1 || !pairs_g2) return fail(G16_ERR_BAD_ARGUMENT, "null argument");
    const uint64_t* src[SRS_MEMBERS] = {srs->tau_g1, srs->tau_g2, srs->alpha_tau_g1, srs->beta_tau_g1, srs->beta_g2};
    const uint64_t len[SRS_MEMBERS] = {srs->tau_g1_len, srs->tau_g2_len, srs->alpha_tau_g1_len, srs->beta_tau_g1_len, 1};
    for (int m = 0; m < SRS_MEMBERS; m++)
      if (!src[m]) return fail(G16_ERR_BAD_ARGUMENT, std::string("null srs member ") + srs_member(m));
    if (flags & ~(uint32_t)G16_SER_VALIDATE) return fail(G16_ERR_BAD_ARGUMENT, "g16_srs_verify_pairs takes 0 or G16_SER_VALIDATE");
    const Fr rho = load_fr(rho_);
    if (rho.is_zero()) return fail(G16_ERR_BAD_ARGUMENT, "the challenge rho must be non-zero");
    const uint64_t need[SRS_MEMBERS] = {2, 2, 1, 1, 1};
    for (int m = 0; m < SRS_MEMBERS; m++) {
      if (len[m] < need[m])
        return fail(G16_ERR_BAD_ARGUMENT, std::string(srs_member(m)) + " holds " + std::to_string(len[m]) + " points, at least " +
                                              std::to_string(need[m]) + " are needed");
      if (len[m] >> 32)
        return fail(G16_ERR_BAD_ARGUMENT, std::string(srs_member(m)) + " holds " + std::to_string(len[m]) +
                                              " points, at most 2^32 - 1 are allowed");
    }
    G16_NOT_BUSY();
    G16_CUDA(cudaSetDevice(device));
    const auto t0 = std::chrono::steady_clock::now();
    auto ms_since = [](std::chrono::steady_clock::time_point a) {
      return (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count();
    };
    tm = g16_timings{};
    cudaStream_t st = S0.st_main;
    size_t free_b = 0, total_b = 0;
    G16_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const uint64_t longest = *std::max_element(len, len + SRS_BETA_G2);
    // one workspace is alive at a time (per member), so a chunk needs the larger of the two groups' workspaces
    auto ws_bytes = [&](uint64_t cnt) {
      MsmGeom g[2] = {srs_verify_geom(cnt, false), srs_verify_geom(cnt, true)};
      MsmBaPlan bap[2];
      MsmRedPlan plan[2];
      for (int k = 0; k < 2; k++) { bap[k].make(g[k]); plan[k].make(g[k].c - 1); }
      return std::max(msm_ws_bytes<Fq>(g[0], bap[0], plan[0]).total(), msm_ws_bytes<Fq2>(g[1], bap[1], plan[1]).total());
    };
    const uint64_t per_point = std::max(sizeof(A1), sizeof(A2)) + sizeof(Fr) + 1;
    const uint64_t cap = srs_verify_chunk_cap(chunk_points, longest, free_b, per_point, ws_bytes);
    DevBuf buf, dsc, dmask, err, dtab;
    G16_CUDA(buf.reserve(cap * std::max(sizeof(A1), sizeof(A2))));
    G16_CUDA(dsc.reserve(cap * sizeof(Fr)));
    G16_CUDA(dmask.reserve(cap));
    G16_CUDA(err.reserve(8));
    Fr tab[32];
    tab[0] = rho;
    for (int k = 1; k < 32; k++) tab[k] = Fr::sqr(tab[k - 1]);
    G16_CUDA(dtab.reserve(sizeof(tab)));
    G16_CUDA(cudaMemcpyAsync(dtab.p, tab, sizeof(tab), cudaMemcpyHostToDevice, st));
    tm.h2d_bytes += sizeof(tab);
    P1 s1[4];
    P2 s2;
    int rc;
    for (int m = 0; m < 4; m++) {
      const auto t1 = std::chrono::steady_clock::now();
      if (m == SRS_TAU_G2)
        rc = srs_verify_member<Fq2>(m, true, src[m], len[m], g2_, flags, cap, buf, dsc, dmask, err, dtab.template as<Fr>(), tab, s2);
      else
        rc = srs_verify_member<Fq>(m, false, src[m], len[m], m == SRS_TAU_G1 ? g1_ : nullptr, flags, cap, buf, dsc, dmask, err,
                                   dtab.template as<Fr>(), tab, s1[m]);
      if (rc) return rc;
      tm.msm_ms[m] = ms_since(t1);
      tm.msm_pairs[m] = len[m];
    }
    // beta_g2 is one point: checked on the device with the others, used on the host
    G16_CUDA(cudaMemcpyAsync(buf.p, src[SRS_BETA_G2], sizeof(A2), cudaMemcpyHostToDevice, st));
    G16_CUDA(cudaMemsetAsync(err.p, 0xff, 8, st));
    G16_CUDA((srs_check<CP, true>(st, buf.p, 1, flags | SRS_REFUSE_IDENTITY, SRS_BETA_G2, err.template as<unsigned long long>())));
    unsigned long long first_err = 0;
    G16_CUDA(cudaMemcpyAsync(&first_err, err.p, 8, cudaMemcpyDeviceToHost, st));
    G16_CUDA(cudaStreamSynchronize(st));
    tm.h2d_bytes += sizeof(A2);
    tm.d2h_bytes += 8;
    tm.launches++;
    if (first_err != ~0ull) return fail(G16_ERR_INVALID_DATA, std::string("beta_g2[0]: ") + srs_reason(first_err & 0xff));
    // lo and hi of every member: two scalar multiplications and one shared inversion
    const Fr rho_inv = Fr::inv(rho);
    uint32_t k[Fr::N];
    auto lo_hi = [&](auto S, auto pt, int m, auto& lo, auto& hi) {
      using PT = decltype(S);
      const uint64_t w = srs_point_limbs(m);
      const PT x0 = PT::from_affine(pt(src[m])), xl = PT::from_affine(pt(src[m] + (len[m] - 1) * w));
      fr_to_canon(srs_power(Fr::one(), tab, len[m] - 1), k);
      PT t = xl.mul_u32(k, Fr::N);
      t.negate();
      lo = S;
      lo.add(t);
      PT d = x0;
      d.negate();
      d.add(S);
      fr_to_canon(rho_inv, k);
      hi = d.mul_u32(k, Fr::N);
    };
    P1 lo1[4], hi1[4];
    P2 lo2, hi2;
    for (int m : {SRS_TAU_G1, SRS_ALPHA, SRS_BETA}) lo_hi(s1[m], load_a1, m, lo1[m], hi1[m]);
    lo_hi(s2, load_a2, SRS_TAU_G2, lo2, hi2);
    const A1 g1 = load_a1(g1_), t1 = load_a1(src[SRS_TAU_G1] + 2 * NQ64), b0 = load_a1(src[SRS_BETA]);
    const A2 g2 = load_a2(g2_), t2 = load_a2(src[SRS_TAU_G2] + G2_64), bg2 = load_a2(src[SRS_BETA_G2]);
    // equation k: e(P_k, Q_k) = e(P'_k, Q'_k), written as P_0, P'_0, .., P_4, P'_4 and Q_0, Q'_0, .., Q_4, Q'_4
    const A1 ps[10] = {hi1[SRS_TAU_G1].to_affine(), lo1[SRS_TAU_G1].to_affine(), g1, t1, hi1[SRS_ALPHA].to_affine(),
                       lo1[SRS_ALPHA].to_affine(), hi1[SRS_BETA].to_affine(), lo1[SRS_BETA].to_affine(), b0, g1};
    const A2 qs[10] = {g2, t2, hi2.to_affine(), lo2.to_affine(), g2, t2, g2, t2, g2, bg2};
    for (int i = 0; i < 10; i++) {
      store_a1(pairs_g1 + (size_t)i * 2 * NQ64, ps[i]);
      store_a2(pairs_g2 + (size_t)i * G2_64, qs[i]);
    }
    tm.total_ms = ms_since(t0);
    return G16_OK;
  }
  // u64 limbs of one point of transcript member m
  static uint64_t srs_point_limbs(int m) { return (m == SRS_TAU_G2 || m == SRS_BETA_G2) ? (uint64_t)G2_64 : (uint64_t)(2 * NQ64); }

  // ---- checking a proving key against the resident circuit and a transcript (g16_pk_verify_pairs) ----
  // Members of the key in the order their points are checked; the error word names transcript member m as PKV_SRS + m, so
  // that the first bad point is the key's before the transcript's.
  enum { PKV_A = 0, PKV_B1, PKV_B2, PKV_H, PKV_L, PKV_ABC, PKV_ALPHA, PKV_BETA, PKV_DELTA1, PKV_BETA2, PKV_GAMMA2, PKV_DELTA2,
         PKV_MEMBERS, PKV_SRS = 16 };
  static const char* pkv_member(int m) {
    static const char* t[PKV_MEMBERS] = {"a_query", "b_g1_query", "b_g2_query", "h_query",  "l_query",  "gamma_abc_g1",
                                         "alpha_g1", "beta_g1",   "delta_g1",   "beta_g2", "gamma_g2", "delta_g2"};
    return m >= PKV_SRS ? srs_member(m - PKV_SRS) : t[m];
  }
  static bool pkv_g2(int m) { return m == PKV_B2 || m == PKV_BETA2 || m == PKV_GAMMA2 || m == PKV_DELTA2; }
  // g16_pk_verify_pairs.  With z_j = rho^j (j < nv), z^I = z on the instance variables and 0 elsewhere, z^L = z - z^I, the
  // combination sum_j rho^j K_j of each key member equals one MSM per transcript member over the transcript-side weights,
  // which are field transforms of z (DESIGN.md section 16):
  //   a_query, b_g1_query, b_g2_query  tau_g1 / tau_g2 [0, n) by the inverse transforms a^, b^ of A z, B z (instance rows
  //                                    included, as the witness map forms them)
  //   l_query (x delta), gamma_abc_g1 (x gamma)  beta_tau_g1 by a^, alpha_tau_g1 by b^, tau_g1 by c^, of z^L and z^I
  //   h_query (x delta)                 tau_g1 [0, 2n - 1) by srs_h_weights
  // On the device: rho^j, one matvec of the three assignments z^I, z^L, z, one batch of nine inverse transforms, the H
  // weights, and fifteen MSMs (more past SRS_VERIFY_MSM_MAX pairs).  The host compares the A and B sums and writes the
  // four equations.  Nothing is written until every check passed.
  // Timings (host clock around work that ends in a stream synchronise): h2d_ms = upload and point checks, witness_map_ms
  // = the field work, msm_ms[0] / msm_ms[1] = the key-side / transcript-side MSMs, total_ms = the whole call.
  int pk_verify_pairs(const g16_srs_desc* srs, const g16_pk_check_desc* pk, const uint64_t* rho_, uint32_t flags,
                      uint64_t* pairs_g1, uint64_t* pairs_g2) override {
    if (!srs || !pk || !rho_ || !pairs_g1 || !pairs_g2) return fail(G16_ERR_BAD_ARGUMENT, "null argument");
    if (flags & ~(uint32_t)(G16_SER_VALIDATE | G16_PK_UNCONTRIBUTED))
      return fail(G16_ERR_BAD_ARGUMENT, "g16_pk_verify_pairs takes G16_SER_VALIDATE and G16_PK_UNCONTRIBUTED only");
    const Fr rho = load_fr(rho_);
    if (rho.is_zero()) return fail(G16_ERR_BAD_ARGUMENT, "the challenge rho must be non-zero");
    if (!have_circuit) return fail(G16_ERR_BAD_ARGUMENT, "g16_circuit_load must precede g16_pk_verify_pairs");
    const uint64_t n = 1ull << L, nv = nvars(), hn = h_query_len(), ni = num_inputs, nw = num_witness;
    const uint32_t nc = num_constraints;
    const uint64_t* kp[PKV_MEMBERS] = {pk->a_query, pk->b_g1_query, pk->b_g2_query, pk->h_query, pk->l_query, pk->gamma_abc_g1,
                                       pk->alpha_g1, pk->beta_g1,    pk->delta_g1,   pk->beta_g2, pk->gamma_g2, pk->delta_g2};
    const uint64_t klen[PKV_MEMBERS] = {nv, nv, nv, hn, nw, ni, 1, 1, 1, 1, 1, 1};
    for (int m = 0; m < PKV_MEMBERS; m++)
      if (!kp[m] && klen[m]) return fail(G16_ERR_BAD_ARGUMENT, std::string("null pk member ") + pkv_member(m));
    const uint64_t* sp[SRS_MEMBERS] = {srs->tau_g1, srs->tau_g2, srs->alpha_tau_g1, srs->beta_tau_g1, srs->beta_g2};
    const uint64_t have[SRS_MEMBERS] = {srs->tau_g1_len, srs->tau_g2_len, srs->alpha_tau_g1_len, srs->beta_tau_g1_len, 1};
    const uint64_t need[SRS_MEMBERS] = {2 * n - 1, n, n, n, 1};   // the prefixes g16_setup_from_srs reads
    for (int m = 0; m < SRS_MEMBERS; m++) {
      if (!sp[m]) return fail(G16_ERR_BAD_ARGUMENT, std::string("null srs member ") + srs_member(m));
      if (have[m] < need[m])
        return fail(G16_ERR_BAD_ARGUMENT, std::string(srs_member(m)) + " holds " + std::to_string(have[m]) +
                                              " points, the circuit (domain 2^" + std::to_string(L) + ") needs at least " +
                                              std::to_string(need[m]));
    }
    G16_NOT_BUSY();
    G16_CUDA(cudaSetDevice(device));
    int rc = ensure_circuit_domain();   // dom: the circuit's twiddles and n^-1
    if (rc) return rc;
    const auto t0 = std::chrono::steady_clock::now();
    auto ms_since = [](std::chrono::steady_clock::time_point a) {
      return (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count();
    };
    tm = g16_timings{};
    cudaStream_t st = S0.st_main;
    // --- upload and check every key member and transcript prefix; one error word ---
    DevBuf kd[PKV_MEMBERS], sd[SRS_MEMBERS], err;
    G16_CUDA(err.reserve(8));
    G16_CUDA(cudaMemsetAsync(err.p, 0xff, 8, st));
    unsigned long long* e = err.template as<unsigned long long>();
    auto upload = [&](DevBuf& d, const uint64_t* p, uint64_t cnt, bool g2, uint32_t member) -> cudaError_t {
      const size_t bytes = cnt * (g2 ? sizeof(A2) : sizeof(A1));
      cudaError_t x = d.reserve(bytes + sizeof(A2));
      if (x != cudaSuccess || !cnt) return x;
      if ((x = cudaMemcpyAsync(d.p, p, bytes, cudaMemcpyHostToDevice, st)) != cudaSuccess) return x;
      tm.h2d_bytes += bytes;
      tm.launches++;
      const uint32_t fl = flags & G16_SER_VALIDATE;
      return g2 ? srs_check<CP, true>(st, d.p, (uint32_t)cnt, fl, member, e) : srs_check<CP, false>(st, d.p, (uint32_t)cnt, fl, member, e);
    };
    for (int m = 0; m < PKV_MEMBERS; m++) G16_CUDA(upload(kd[m], kp[m], klen[m], pkv_g2(m), m));
    for (int m = 0; m < SRS_MEMBERS; m++)
      G16_CUDA(upload(sd[m], sp[m], need[m], m == SRS_TAU_G2 || m == SRS_BETA_G2, PKV_SRS + m));
    unsigned long long first_err = 0;
    G16_CUDA(cudaMemcpyAsync(&first_err, err.p, 8, cudaMemcpyDeviceToHost, st));
    G16_CUDA(cudaStreamSynchronize(st));
    tm.d2h_bytes += 8;
    if (first_err != ~0ull)
      return fail(G16_ERR_INVALID_DATA, std::string(pkv_member((int)(first_err >> 48))) + "[" +
                                            std::to_string((first_err >> 8) & ((1ull << 40) - 1)) + "]: " + ser_reason(first_err & 0xff));
    tm.h2d_ms = ms_since(t0);
    // --- the checks that need no MSM: affine limbs are canonical here, so equal points have equal limbs ---
    auto same = [](const uint64_t* a, const uint64_t* b, size_t bytes) { return memcmp(a, b, bytes) == 0; };
    auto is_inf = [](const uint64_t* a, size_t bytes) { return std::all_of(a, a + bytes / 8, [](uint64_t x) { return x == 0; }); };
    if (is_inf(sp[SRS_TAU_G1], sizeof(A1))) return fail(G16_ERR_INVALID_DATA, "tau_g1[0]: point is the identity");
    if (is_inf(sp[SRS_TAU_G2], sizeof(A2))) return fail(G16_ERR_INVALID_DATA, "tau_g2[0]: point is the identity");
    if (!same(kp[PKV_ALPHA], sp[SRS_ALPHA], sizeof(A1)))
      return fail(G16_ERR_INVALID_DATA, "alpha_g1: not alpha_tau_g1[0] of the transcript");
    if (!same(kp[PKV_BETA], sp[SRS_BETA], sizeof(A1))) return fail(G16_ERR_INVALID_DATA, "beta_g1: not beta_tau_g1[0] of the transcript");
    if (!same(kp[PKV_BETA2], sp[SRS_BETA_G2], sizeof(A2))) return fail(G16_ERR_INVALID_DATA, "beta_g2: not beta_g2 of the transcript");
    for (int m : {PKV_DELTA1, PKV_DELTA2, PKV_GAMMA2})
      if (is_inf(kp[m], pkv_g2(m) ? sizeof(A2) : sizeof(A1))) return fail(G16_ERR_INVALID_DATA, std::string(pkv_member(m)) + ": point is the identity");
    if (!(flags & G16_PK_UNCONTRIBUTED) && same(kp[PKV_GAMMA2], kp[PKV_DELTA2], sizeof(A2)))
      return fail(G16_ERR_INVALID_DATA, "gamma_g2 equals delta_g2: anyone can forge proofs under this key (G16_PK_UNCONTRIBUTED "
                                        "accepts the uncontributed key of a ceremony)");
    // --- field work: P = rho^j (j < max(nv, n)); Z = [z^I | z^L | z]; X = A, B, C times the three (9 vectors of n); T = their
    // inverse transforms (a^I, a^L, a^, b^I, b^L, b^, c^I, c^L, c^); H = the H weights ---
    auto t1 = std::chrono::steady_clock::now();
    const unsigned long long nl0 = ntt_launches;
    const bool circom = qap == G16_QAP_CIRCOM;
    const uint64_t np = std::max(nv, n), nh = 2 * n - 1;
    Fr tab[64];   // rho^(2^k), then omega_2n^-(2^k)
    tab[0] = rho;
    tab[32] = Fr::inv(fr_domain_root<Fr>(L + 1));
    for (int k = 1; k < 32; k++) { tab[k] = Fr::sqr(tab[k - 1]); tab[32 + k] = Fr::sqr(tab[31 + k]); }
    DevBuf dtab, dpow, dz, dx, dt, dh, df;
    G16_CUDA(dtab.reserve(sizeof(tab)));
    G16_CUDA(dpow.reserve(np * sizeof(Fr)));
    G16_CUDA(dz.reserve(3 * nv * sizeof(Fr)));
    G16_CUDA(dx.reserve(9 * n * sizeof(Fr)));
    G16_CUDA(dt.reserve(9 * n * sizeof(Fr)));
    G16_CUDA(dh.reserve(2 * n * sizeof(Fr)));
    G16_CUDA(cudaMemcpyAsync(dtab.p, tab, sizeof(tab), cudaMemcpyHostToDevice, st));
    tm.h2d_bytes += sizeof(tab);
    const Fr* dtab_rho = dtab.template as<Fr>();
    Fr *P = dpow.template as<Fr>(), *Z = dz.template as<Fr>(), *X = dx.template as<Fr>(), *T = dt.template as<Fr>();
    Fr* H = dh.template as<Fr>();
    G16_CUDA(srs_powers<Fr>(st, dtab_rho, Fr::one(), (uint32_t)np, P));
    G16_CUDA(cudaMemsetAsync(Z, 0, 2 * nv * sizeof(Fr), st));
    G16_CUDA(cudaMemcpyAsync(Z, P, ni * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
    if (nw) G16_CUDA(cudaMemcpyAsync(Z + nv + ni, P + ni, nw * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
    G16_CUDA(cudaMemcpyAsync(Z + 2 * nv, P, nv * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
    CsrDev cs[3];
    csr_dev(cs);
    r1cs_matvec<Fr>(st, cs, Z, nc, (uint32_t)ni, (uint32_t)n, X, X + 3 * n, X + 6 * n, 3, (uint32_t)nv, true);
    const Fr zero = Fr::zero();
    ntt_any(st, dom, true, X, X, T, NTT_LOAD_PLAIN, nullptr, nullptr, nullptr, zero, NTT_STORE_MUL_CONST, nullptr, dom.n_inv, 9);
    if (!circom) {
      G16_CUDA(srs_h_weights<Fr>(st, dtab_rho, Fr::one(), nullptr, (uint32_t)n, (uint32_t)nh, H));
    } else {   // F = the unscaled inverse transform of rho^i (i < n) into df + n, df as the work buffer
      G16_CUDA(df.reserve(2 * n * sizeof(Fr)));
      Fr* F = df.template as<Fr>();
      ntt_any(st, dom, true, P, F, F + n, NTT_LOAD_PLAIN, nullptr, nullptr, nullptr, zero, NTT_STORE_PLAIN, nullptr, zero);
      G16_CUDA(srs_h_weights<Fr>(st, dtab_rho + 32, Fr::inv(fr_from_u64<Fr>(2 * n)), F + n, (uint32_t)n, (uint32_t)nh, H));
    }
    G16_CUDA(cudaGetLastError());
    G16_CUDA(cudaStreamSynchronize(st));
    dx.release();
    df.release();
    tm.launches += 3 + (ntt_launches - nl0);   // powers, matvec, H weights, the transforms
    tm.witness_map_ms = ms_since(t1);
    // --- MSMs: the key's sums under rho^j, then the transcript's under the weights ---
    t1 = std::chrono::steady_clock::now();
    MsmWorkspace<Fq> ws1;
    MsmWorkspace<Fq2> ws2;
    MsmCounters mc;
    DevBuf dmask;
    G16_CUDA(dmask.reserve(std::max(nv, 2 * n)));
    uint8_t* mk = dmask.template as<uint8_t>();
    auto g1sum = [&](DevBuf& b, const Fr* sc, uint64_t cnt, P1& acc) { return msm_device<Fq>(ws1, mc, false, b.template as<A1>(), sc, cnt, mk, acc); };
    auto g2sum = [&](DevBuf& b, const Fr* sc, uint64_t cnt, P2& acc) { return msm_device<Fq2>(ws2, mc, true, b.template as<A2>(), sc, cnt, mk, acc); };
    P1 kA = P1::inf(), kB1 = P1::inf(), kH = P1::inf(), kL = P1::inf(), kIC = P1::inf();
    P2 kB2 = P2::inf();
    if ((rc = g1sum(kd[PKV_A], P, nv, kA)) || (rc = g1sum(kd[PKV_B1], P, nv, kB1)) || (rc = g2sum(kd[PKV_B2], P, nv, kB2)) ||
        (rc = g1sum(kd[PKV_H], P, hn, kH)) || (rc = g1sum(kd[PKV_L], P + ni, nw, kL)) || (rc = g1sum(kd[PKV_ABC], P, ni, kIC)))
      return rc;
    tm.msm_ms[0] = ms_since(t1);
    tm.msm_pairs[0] = 3 * nv + hn + nw + ni;
    t1 = std::chrono::steady_clock::now();
    P1 tA = P1::inf(), tB1 = P1::inf(), tH = P1::inf(), tL = P1::inf(), tIC = P1::inf();
    P2 tB2 = P2::inf();
    DevBuf &t1d = sd[SRS_TAU_G1], &ad = sd[SRS_ALPHA], &bd = sd[SRS_BETA];
    if ((rc = g1sum(t1d, T + 2 * n, n, tA)) || (rc = g1sum(t1d, T + 5 * n, n, tB1)) || (rc = g2sum(sd[SRS_TAU_G2], T + 5 * n, n, tB2)) ||
        (rc = g1sum(bd, T + n, n, tL)) || (rc = g1sum(ad, T + 4 * n, n, tL)) || (rc = g1sum(t1d, T + 7 * n, n, tL)) ||
        (rc = g1sum(bd, T, n, tIC)) || (rc = g1sum(ad, T + 3 * n, n, tIC)) || (rc = g1sum(t1d, T + 6 * n, n, tIC)) ||
        (rc = g1sum(t1d, H, nh, tH)))
      return rc;
    tm.msm_ms[1] = ms_since(t1);
    tm.msm_pairs[1] = 9 * n + nh;
    tm.launches += mc.launches;
    // --- the sums the call decides itself ---
    const A1 sA[2] = {kA.to_affine(), tA.to_affine()}, sB1[2] = {kB1.to_affine(), tB1.to_affine()};
    const A2 sB2[2] = {kB2.to_affine(), tB2.to_affine()};
    const char* bad = memcmp(&sA[0], &sA[1], sizeof(A1))     ? "a_query"
                      : memcmp(&sB1[0], &sB1[1], sizeof(A1)) ? "b_g1_query"
                      : memcmp(&sB2[0], &sB2[1], sizeof(A2)) ? "b_g2_query"
                                                             : nullptr;
    if (bad) return fail(G16_ERR_INVALID_DATA, std::string(bad) + ": not the key of the resident circuit under this transcript");
    // equation k: e(P_k, Q_k) = e(P'_k, Q'_k), written as P_0, P'_0, .., P_3, P'_3 and Q_0, Q'_0, .., Q_3, Q'_3
    const A1 g1 = load_a1(sp[SRS_TAU_G1]), d1 = load_a1(kp[PKV_DELTA1]);
    const A2 g2 = load_a2(sp[SRS_TAU_G2]), d2 = load_a2(kp[PKV_DELTA2]), gm2 = load_a2(kp[PKV_GAMMA2]);
    const A1 ps[8] = {d1, g1, kH.to_affine(), tH.to_affine(), kL.to_affine(), tL.to_affine(), kIC.to_affine(), tIC.to_affine()};
    const A2 qs[8] = {g2, d2, d2, g2, d2, g2, gm2, g2};
    for (int i = 0; i < 8; i++) {
      store_a1(pairs_g1 + (size_t)i * 2 * NQ64, ps[i]);
      store_a2(pairs_g2 + (size_t)i * G2_64, qs[i]);
    }
    tm.total_ms = ms_since(t0);
    return G16_OK;
  }

  // ---- phase-2 contributions to a key in host memory (g16_pk_contribute) and the proofs of knowledge of a chain of
  // contributions (g16_contribution_chain_pairs) ----
  enum { PKD_H = 0, PKD_L, PKD_DELTA1, PKD_DELTA2, PKD_MEMBERS };
  static const char* pkd_member(int m) {
    static const char* t[PKD_MEMBERS] = {"h_query", "l_query", "delta_g1", "delta_g2"};
    return t[m];
  }
  // g16_pk_contribute: delta_g1, delta_g2 times delta; every h_query and l_query point times delta^-1.  Two passes over h_query
  // and l_query in chunks of at most `cap` points through one device buffer, as g16_srs_contribute: every point (delta_g1 and
  // delta_g2 too, the identity refused there) is uploaded and checked before anything is written to `out`, then each chunk is
  // uploaded again, multiplied in place on the device (srs_scale_affine_kernel) and copied out.  The two single points are
  // multiplied on the host, as g16_setup_contribute does.
  // Timings (host clock around work that ends in a stream synchronise): h2d_ms = the check pass, msm_ms[0] / msm_ms[1] = the
  // transform of h_query / l_query, total_ms = the whole call.
  int pk_contribute(const g16_pk_delta_desc* in, const uint64_t* delta_, uint32_t flags, uint64_t chunk_points,
                    const g16_pk_delta_out* out) override {
    if (!in || !out || !delta_) return fail(G16_ERR_BAD_ARGUMENT, "null argument");
    if (flags & ~(uint32_t)G16_SER_VALIDATE) return fail(G16_ERR_BAD_ARGUMENT, "g16_pk_contribute takes 0 or G16_SER_VALIDATE");
    const uint64_t* src[PKD_MEMBERS] = {in->h_query, in->l_query, in->delta_g1, in->delta_g2};
    uint64_t* dst[PKD_MEMBERS] = {out->h_query, out->l_query, out->delta_g1, out->delta_g2};
    const uint64_t len[PKD_MEMBERS] = {in->h_len, in->l_len, 1, 1};
    const uint64_t olen[PKD_MEMBERS] = {out->h_len, out->l_len, 1, 1};
    const uint64_t esz[PKD_MEMBERS] = {sizeof(A1), sizeof(A1), sizeof(A1), sizeof(A2)};
    for (int m = 0; m < PKD_MEMBERS; m++) {
      const std::string name = pkd_member(m);
      if (olen[m] != len[m])
        return fail(G16_ERR_BAD_ARGUMENT, "out " + name + " holds " + std::to_string(olen[m]) + " points, in " + name + " " +
                                              std::to_string(len[m]) + ": the lengths must be equal");
      if (len[m] >> 32)
        return fail(G16_ERR_BAD_ARGUMENT, name + " holds " + std::to_string(len[m]) + " points, at most 2^32 - 1 are allowed");
      if (len[m] && (!src[m] || !dst[m])) return fail(G16_ERR_BAD_ARGUMENT, "null key member " + name);
    }
    // an output range may be its own input range (in place) and must overlap no other input or output range
    auto overlap = [&](const void* a, int ma, const void* b, int mb) {
      return srs_overlap((uintptr_t)a, len[ma] * esz[ma], (uintptr_t)b, len[mb] * esz[mb]);
    };
    for (int o = 0; o < PKD_MEMBERS; o++)
      for (int m = 0; m < PKD_MEMBERS; m++) {
        if (overlap(dst[o], o, src[m], m) && !(o == m && (const void*)dst[o] == (const void*)src[m]))
          return fail(G16_ERR_BAD_ARGUMENT, std::string("out ") + pkd_member(o) + " overlaps in " + pkd_member(m) +
                                                ": an output may only be the very same array as its own input");
        if (m > o && overlap(dst[o], o, dst[m], m))
          return fail(G16_ERR_BAD_ARGUMENT, std::string("out ") + pkd_member(o) + " overlaps out " + pkd_member(m));
      }
    const Fr d = load_fr(delta_);
    if (d.is_zero()) return fail(G16_ERR_BAD_ARGUMENT, "delta must be invertible (UnexpectedIdentity)");
    G16_NOT_BUSY();
    G16_CUDA(cudaSetDevice(device));
    const auto t0 = std::chrono::steady_clock::now();
    auto ms_since = [](std::chrono::steady_clock::time_point a) {
      return (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count();
    };
    tm = g16_timings{};
    cudaStream_t st = S0.st_main;
    size_t free_b = 0, total_b = 0;
    G16_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const uint64_t cap = srs_chunk_cap(chunk_points, std::max(len[PKD_H], len[PKD_L]), free_b, sizeof(A1));
    DevBuf buf, err;
    G16_CUDA(buf.reserve(std::max<uint64_t>(cap * sizeof(A1), sizeof(A2))));
    G16_CUDA(err.reserve(8));
    // --- check pass: every point, chunk by chunk; the first bad one by member, then index ---
    for (int m = 0; m < PKD_MEMBERS; m++) {
      const bool single = m == PKD_DELTA1 || m == PKD_DELTA2;
      const uint32_t fl = flags | (single ? (uint32_t)SRS_REFUSE_IDENTITY : 0u);
      for (uint64_t i0 = 0; i0 < len[m];) {
        const uint32_t cnt = srs_chunk_len(len[m], i0, cap);
        G16_CUDA(cudaMemcpyAsync(buf.p, (const char*)src[m] + i0 * esz[m], cnt * esz[m], cudaMemcpyHostToDevice, st));
        G16_CUDA(cudaMemsetAsync(err.p, 0xff, 8, st));
        unsigned long long* e = err.template as<unsigned long long>();
        G16_CUDA((m == PKD_DELTA2 ? srs_check<CP, true>(st, buf.p, cnt, fl, m, e) : srs_check<CP, false>(st, buf.p, cnt, fl, m, e)));
        unsigned long long first_err = 0;
        G16_CUDA(cudaMemcpyAsync(&first_err, err.p, 8, cudaMemcpyDeviceToHost, st));
        G16_CUDA(cudaStreamSynchronize(st));
        tm.h2d_bytes += cnt * esz[m];
        tm.d2h_bytes += 8;
        tm.launches++;
        if (first_err != ~0ull)
          return fail(G16_ERR_INVALID_DATA, std::string(pkd_member(m)) +
                                                (single ? std::string()
                                                        : "[" + std::to_string(i0 + ((first_err >> 8) & ((1ull << 40) - 1))) + "]") +
                                                ": " + srs_reason(first_err & 0xff));
        i0 += cnt;
      }
    }
    tm.h2d_ms = ms_since(t0);
    // --- transform pass: h_query and l_query times delta^-1, chunk by chunk ---
    const Fr di = Fr::inv(d);
    for (int m : {PKD_H, PKD_L}) {
      const auto t1 = std::chrono::steady_clock::now();
      for (uint64_t i0 = 0; i0 < len[m];) {
        const uint32_t cnt = srs_chunk_len(len[m], i0, cap);
        G16_CUDA(cudaMemcpyAsync(buf.p, (const char*)src[m] + i0 * esz[m], cnt * esz[m], cudaMemcpyHostToDevice, st));
        G16_CUDA((srs_scale_affine<Fq, Fr>(st, buf.template as<A1>(), cnt, di)));
        G16_CUDA(cudaMemcpyAsync((char*)dst[m] + i0 * esz[m], buf.p, cnt * esz[m], cudaMemcpyDeviceToHost, st));
        tm.h2d_bytes += cnt * esz[m];
        tm.d2h_bytes += cnt * esz[m];
        tm.launches++;
        i0 += cnt;
      }
      G16_CUDA(cudaStreamSynchronize(st));
      tm.msm_ms[m] = ms_since(t1);
    }
    // delta_g1 and delta_g2 are one point each: on the host, as g16_setup_contribute does
    uint32_t k[Fr::N];
    fr_to_canon(d, k);
    store_a1(dst[PKD_DELTA1], P1::from_affine(load_a1(src[PKD_DELTA1])).mul_u32(k, Fr::N).to_affine());
    store_a2(dst[PKD_DELTA2], P2::from_affine(load_a2(src[PKD_DELTA2])).mul_u32(k, Fr::N).to_affine());
    tm.total_ms = ms_since(t0);
    return G16_OK;
  }
  // Members of a contribution record, in the order a refusal names them within one record.  G1 points go to one device
  // buffer as start_g1, end_g1, then (after_g1, s_g1, s_x_g1) per record; G2 points to another as (r_g2, r_x_g2) per record.
  enum { CR_AFTER = 0, CR_S, CR_SX, CR_R, CR_RX, CR_MEMBERS };
  static const char* cr_member(int m) {
    static const char* t[CR_MEMBERS] = {"after_g1", "s_g1", "s_x_g1", "r_g2", "r_x_g2"};
    return t[m];
  }
  // g16_contribution_chain_pairs: every point uploaded once and checked by srs_check_kernel (the identity refused), the end
  // compared with the last record's after_g1, then the 2 count equations written from the host copies.  The G1 and G2
  // uploads have an error word each; the refusal names the earlier of the two bad points by record, then member.
  // Timings (host clock around work that ends in a stream synchronise): h2d_ms = upload and checks, total_ms = the call.
  int contribution_chain_pairs(const uint64_t* start_g1, const uint64_t* end_g1, const g16_contribution_record* rec, uint32_t count,
                               uint32_t flags, uint64_t* pairs_g1, uint64_t* pairs_g2) override {
    if (!start_g1 || !end_g1 || !rec || !pairs_g1 || !pairs_g2) return fail(G16_ERR_BAD_ARGUMENT, "null argument");
    if (count == 0 || count >= (1u << 30))
      return fail(G16_ERR_BAD_ARGUMENT, "count is " + std::to_string(count) + ": a chain has 1 to 2^30 - 1 records");
    if (flags & ~(uint32_t)G16_SER_VALIDATE)
      return fail(G16_ERR_BAD_ARGUMENT, "g16_contribution_chain_pairs takes 0 or G16_SER_VALIDATE");
    for (uint32_t i = 0; i < count; i++) {
      const uint64_t* p[CR_MEMBERS] = {rec[i].after_g1, rec[i].s_g1, rec[i].s_x_g1, rec[i].r_g2, rec[i].r_x_g2};
      for (int m = 0; m < CR_MEMBERS; m++)
        if (!p[m]) return fail(G16_ERR_BAD_ARGUMENT, "records[" + std::to_string(i) + "]." + cr_member(m) + " is null");
    }
    G16_NOT_BUSY();
    G16_CUDA(cudaSetDevice(device));
    const auto t0 = std::chrono::steady_clock::now();
    auto ms_since = [](std::chrono::steady_clock::time_point a) {
      return (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count();
    };
    tm = g16_timings{};
    cudaStream_t st = S0.st_main;
    const uint64_t n1 = 2 + 3ull * count, n2 = 2ull * count, w1 = 2 * NQ64, w2 = G2_64;
    std::vector<uint64_t> h1(n1 * w1), h2(n2 * w2);   // the points as the ABI lays them out, then uploaded as they are
    auto put = [](std::vector<uint64_t>& v, uint64_t at, const uint64_t* p, uint64_t w) { memcpy(v.data() + at * w, p, w * 8); };
    put(h1, 0, start_g1, w1);
    put(h1, 1, end_g1, w1);
    for (uint32_t i = 0; i < count; i++) {
      put(h1, 2 + 3ull * i, rec[i].after_g1, w1);
      put(h1, 3 + 3ull * i, rec[i].s_g1, w1);
      put(h1, 4 + 3ull * i, rec[i].s_x_g1, w1);
      put(h2, 2ull * i, rec[i].r_g2, w2);
      put(h2, 2ull * i + 1, rec[i].r_x_g2, w2);
    }
    DevBuf d1, d2, err;
    G16_CUDA(d1.reserve(n1 * w1 * 8));
    G16_CUDA(d2.reserve(n2 * w2 * 8));
    G16_CUDA(err.reserve(16));
    unsigned long long* e = err.template as<unsigned long long>();
    const uint32_t fl = flags | SRS_REFUSE_IDENTITY;
    G16_CUDA(cudaMemsetAsync(err.p, 0xff, 16, st));
    G16_CUDA(cudaMemcpyAsync(d1.p, h1.data(), n1 * w1 * 8, cudaMemcpyHostToDevice, st));
    G16_CUDA(cudaMemcpyAsync(d2.p, h2.data(), n2 * w2 * 8, cudaMemcpyHostToDevice, st));
    G16_CUDA((srs_check<CP, false>(st, d1.p, (uint32_t)n1, fl, 0, e)));
    G16_CUDA((srs_check<CP, true>(st, d2.p, (uint32_t)n2, fl, 0, e + 1)));
    unsigned long long first_err[2] = {0, 0};
    G16_CUDA(cudaMemcpyAsync(first_err, err.p, 16, cudaMemcpyDeviceToHost, st));
    G16_CUDA(cudaStreamSynchronize(st));
    tm.h2d_bytes = (n1 * w1 + n2 * w2) * 8;
    tm.d2h_bytes = 16;
    tm.launches = 2;
    tm.h2d_ms = ms_since(t0);
    // position of a bad point: (record, member) as a sortable key, start_g1 and end_g1 before every record
    auto where = [](unsigned long long w, bool g2) -> uint64_t {
      const uint64_t k = (w >> 8) & ((1ull << 40) - 1);
      if (g2) return (k / 2 + 1) * CR_MEMBERS + CR_R + k % 2;
      return k < 2 ? k : ((k - 2) / 3 + 1) * CR_MEMBERS + (k - 2) % 3;
    };
    if (first_err[0] != ~0ull || first_err[1] != ~0ull) {
      const bool g2 = first_err[0] == ~0ull || (first_err[1] != ~0ull && where(first_err[1], true) < where(first_err[0], false));
      const uint64_t at = where(first_err[g2], g2);
      const std::string name = at < 2 ? std::string(at ? "end_g1" : "start_g1")
                                       : "records[" + std::to_string(at / CR_MEMBERS - 1) + "]." + cr_member((int)(at % CR_MEMBERS));
      return fail(G16_ERR_INVALID_DATA, name + ": " + srs_reason(first_err[g2] & 0xff));
    }
    // affine limbs are canonical here, so equal points have equal limbs
    if (memcmp(end_g1, rec[count - 1].after_g1, w1 * 8))
      return fail(G16_ERR_INVALID_DATA, "records[" + std::to_string(count - 1) + "].after_g1: not end_g1");
    // equation 2i: (s_i, r_x_i) = (s_x_i, r_i); equation 2i + 1: (D_i, r_x_i) = (D_(i+1), r_i), D_0 = start_g1
    for (uint64_t i = 0; i < count; i++) {
      const uint64_t ps[4] = {3 + 3 * i, 4 + 3 * i, i ? 2 + 3 * (i - 1) : 0, 2 + 3 * i};   // indices into h1
      const uint64_t qs[4] = {2 * i + 1, 2 * i, 2 * i + 1, 2 * i};                         // indices into h2
      for (uint64_t j = 0; j < 4; j++) {
        memcpy(pairs_g1 + (4 * i + j) * w1, h1.data() + ps[j] * w1, w1 * 8);
        memcpy(pairs_g2 + (4 * i + j) * w2, h2.data() + qs[j] * w2, w2 * 8);
      }
    }
    tm.total_ms = ms_since(t0);
    return G16_OK;
  }
  // CircomReduction::h_query_scalars(n - 1, tau, _, delta^-1): the odd entries 1, 3, .., 2n - 1 of the size-2n ifft of
  // v[i] = delta^-1 tau^i (i < 2n - 1), v[2n - 1] = 0.  With w = omega_2n, k = 2j + 1 and the geometric sum in closed form:
  //   out[j] = delta^-1 / (2n) * [ (tau^2n - 1) / (tau w^-k - 1) - tau^(2n-1) w^k ]
  // O(n), one batch inversion.  tn = tau^n; tau^2n != 1 is checked by the caller.
  void circom_h_scalars(const Fr& tau, const Fr& tn, const Fr& di, std::vector<Fr>& hs) const {
    const uint64_t n = hs.size();
    const Fr w = fr_domain_root<Fr>(L + 1), w_inv = Fr::inv(w);
    const Fr w2 = Fr::sqr(w), w2_inv = Fr::sqr(w_inv);
    const Fr t2n = Fr::sqr(tn), t2n_m1 = Fr::sub(t2n, Fr::one());
    Fr tn1 = Fr::one();                                                           // tau^(n-1): n - 1 = L one bits
    for (int i = 0; i < L; i++) tn1 = Fr::mul(Fr::sqr(tn1), tau);
    const Fr t2n1 = Fr::mul(tn, tn1);                                             // tau^(2n-1)
    const Fr c = Fr::mul(di, Fr::inv(fr_from_u64<Fr>(2 * n)));
    std::vector<Fr> den(n), pref(n);
    Fr wk_inv = w_inv;
    for (uint64_t j = 0; j < n; j++) { den[j] = Fr::sub(Fr::mul(tau, wk_inv), Fr::one()); wk_inv = Fr::mul(wk_inv, w2_inv); }
    Fr acc = Fr::one();
    for (uint64_t j = 0; j < n; j++) { pref[j] = acc; acc = Fr::mul(acc, den[j]); }
    Fr ai = Fr::inv(acc);
    for (uint64_t j = n; j-- > 0;) { const Fr t = Fr::mul(ai, pref[j]); ai = Fr::mul(ai, den[j]); den[j] = t; }
    Fr wk = w;
    for (uint64_t j = 0; j < n; j++) {
      hs[j] = Fr::mul(c, Fr::sub(Fr::mul(t2n_m1, den[j]), Fr::mul(t2n1, wk)));
      wk = Fr::mul(wk, w2);
    }
  }
  int pk_export(const g16_pk_export_desc* o) override {
    if (!have_pk || !from_setup) return fail(G16_ERR_BAD_ARGUMENT, "g16_pk_export needs a key produced by g16_setup");
    if (!o) return fail(G16_ERR_BAD_ARGUMENT, "null");
    G16_CUDA(cudaSetDevice(device));
    const uint64_t nv = nvars(), hn = h_query_len();
    if (o->a_query) G16_CUDA(cudaMemcpy(o->a_query, full_a.p, nv * sizeof(A1), cudaMemcpyDeviceToHost));
    if (o->b_g1_query) G16_CUDA(cudaMemcpy(o->b_g1_query, full_b1.p, nv * sizeof(A1), cudaMemcpyDeviceToHost));
    if (o->b_g2_query) G16_CUDA(cudaMemcpy(o->b_g2_query, full_b2.p, nv * sizeof(A2), cudaMemcpyDeviceToHost));
    if (o->h_query && hn) G16_CUDA(cudaMemcpy(o->h_query, q[M_H].bases.p, hn * sizeof(A1), cudaMemcpyDeviceToHost));
    if (o->l_query && num_witness) G16_CUDA(cudaMemcpy(o->l_query, q[M_L].bases.p, (size_t)num_witness * sizeof(A1), cudaMemcpyDeviceToHost));
    if (o->gamma_abc_g1) G16_CUDA(cudaMemcpy(o->gamma_abc_g1, d_gamma_abc.p, (size_t)num_inputs * sizeof(A1), cudaMemcpyDeviceToHost));
    store_vk_points(o, gamma_g2);
    return G16_OK;
  }
  // the verifying key's six single points into the non-null members of o
  void store_vk_points(const g16_pk_export_desc* o, const A2& gamma) const {
    if (o->alpha_g1) store_a1(o->alpha_g1, alpha_g1);
    if (o->beta_g1) store_a1(o->beta_g1, beta_g1);
    if (o->delta_g1) store_a1(o->delta_g1, delta_g1);
    if (o->beta_g2) store_a2(o->beta_g2, beta_g2);
    if (o->gamma_g2) store_a2(o->gamma_g2, gamma);
    if (o->delta_g2) store_a2(o->delta_g2, delta_g2);
  }

  // ---- ark-serialized proving keys (ser.cuh) ----
  // Points are decoded in chunks of at most SER_CHUNK (every query of a 2^20 key spans several), staged through two pinned
  // buffers so that the copy of chunk i + 1 overlaps the decode of chunk i; extra device memory does not grow with the key.
  static constexpr uint32_t SER_CHUNK = 1u << 17;
  struct SerStaging {   // released on every return path
    cudaStream_t st_copy = nullptr, st_dec = nullptr;
    cudaEvent_t ev_h2d[2] = {}, ev_dec[2] = {};
    uint8_t* host[2] = {};
    DevBuf dev[2], aux, err;
    uint64_t chunks = 0, h2d_bytes = 0;   // chunks staged so far (buffer chunks & 1 is next), bytes copied up
    unsigned long long launches = 0;      // kernels
    ~SerStaging() {
      if (st_dec) cudaStreamSynchronize(st_dec);
      if (st_copy) cudaStreamSynchronize(st_copy);
      for (int k = 0; k < 2; k++) {
        if (ev_h2d[k]) cudaEventDestroy(ev_h2d[k]);
        if (ev_dec[k]) cudaEventDestroy(ev_dec[k]);
        if (host[k]) cudaFreeHost(host[k]);
      }
      if (st_dec) cudaStreamDestroy(st_dec);
      if (st_copy) cudaStreamDestroy(st_copy);
    }
  };
  // host-bound points in sg.aux: the seven single points, element 0 of a / b_g1 / b_g2, gamma_abc_g1
  enum { AUX_A0 = 7, AUX_B10 = 8, AUX_B20 = 9, AUX_ABC = 10 };
  static size_t ser_aux_bytes(uint64_t n_abc) { return AUX_ABC * sizeof(A2) + (size_t)n_abc * sizeof(A1); }
  // streams, events, the error word (all ones: no error) and zeroed aux; two pinned and two device buffers of `stage` bytes
  int ser_staging_init(SerStaging& sg, size_t stage, size_t aux_bytes) {
    G16_CUDA(cudaStreamCreateWithFlags(&sg.st_copy, cudaStreamNonBlocking));
    G16_CUDA(cudaStreamCreateWithFlags(&sg.st_dec, cudaStreamNonBlocking));
    // reset on the decode stream itself: st_dec does not wait for the legacy default stream, so a plain cudaMemset there
    // could land after the first decodes and wipe their points or their error
    G16_CUDA(sg.aux.reserve(aux_bytes));
    G16_CUDA(cudaMemsetAsync(sg.aux.p, 0, aux_bytes, sg.st_dec));
    G16_CUDA(sg.err.reserve(8));
    G16_CUDA(cudaMemsetAsync(sg.err.p, 0xff, 8, sg.st_dec));
    for (int k = 0; k < 2; k++) {
      G16_CUDA(cudaEventCreateWithFlags(&sg.ev_h2d[k], cudaEventDisableTiming));
      G16_CUDA(cudaEventCreateWithFlags(&sg.ev_dec[k], cudaEventDisableTiming));
      G16_CUDA(cudaHostAlloc((void**)&sg.host[k], stage + 1, cudaHostAllocDefault));
      G16_CUDA(sg.dev[k].reserve(stage + 1));
    }
    return G16_OK;
  }
  // Copies bytes [src, src + n) of the host stream to dst (null: device staging buffer chunks & 1) through pinned buffer
  // chunks & 1, so that the copy of chunk i + 1 overlaps the kernel of chunk i.  On return st_dec waits for the copy: the
  // caller enqueues the chunk's kernel there, then ser_chunk_done.
  int ser_chunk_upload(SerStaging& sg, const uint8_t* src, size_t n, void* dst) {
    const int k = (int)(sg.chunks & 1);
    if (sg.chunks >= 2) G16_CUDA(cudaEventSynchronize(sg.ev_h2d[k]));   // pinned buffer k is free again
    memcpy(sg.host[k], src, n);
    if (sg.chunks >= 2) G16_CUDA(cudaStreamWaitEvent(sg.st_copy, sg.ev_dec[k], 0));   // the kernel that read dev[k] is done
    G16_CUDA(cudaMemcpyAsync(dst ? dst : sg.dev[k].p, sg.host[k], n, cudaMemcpyHostToDevice, sg.st_copy));
    G16_CUDA(cudaEventRecord(sg.ev_h2d[k], sg.st_copy));
    G16_CUDA(cudaStreamWaitEvent(sg.st_dec, sg.ev_h2d[k], 0));
    sg.h2d_bytes += n;
    return G16_OK;
  }
  int ser_chunk_done(SerStaging& sg) {
    G16_CUDA(cudaEventRecord(sg.ev_dec[sg.chunks & 1], sg.st_dec));
    sg.chunks++;
    sg.launches++;
    return G16_OK;
  }
  // Decodes the points of `plan` (MONT: the .zkey encoding, else the ark one `flags` selects) into this rank's bases of
  // every query and the host-bound points of sg.aux, as g16_pk_load places them.  place = false only checks them.  A refused
  // point lands in sg.err.
  template <bool MONT>
  int ser_decode_points(SerStaging& sg, const uint8_t* bytes, const SerItem it[SER_ITEMS], const std::vector<SerChunk>& plan,
                        uint32_t flags, bool place) {
    auto aux_at = [&](int slot) { return (char*)sg.aux.p + (size_t)slot * sizeof(A2); };
    for (const SerChunk& c : plan) {
      const SerItem& x = it[c.member];
      int rc = ser_chunk_upload(sg, bytes + c.off, (size_t)c.count * x.psize, nullptr);
      if (rc) return rc;
      SerDest d;
      d.rank = rank;
      d.world = world;
      d.aux_n = 1;
      switch (c.member) {
        case SER_GAMMA_ABC: d.aux = aux_at(AUX_ABC); d.aux_n = x.len; break;
        case SER_A: d.aux = aux_at(AUX_A0); d.bases = q[M_A].bases.p; d.skip = 1; d.pairs = q[M_A].pairs; break;
        case SER_B_G1: d.aux = aux_at(AUX_B10); d.bases = q[M_B1].bases.p; d.skip = 1; d.pairs = q[M_B1].pairs; break;
        case SER_B_G2: d.aux = aux_at(AUX_B20); d.bases = q[M_B2].bases.p; d.skip = 1; d.pairs = q[M_B2].pairs; break;
        case SER_H: d.aux_n = 0; d.bases = q[M_H].bases.p; d.pairs = q[M_H].pairs; break;
        case SER_L: d.aux_n = 0; d.bases = q[M_L].bases.p; d.pairs = q[M_L].pairs; break;
        default: d.aux = aux_at(c.member); break;   // single points: slots 0 .. 6 in stream order
      }
      if (!place) d = SerDest{};
      const uint8_t* src = sg.dev[sg.chunks & 1].template as<uint8_t>();
      unsigned long long* err = sg.err.template as<unsigned long long>();
      const cudaError_t e = x.g2 ? ser_decode_enqueue<CP, true, MONT>(sg.st_dec, src, c.first, c.count, flags, c.off, d, err)
                                 : ser_decode_enqueue<CP, false, MONT>(sg.st_dec, src, c.first, c.count, flags, c.off, d, err);
      G16_CUDA(e);
      if ((rc = ser_chunk_done(sg))) return rc;
    }
    return G16_OK;
  }
  // After the decodes: the single points from sg.aux into the key, commit_key, and the verifying key into vk (if non-null)
  int ser_commit(SerStaging& sg, const g16_pk_export_desc* vk) {
    const size_t aux_bytes = ser_aux_bytes(num_inputs);
    std::vector<char> aux(aux_bytes);
    G16_CUDA(cudaMemcpy(aux.data(), sg.aux.p, aux_bytes, cudaMemcpyDeviceToHost));
    auto a1 = [&](int slot) { A1 r; memcpy(&r, aux.data() + (size_t)slot * sizeof(A2), sizeof(A1)); return r; };
    auto a2 = [&](int slot) { A2 r; memcpy(&r, aux.data() + (size_t)slot * sizeof(A2), sizeof(A2)); return r; };
    alpha_g1 = a1(SER_ALPHA_G1); beta_g1 = a1(SER_BETA_G1); delta_g1 = a1(SER_DELTA_G1);
    beta_g2 = a2(SER_BETA_G2); delta_g2 = a2(SER_DELTA_G2);
    int rc = commit_key(a1(AUX_A0), a1(AUX_B10), a2(AUX_B20), false);
    if (rc) return rc;
    if (vk) {
      store_vk_points(vk, a2(SER_GAMMA_G2));
      if (vk->gamma_abc_g1)
        for (uint32_t i = 0; i < num_inputs; i++) {
          A1 p;
          memcpy(&p, aux.data() + AUX_ABC * sizeof(A2) + (size_t)i * sizeof(A1), sizeof(A1));
          store_a1(vk->gamma_abc_g1 + (size_t)i * 2 * NQ64, p);
        }
    }
    return G16_OK;
  }
  static size_t ser_stage_bytes(const SerItem it[SER_ITEMS], const std::vector<SerChunk>& plan) {
    size_t stage = 0;
    for (const SerChunk& c : plan) stage = std::max<size_t>(stage, (size_t)c.count * it[c.member].psize);
    return stage;
  }
  int pk_load_serialized(const uint8_t* bytes, uint64_t len, uint32_t flags, uint32_t rk, uint32_t wd,
                         const g16_pk_export_desc* vk) override {
    using Fmt = SerFormat<CP>;
    if (!have_circuit) return fail(G16_ERR_BAD_ARGUMENT, "g16_circuit_load must precede g16_pk_load_serialized");
    if ((!bytes && len) || wd == 0 || rk >= wd) return fail(G16_ERR_BAD_ARGUMENT, "bad bytes / rank / world");
    if (flags & ~(uint32_t)(G16_SER_COMPRESSED | G16_SER_VALIDATE)) return fail(G16_ERR_BAD_ARGUMENT, "unknown serialization flags");
    if (vk && (vk->a_query || vk->b_g1_query || vk->b_g2_query || vk->h_query || vk->l_query))
      return fail(G16_ERR_BAD_ARGUMENT, "vk_out receives the verifying key only: its query members must be NULL");
    G16_NOT_BUSY();
    G16_CUDA(cudaSetDevice(device));
    drop_key();   // from here on a rejected key leaves no key resident
    SerItem it[SER_ITEMS];
    const std::string why = ser_walk(bytes, len, Fmt::NB, flags & G16_SER_COMPRESSED, it, Fmt::G2_NC);
    if (!why.empty()) return fail(G16_ERR_INVALID_DATA, why);
    if (it[SER_GAMMA_ABC].len != num_inputs)
      return fail(G16_ERR_MALFORMED_KEY, "vk.gamma_abc_g1 holds " + std::to_string(it[SER_GAMMA_ABC].len) +
                                             " points, the circuit has " + std::to_string(num_inputs) + " instance variables");
    const uint64_t qlen[5] = {it[SER_H].len, it[SER_L].len, it[SER_A].len, it[SER_B_G1].len, it[SER_B_G2].len};
    int rc = begin_key(rk, wd, qlen);   // the same truncation and shards as g16_pk_load
    if (rc) return rc;
    const std::vector<SerChunk> plan = ser_plan(it, SER_CHUNK);
    SerStaging sg;
    if ((rc = ser_staging_init(sg, ser_stage_bytes(it, plan), ser_aux_bytes(num_inputs)))) return rc;
    if ((rc = ser_decode_points<false>(sg, bytes, it, plan, flags, true))) return rc;
    G16_CUDA(cudaStreamSynchronize(sg.st_dec));
    unsigned long long first_err = 0;
    G16_CUDA(cudaMemcpy(&first_err, sg.err.p, 8, cudaMemcpyDeviceToHost));
    if (first_err != ~0ull) {
      const uint64_t off = first_err >> 8;
      return fail(G16_ERR_INVALID_DATA, ser_locate(it, off) + " (byte " + std::to_string(off) + "): " + ser_reason(first_err & 0xff));
    }
    return ser_commit(sg, vk);
  }

  // ---- snarkjs .zkey files (zkey.cuh): the circuit's A and B and its key in one call ----
  // Host: zkey_walk decides the section table, every size and the header before anything resident is released.  Device,
  // on the staging streams: the coefficient section goes chunk by chunk into one device copy, each chunk decoded in place
  // (zkey_coef_kernel); then the circuit is derived from the largest constraint index and the CSR arrays are built
  // (zkey_csr_enqueue) while the points are decoded and placed like an ark key's.  Every refusal after the host checks
  // leaves neither a circuit nor a key resident.
  int zkey_load(const uint8_t* bytes, uint64_t len, uint32_t flags, uint32_t rk, uint32_t wd, const g16_pk_export_desc* vk,
                g16_zkey_info* info) override {
    if constexpr (CP::CURVE_ID != 0 && CP::CURVE_ID != 1) {
      return fail(G16_ERR_BAD_ARGUMENT, "snarkjs .zkey files exist for BN254 and BLS12-381 only");
    } else {
      if ((!bytes && len) || wd == 0 || rk >= wd) return fail(G16_ERR_BAD_ARGUMENT, "bad bytes / rank / world");
      if (flags & ~(uint32_t)(G16_SER_VALIDATE | G16_ZKEY_KEY_ONLY))
        return fail(G16_ERR_BAD_ARGUMENT, "g16_zkey_load takes G16_SER_VALIDATE and G16_ZKEY_KEY_ONLY only");
      if (vk && (vk->a_query || vk->b_g1_query || vk->b_g2_query || vk->h_query || vk->l_query))
        return fail(G16_ERR_BAD_ARGUMENT, "vk_out receives the verifying key only: its query members must be NULL");
      G16_NOT_BUSY();
      const bool key_only = flags & G16_ZKEY_KEY_ONLY;
      flags &= ~(uint32_t)G16_ZKEY_KEY_ONLY;
      if (key_only && (!have_circuit || qap != G16_QAP_CIRCOM))
        return fail(G16_ERR_BAD_ARGUMENT, "G16_ZKEY_KEY_ONLY needs a resident circuit under G16_QAP_CIRCOM (a .zkey holds a "
                                          "CircomReduction key)");
      ZkeyLayout z;
      const std::string why = zkey_walk<CP>(bytes, len, z);
      if (!why.empty()) return fail(G16_ERR_INVALID_DATA, why);
      if (key_only) return zkey_key_only(bytes, z, flags, rk, wd, vk, info);
      int Ln = 0;
      while ((1u << Ln) < z.domain_size) Ln++;
      int rc = check_log((uint32_t)Ln);
      if (rc) return rc;
      if (Ln + 1 > CP::FrP::TWO_ADICITY)
        return fail(G16_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "CircomReduction needs a domain of twice the size, which exceeds the field's two-adicity (PolynomialDegreeTooLarge)");
      G16_CUDA(cudaSetDevice(device));
      const auto t0 = std::chrono::steady_clock::now();
      const unsigned long long launches0 = ntt_launches + ctr.launches;
      tm = g16_timings{};
      // from here on a refusal leaves neither a circuit nor a key resident
      drop_key();
      have_circuit = false;
      circuit_without_c = true;
      for (int m = 0; m < 3; m++) { h_rp[m].clear(); h_col[m].clear(); h_val[m].clear(); }
      const uint32_t ds = z.domain_size;
      const std::vector<SerChunk> plan = ser_plan(z.it, SER_CHUNK);
      SerStaging sg;
      if ((rc = ser_staging_init(sg, std::max<size_t>(ser_stage_bytes(z.it, plan), (size_t)SER_CHUNK * z.rs),
                                 ser_aux_bytes(z.npub + 1ull))))
        return rc;
      // coefficients: every record into one device copy, decoded in place chunk by chunk
      DevBuf d_rec, d_counts, d_small;
      G16_CUDA(d_rec.reserve((size_t)z.ncoefs * z.rs + 4));
      G16_CUDA(d_counts.reserve((size_t)2 * ds * 4));
      G16_CUDA(d_small.reserve(8));   // row_end, then pub_err
      G16_CUDA(cudaMemsetAsync(d_counts.p, 0, (size_t)2 * ds * 4, sg.st_dec));
      G16_CUDA(cudaMemsetAsync(d_small.p, 0, 4, sg.st_dec));
      G16_CUDA(cudaMemsetAsync((char*)d_small.p + 4, 0xff, 4, sg.st_dec));
      uint8_t* rec = d_rec.template as<uint8_t>();
      uint32_t* counts = d_counts.template as<uint32_t>();
      uint32_t* row_end = d_small.template as<uint32_t>();
      uint32_t* pub_err = row_end + 1;
      unsigned long long* err = sg.err.template as<unsigned long long>();
      for (uint64_t f = 0; f < z.ncoefs; f += SER_CHUNK) {
        const uint32_t cnt = (uint32_t)std::min<uint64_t>(SER_CHUNK, z.ncoefs - f);
        if ((rc = ser_chunk_upload(sg, bytes + z.coef_off + f * z.rs, (size_t)cnt * z.rs, rec + f * z.rs))) return rc;
        G16_CUDA(zkey_coef_enqueue<Fr>(sg.st_dec, rec + f * z.rs, cnt, z.rs, z.coef_off + f * z.rs, ds, z.nvars, counts, row_end, err));
        if ((rc = ser_chunk_done(sg))) return rc;
      }
      uint32_t small[2];
      unsigned long long coef_err = 0;
      G16_CUDA(cudaStreamSynchronize(sg.st_dec));
      G16_CUDA(cudaMemcpy(small, d_small.p, 8, cudaMemcpyDeviceToHost));
      G16_CUDA(cudaMemcpy(&coef_err, sg.err.p, 8, cudaMemcpyDeviceToHost));
      uint32_t nc = 0;
      std::string derived;   // why the coefficients do not make a circuit of this file, decided once every item has passed
      if (coef_err == ~0ull) derived = zkey_derive(z, small[0], &nc);
      const bool place = coef_err == ~0ull && derived.empty();
      uint64_t nnz[2] = {0, 0};
      uint32_t nnz_u32[2] = {0, 0};
      if (place) {
        // the circuit: A and B in CSR, C resident empty, the CircomReduction domain
        num_inputs = z.npub + 1; num_constraints = nc; num_witness = z.nvars - z.npub - 1; L = Ln; qap = G16_QAP_CIRCOM;
        for (int m = 0; m < 3; m++) {
          G16_CUDA(csr_rp[m].reserve((size_t)(nc + 1) * 4));
          G16_CUDA(cudaMemsetAsync(csr_rp[m].p, 0, (size_t)(nc + 1) * 4, sg.st_dec));
        }
        DevBuf block_tot;
        G16_CUDA(block_tot.reserve(((size_t)nc + 1 + 1023) / 1024 * 4 + 4));
        G16_CUDA(zkey_row_ptr_enqueue(sg.st_dec, counts, nc, z.npub, ds, csr_rp[0].template as<uint32_t>(),
                                      csr_rp[1].template as<uint32_t>(), block_tot.template as<uint32_t>(), pub_err, &sg.launches));
        for (int m = 0; m < 2; m++)   // the sizes of col / val: the last entry of each row_ptr
          G16_CUDA(cudaMemcpyAsync(&nnz_u32[m], csr_rp[m].template as<uint32_t>() + nc, 4, cudaMemcpyDeviceToHost, sg.st_dec));
        G16_CUDA(cudaStreamSynchronize(sg.st_dec));
        for (int m = 0; m < 3; m++) {
          const uint64_t e = m < 2 ? nnz_u32[m] : 0;
          if (m < 2) nnz[m] = e;
          G16_CUDA(csr_col[m].reserve((size_t)e * 4 + 4));
          G16_CUDA(csr_val[m].reserve((size_t)e * sizeof(Fr) + sizeof(Fr)));
        }
        const ZkeyCsr ca{csr_rp[0].template as<uint32_t>(), csr_col[0].template as<uint32_t>(), csr_val[0].p};
        const ZkeyCsr cb{csr_rp[1].template as<uint32_t>(), csr_col[1].template as<uint32_t>(), csr_val[1].p};
        G16_CUDA(zkey_scatter_enqueue<Fr>(sg.st_dec, rec, z.ncoefs, SER_CHUNK, z.rs, nc, ds, counts, ca, cb, pub_err, &sg.launches));
        G16_CUDA(cudaStreamSynchronize(sg.st_dec));
        // the records and counts are done with: freed before begin_key reserves the bases and commit_key weighs the free
        // memory (a 2^24 circuit's records take gigabytes)
        d_rec.release();
        d_counts.release();
        G16_CUDA(cudaMemcpy(&small[1], pub_err, 4, cudaMemcpyDeviceToHost));
        if (small[1] != UINT32_MAX) {
          const uint32_t s = small[1] >> 1;
          return fail(G16_ERR_INVALID_DATA, "coefficients: public-input row " + std::to_string(s) +
                                                (small[1] & 1 ? " of B is not empty" : " of A is not {(" + std::to_string(s) + ", 1)}"));
        }
        G16_CUDA(S0.d_z.reserve((size_t)z.nvars * sizeof(Fr)));
        if ((rc = ensure_circuit_domain())) return rc;
        // the key, placed for this circuit
        const uint64_t qlen[5] = {z.it[SER_H].len, z.it[SER_L].len, z.it[SER_A].len, z.it[SER_B_G1].len, z.it[SER_B_G2].len};
        if ((rc = begin_key(rk, wd, qlen))) return rc;
      }
      const auto t2 = std::chrono::steady_clock::now();
      // the points: placed when the circuit stands, otherwise only checked, so that the first bad item in the file is named
      if ((rc = ser_decode_points<true>(sg, bytes, z.it, plan, flags, place))) return rc;
      G16_CUDA(cudaStreamSynchronize(sg.st_dec));
      unsigned long long first_err = 0;
      G16_CUDA(cudaMemcpy(&first_err, sg.err.p, 8, cudaMemcpyDeviceToHost));
      if (first_err != ~0ull) {
        const uint64_t off = first_err >> 8;
        const uint32_t code = first_err & 0xff;
        if (off >= z.coef_off && off < z.coef_off + (uint64_t)z.ncoefs * z.rs)
          return fail(G16_ERR_INVALID_DATA, zkey_coef_reason(bytes, z, off, code));
        return fail(G16_ERR_INVALID_DATA, zkey_locate(z, off) + " (byte " + std::to_string(off) + "): " + ser_reason(code));
      }
      if (!derived.empty()) return fail(G16_ERR_INVALID_DATA, derived);
      for (DevBuf& b : sg.dev) b.release();   // likewise the staging buffers, before commit_key weighs the free memory
      have_circuit = true;
      if ((rc = ser_commit(sg, vk))) { have_circuit = false; return rc; }
      const auto t3 = std::chrono::steady_clock::now();
      auto ms = [](auto a, auto b) { return std::chrono::duration<float, std::milli>(b - a).count(); };
      tm.total_ms = ms(t0, t3);
      tm.witness_map_ms = ms(t0, t2);
      tm.h2d_ms = ms(t2, t3);
      tm.h2d_bytes = sg.h2d_bytes;
      tm.d2h_bytes = 8 + 8 + 4 + 8 + ser_aux_bytes(num_inputs);
      tm.launches = sg.launches + (ntt_launches + ctr.launches - launches0);
      if (info) *info = g16_zkey_info{num_inputs, num_constraints, num_witness, (uint32_t)L, nnz[0], nnz[1]};
      return G16_OK;
    }
  }
  // G16_ZKEY_KEY_ONLY: the walked file's key onto the resident circuit (section 4 is not read).  The sizes are decided
  // before begin_key drops the previous key; a refused point leaves the circuit and no key.
  int zkey_key_only(const uint8_t* bytes, const ZkeyLayout& z, uint32_t flags, uint32_t rk, uint32_t wd, const g16_pk_export_desc* vk,
                    g16_zkey_info* info) {
    if ((uint64_t)z.nvars != nvars())
      return fail(G16_ERR_MALFORMED_KEY, "section 2: nVars = " + std::to_string(z.nvars) + ", the resident circuit has " +
                                             std::to_string(nvars()) + " variables");
    if (z.npub + 1ull != num_inputs)
      return fail(G16_ERR_MALFORMED_KEY, "section 2: nPublic + 1 = " + std::to_string(z.npub + 1ull) +
                                             ", the resident circuit has " + std::to_string(num_inputs) + " instance variables");
    if ((uint64_t)z.domain_size != 1ull << L)
      return fail(G16_ERR_MALFORMED_KEY, "section 2: domainSize = " + std::to_string(z.domain_size) +
                                             ", the resident circuit's domain is " + std::to_string(1ull << L));
    G16_CUDA(cudaSetDevice(device));
    const auto t0 = std::chrono::steady_clock::now();
    tm = g16_timings{};
    const uint64_t qlen[5] = {z.it[SER_H].len, z.it[SER_L].len, z.it[SER_A].len, z.it[SER_B_G1].len, z.it[SER_B_G2].len};
    int rc = begin_key(rk, wd, qlen);
    if (rc) return rc;
    const std::vector<SerChunk> plan = ser_plan(z.it, SER_CHUNK);
    SerStaging sg;
    if ((rc = ser_staging_init(sg, ser_stage_bytes(z.it, plan), ser_aux_bytes(num_inputs)))) return rc;
    if ((rc = ser_decode_points<true>(sg, bytes, z.it, plan, flags, true))) return rc;
    G16_CUDA(cudaStreamSynchronize(sg.st_dec));
    unsigned long long first_err = 0;
    G16_CUDA(cudaMemcpy(&first_err, sg.err.p, 8, cudaMemcpyDeviceToHost));
    if (first_err != ~0ull) {
      const uint64_t off = first_err >> 8;
      return fail(G16_ERR_INVALID_DATA, zkey_locate(z, off) + " (byte " + std::to_string(off) + "): " + ser_reason(first_err & 0xff));
    }
    for (DevBuf& b : sg.dev) b.release();
    if ((rc = ser_commit(sg, vk))) return rc;
    tm.total_ms = tm.h2d_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    tm.h2d_bytes = sg.h2d_bytes;
    tm.d2h_bytes = 8 + ser_aux_bytes(num_inputs);
    tm.launches = sg.launches;
    const uint64_t nnz[2] = {h_rp[0].empty() ? 0 : h_rp[0].back(), h_rp[1].empty() ? 0 : h_rp[1].back()};
    if (info) *info = g16_zkey_info{num_inputs, num_constraints, num_witness, (uint32_t)L, nnz[0], nnz[1]};
    return G16_OK;
  }

  // ---- circom .r1cs circuits and .wtns witnesses (r1cs.cuh) ----
  // Host: r1cs_walk decides the section table, the header, every term count, the three row_ptr arrays and the domain
  // before anything resident is released; reading the counts is the format's only serial dependence.  Device, on the
  // staging streams: the constraint section goes up in chunks of at most SER_CHUNK terms (and of at most the staging size in
  // bytes), each decoded by one thread per term straight into the resident CSR arrays.  A refused term leaves neither a
  // circuit nor a key resident.
  int r1cs_load(int qp, const uint8_t* bytes, uint64_t len, g16_r1cs_info* info) override {
    if (qp != G16_QAP_LIBSNARK && qp != G16_QAP_CIRCOM) return fail(G16_ERR_BAD_ARGUMENT, "unknown R1CS-to-QAP reduction");
    if (!bytes) return fail(G16_ERR_BAD_ARGUMENT, "null bytes");
    G16_NOT_BUSY();
    const auto t0 = std::chrono::steady_clock::now();
    R1csLayout z;
    const std::string why = r1cs_walk<typename CP::FrP>(bytes, len, z);
    if (!why.empty()) return fail(G16_ERR_INVALID_DATA, why);
    int Ln = 0;
    while ((1ull << Ln) < (uint64_t)z.m + z.num_inputs) Ln++;
    int rc = check_log((uint32_t)Ln);
    if (rc) return rc;
    if (qp == G16_QAP_CIRCOM && Ln + 1 > CP::FrP::TWO_ADICITY)
      return fail(G16_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "CircomReduction needs a domain of twice the size, which exceeds the field's two-adicity (PolynomialDegreeTooLarge)");
    G16_CUDA(cudaSetDevice(device));
    const auto t1 = std::chrono::steady_clock::now();
    const unsigned long long launches0 = ntt_launches + ctr.launches;
    tm = g16_timings{};
    // from here on a refusal leaves neither a circuit nor a key resident
    drop_key();
    have_circuit = false;
    circuit_without_c = false;
    const uint32_t nc = z.m;
    const uint64_t T = z.tp[nc];
    R1csCsr csr;
    for (int m = 0; m < 3; m++) {
      const uint64_t nnz = z.rp[m][nc];
      G16_CUDA(csr_rp[m].reserve((size_t)(nc + 1) * 4));
      G16_CUDA(csr_col[m].reserve((size_t)nnz * 4 + 4));
      G16_CUDA(csr_val[m].reserve((size_t)nnz * sizeof(Fr) + sizeof(Fr)));
      G16_CUDA(cudaMemcpy(csr_rp[m].p, z.rp[m].data(), (size_t)(nc + 1) * 4, cudaMemcpyHostToDevice));
      csr.row_ptr[m] = csr_rp[m].template as<uint32_t>();
      csr.col[m] = csr_col[m].template as<uint32_t>();
      csr.val[m] = csr_val[m].p;
    }
    DevBuf d_tp;
    G16_CUDA(d_tp.reserve((size_t)(nc + 1) * 8));
    G16_CUDA(cudaMemcpy(d_tp.p, z.tp.data(), (size_t)(nc + 1) * 8, cudaMemcpyHostToDevice));
    const size_t stage = (size_t)SER_CHUNK * (z.ts + 12);   // SER_CHUNK terms and a count word per constraint among them
    SerStaging sg;
    if ((rc = ser_staging_init(sg, stage, 8))) return rc;
    unsigned long long* err = sg.err.template as<unsigned long long>();
    // the constraint holding term t: the last i with tp[i] <= t
    auto constraint_of = [&](uint64_t t) {
      return (uint32_t)(std::upper_bound(z.tp.begin(), z.tp.end(), t) - z.tp.begin() - 1);
    };
    auto term_off = [&](uint64_t t) { const uint32_t i = constraint_of(t); return r1cs_term_off(z, i, t - z.tp[i]); };
    for (uint64_t a = 0; a < T;) {
      // terms [a, b): SER_CHUNK of them unless their bytes (counts between them included) outgrow the staging buffers,
      // which only runs of empty combinations can make them do
      uint64_t b = std::min<uint64_t>(T, a + SER_CHUNK);
      const uint64_t base = term_off(a);
      while (b - a > 1 && term_off(b - 1) + z.ts - base > stage) b = a + (b - a) / 2;
      const uint64_t span = term_off(b - 1) + z.ts - base;
      if ((rc = ser_chunk_upload(sg, bytes + z.sec2_off + base, (size_t)span, nullptr))) return rc;
      const uint8_t* chunk = sg.dev[sg.chunks & 1].template as<uint8_t>();
      G16_CUDA(r1cs_term_enqueue<Fr>(sg.st_dec, chunk, base, z.sec2_off, a, (uint32_t)(b - a), constraint_of(a), constraint_of(b - 1),
                                     d_tp.template as<uint64_t>(), z.ts, z.nwires, csr, err));
      if ((rc = ser_chunk_done(sg))) return rc;
      a = b;
    }
    G16_CUDA(cudaStreamSynchronize(sg.st_dec));
    unsigned long long first_err = 0;
    G16_CUDA(cudaMemcpy(&first_err, sg.err.p, 8, cudaMemcpyDeviceToHost));
    if (first_err != ~0ull) return fail(G16_ERR_INVALID_DATA, r1cs_reason(bytes, z, first_err >> 8, (uint32_t)(first_err & 0xff)));
    d_tp.release();
    for (DevBuf& x : sg.dev) x.release();
    // the host copies g16_setup and g16_setup_from_srs read: one download of the decoded CSR
    uint64_t d2h = 8;
    for (int m = 0; m < 3; m++) {
      const uint32_t nnz = z.rp[m][nc];
      h_col[m].resize(nnz);
      h_val[m].resize(nnz);
      if (nnz) {
        G16_CUDA(cudaMemcpy(h_col[m].data(), csr_col[m].p, (size_t)nnz * 4, cudaMemcpyDeviceToHost));
        G16_CUDA(cudaMemcpy(h_val[m].data(), csr_val[m].p, (size_t)nnz * sizeof(Fr), cudaMemcpyDeviceToHost));
      }
      d2h += (uint64_t)nnz * (4 + sizeof(Fr));
      h_rp[m] = std::move(z.rp[m]);
    }
    num_inputs = z.num_inputs; num_constraints = nc; num_witness = z.num_witness; L = Ln; qap = qp;
    G16_CUDA(S0.d_z.reserve((size_t)nvars() * sizeof(Fr)));
    if ((rc = ensure_circuit_domain())) return rc;
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    have_circuit = true;
    const auto t2 = std::chrono::steady_clock::now();
    auto ms = [](auto x, auto y) { return std::chrono::duration<float, std::milli>(y - x).count(); };
    tm.total_ms = ms(t0, t2);
    tm.h2d_ms = ms(t0, t1);
    tm.witness_map_ms = ms(t1, t2);
    tm.h2d_bytes = sg.h2d_bytes + (uint64_t)(nc + 1) * (3 * 4 + 8);
    tm.d2h_bytes = d2h;
    tm.launches = sg.launches + (ntt_launches + ctr.launches - launches0);
    if (info)
      *info = g16_r1cs_info{num_inputs, num_constraints, num_witness, (uint32_t)L, h_rp[0][nc], h_rp[1][nc], h_rp[2][nc]};
    return G16_OK;
  }
  int wtns_read(const uint8_t* bytes, uint64_t len, uint64_t* out, uint64_t cap, uint64_t* count) override {
    if (!bytes || !count) return fail(G16_ERR_BAD_ARGUMENT, "null bytes / count_out");
    WtnsLayout w;
    const std::string why = wtns_walk<typename CP::FrP>(bytes, len, w);
    if (!why.empty()) return fail(G16_ERR_INVALID_DATA, why);
    *count = w.n;
    if (!out) return G16_OK;
    if (cap < w.n)
      return fail(G16_ERR_BAD_ARGUMENT, "output buffer holds " + std::to_string(cap) + " elements, the witness has " + std::to_string(w.n));
    if (!w.n) return G16_OK;
    G16_CUDA(cudaSetDevice(device));
    DevBuf d_out;
    G16_CUDA(d_out.reserve((size_t)w.n * sizeof(Fr)));
    SerStaging sg;
    int rc = ser_staging_init(sg, (size_t)SER_CHUNK * w.n8, 8);
    if (rc) return rc;
    unsigned long long* err = sg.err.template as<unsigned long long>();
    for (uint64_t e = 0; e < w.n; e += SER_CHUNK) {
      const uint32_t cnt = (uint32_t)std::min<uint64_t>(SER_CHUNK, w.n - e);
      const uint64_t off = w.off + e * w.n8;
      if ((rc = ser_chunk_upload(sg, bytes + off, (size_t)cnt * w.n8, nullptr))) return rc;
      G16_CUDA(wtns_elem_enqueue<Fr>(sg.st_dec, sg.dev[sg.chunks & 1].template as<uint8_t>(), off, e, cnt, d_out.p, err));
      if ((rc = ser_chunk_done(sg))) return rc;
    }
    G16_CUDA(cudaStreamSynchronize(sg.st_dec));
    unsigned long long first_err = 0;
    G16_CUDA(cudaMemcpy(&first_err, sg.err.p, 8, cudaMemcpyDeviceToHost));
    if (first_err != ~0ull) return fail(G16_ERR_INVALID_DATA, wtns_reason(w, first_err >> 8, (uint32_t)(first_err & 0xff)));
    G16_CUDA(cudaMemcpy(out, d_out.p, (size_t)w.n * sizeof(Fr), cudaMemcpyDeviceToHost));
    return G16_OK;
  }
  // g16_ptau_read (ptau.cuh): host copies only.  Every request is decided before anything is copied.
  int ptau_read(const uint8_t* bytes, uint64_t len, const g16_srs_out* so, g16_lagrange_out* lo, g16_ptau_info* info) override {
    if (!bytes || !info) return fail(G16_ERR_BAD_ARGUMENT, "null bytes / info");
    PtauLayout z;
    const std::string why = ptau_walk<CP>(bytes, len, z);
    if (!why.empty()) return fail(G16_ERR_INVALID_DATA, why);
    *info = g16_ptau_info{z.n8, z.power, z.ceremony_power, (uint32_t)z.prepared};
    if (so) {
      const uint64_t* dst[PTAU_MEMBERS] = {so->tau_g1, so->tau_g2, so->alpha_tau_g1, so->beta_tau_g1};
      const uint64_t want[PTAU_MEMBERS] = {so->tau_g1_len, so->tau_g2_len, so->alpha_tau_g1_len, so->beta_tau_g1_len};
      for (int m = 0; m < PTAU_MEMBERS; m++) {
        if (want[m] > z.len[m])
          return fail(G16_ERR_BAD_ARGUMENT, std::string("srs_out.") + srs_member(m) + ": " + std::to_string(want[m]) +
                                                " points asked, the file holds " + std::to_string(z.len[m]));
        if (want[m] && !dst[m]) return fail(G16_ERR_BAD_ARGUMENT, std::string("null srs_out member ") + srs_member(m));
      }
      if (!so->beta_g2) return fail(G16_ERR_BAD_ARGUMENT, "null srs_out member beta_g2");
    }
    if (lo) {
      if (!z.prepared)
        return fail(G16_ERR_BAD_ARGUMENT, z.power + 1 > (uint32_t)CP::FrP::TWO_ADICITY
                                              ? "lag_out: the file's Lagrange sections are not read at power " + std::to_string(z.power)
                                              : std::string("lag_out: the file is not prepared (no sections 12-15)"));
      if (lo->log_n > z.power)
        return fail(G16_ERR_BAD_ARGUMENT, "lag_out.log_n = " + std::to_string(lo->log_n) + " is above the file's power " +
                                              std::to_string(z.power));
    }
    if (so) {
      uint64_t* dst[PTAU_MEMBERS] = {so->tau_g1, so->tau_g2, so->alpha_tau_g1, so->beta_tau_g1};
      const uint64_t want[PTAU_MEMBERS] = {so->tau_g1_len, so->tau_g2_len, so->alpha_tau_g1_len, so->beta_tau_g1_len};
      for (int m = 0; m < PTAU_MEMBERS; m++)
        if (want[m]) memcpy(dst[m], bytes + z.off[m], want[m] * z.bytes(m));
      memcpy(so->beta_g2, bytes + z.beta_g2_off, z.g2_bytes);
    }
    if (lo) {
      const uint64_t k = lo->log_n, cnt = 1ull << k;
      lo->h_over_2n = k < z.power;   // level k + 1 is interior: taken over all 2^(k+1) powers, none of them the identity
      uint64_t* dst[PTAU_MEMBERS] = {lo->tau_g1, lo->tau_g2, lo->alpha_tau_g1, lo->beta_tau_g1};
      for (int m = 0; m < PTAU_MEMBERS; m++)
        if (dst[m]) memcpy(dst[m], bytes + z.lag_off[m] + ptau_level_start(k) * z.bytes(m), cnt * z.bytes(m));
      if (lo->tau_g1_h) {   // entries 2i + 1 of level k + 1 of section 12
        const uint8_t* src = bytes + z.lag_off[PTAU_TAU_G1] + (ptau_level_start(k + 1) + 1) * z.g1_bytes;
        uint8_t* d = reinterpret_cast<uint8_t*>(lo->tau_g1_h);
        for (uint64_t i = 0; i < cnt; i++) memcpy(d + i * z.g1_bytes, src + 2 * i * z.g1_bytes, z.g1_bytes);
      }
    }
    return G16_OK;
  }
  // g16_ptau_prepare (ptau.cuh): every Lagrange level of sections 2..5 by srs_ifft, member by member, one level at a time.
  // Refusals before any point is read write nothing; then a check pass over every point of sections 2..5 (srs_check, the
  // first bad one by member and index), and only after it the output: header and kept sections copied on the host, each
  // level transformed on the device (1/2^k folded into the load, affine store fused into the last stage) and copied to
  // its place.  Level 0 is X_0 itself.  Device memory: one member at a time, its points, one XYZZ buffer and one affine
  // staging buffer for its top level.  Timings as g16_srs_contribute's: h2d_ms = the check pass, msm_ms[m] = member m.
  int ptau_prepare(const uint8_t* in, uint64_t in_len, uint32_t flags, uint8_t* out, uint64_t cap, uint64_t* len_out) override {
    if (!in || !len_out) return fail(G16_ERR_BAD_ARGUMENT, "null in / len_out");
    if (flags & ~(uint32_t)G16_SER_VALIDATE) return fail(G16_ERR_BAD_ARGUMENT, "g16_ptau_prepare takes 0 or G16_SER_VALIDATE");
    G16_NOT_BUSY();
    PtauLayout z;
    BinSection sec[16];
    std::string why = ptau_walk_header<CP>(in, in_len, z, sec);
    if (!why.empty()) return fail(G16_ERR_INVALID_DATA, why);
    const uint32_t two_adicity = (uint32_t)CP::FrP::TWO_ADICITY;
    if (z.power + 1 > two_adicity)
      return fail(G16_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "power " + std::to_string(z.power) + ": level power + 1 = " +
                                                           std::to_string(z.power + 1) + " is above the scalar field's two-adicity " +
                                                           std::to_string(two_adicity));
    if (!(why = ptau_walk<CP>(in, in_len, z)).empty()) return fail(G16_ERR_INVALID_DATA, why);
    const auto kept = ptau_kept_sections(in);
    uint64_t kept_bytes = 0;
    for (const auto& k : kept) kept_bytes += k.second;
    const PtauPrepared pl = ptau_prepared_layout((uint32_t)kept.size(), kept_bytes, z.power, z.g1_bytes, z.g2_bytes);
    *len_out = pl.size;
    if (!out) return G16_OK;
    if (cap < pl.size)
      return fail(G16_ERR_BAD_ARGUMENT, "output buffer holds " + std::to_string(cap) + " bytes, the prepared file needs " +
                                            std::to_string(pl.size));
    if (srs_overlap((uintptr_t)in, in_len, (uintptr_t)out, pl.size)) return fail(G16_ERR_BAD_ARGUMENT, "out overlaps in");
    G16_CUDA(cudaSetDevice(device));
    const auto t0 = std::chrono::steady_clock::now();
    auto ms_since = [](std::chrono::steady_clock::time_point a) {
      return (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count();
    };
    tm = g16_timings{};
    cudaStream_t st = S0.st_main;
    const uint64_t esz[PTAU_MEMBERS] = {sizeof(A1), sizeof(A2), sizeof(A1), sizeof(A1)};
    const uint64_t psz[PTAU_MEMBERS] = {sizeof(P1), sizeof(P2), sizeof(P1), sizeof(P1)};
    // --- memory: member m needs its points, ptau_work_points(top) XYZZ and as many affine points on the device at once ---
    size_t free_b = 0, total_b = 0;
    G16_CUDA(cudaMemGetInfo(&free_b, &total_b));
    for (int m = 0; m < PTAU_MEMBERS; m++) {
      const uint32_t top = ptau_top_level(m, z.power);
      const double need = (double)z.len[m] * esz[m] + (double)(psz[m] + esz[m]) * (double)ptau_work_points(top);
      if (need > (double)free_b)
        return fail(G16_ERR_CUDA, std::string(srs_member(m)) + " level 2^" + std::to_string(top) + " needs " +
                                      std::to_string((uint64_t)need) + " bytes of device memory, " + std::to_string(free_b) +
                                      " are free");
    }
    // --- check pass: every point of sections 2..5 ---
    DevBuf din, work, stage, err, dtab;
    G16_CUDA(err.reserve(8));
    for (int m = 0; m < PTAU_MEMBERS; m++) {
      const uint64_t bytes = z.len[m] * esz[m];
      G16_CUDA(din.reserve(bytes));
      G16_CUDA(cudaMemcpyAsync(din.p, in + z.off[m], bytes, cudaMemcpyHostToDevice, st));
      G16_CUDA(cudaMemsetAsync(err.p, 0xff, 8, st));
      unsigned long long* e = err.template as<unsigned long long>();
      const uint32_t cnt = (uint32_t)z.len[m];
      G16_CUDA((m == PTAU_TAU_G2 ? srs_check<CP, true>(st, din.p, cnt, flags, m, e) : srs_check<CP, false>(st, din.p, cnt, flags, m, e)));
      unsigned long long first_err = 0;
      G16_CUDA(cudaMemcpyAsync(&first_err, err.p, 8, cudaMemcpyDeviceToHost, st));
      G16_CUDA(cudaStreamSynchronize(st));
      tm.h2d_bytes += bytes;
      tm.d2h_bytes += 8;
      tm.launches++;
      if (first_err != ~0ull)
        return fail(G16_ERR_INVALID_DATA, std::string(srs_member(m)) + "[" + std::to_string((first_err >> 8) & ((1ull << 40) - 1)) +
                                              "]: " + ser_reason(first_err & 0xff));
    }
    tm.h2d_ms = ms_since(t0);
    // --- output: header, kept sections, heads of 12..15 and every level 0 on the host ---
    auto put32 = [&](uint64_t at, uint32_t v) { memcpy(out + at, &v, 4); };
    auto put64 = [&](uint64_t at, uint64_t v) { memcpy(out + at, &v, 8); };
    memcpy(out, "ptau", 4);
    put32(4, 1);
    put32(8, pl.nsec);
    uint64_t pos = 12;
    for (const auto& k : kept) { memcpy(out + pos, in + k.first, k.second); pos += k.second; }
    for (int m = 0; m < PTAU_MEMBERS; m++) {
      put32(pl.lag_off[m] - 12, 12 + m);
      put64(pl.lag_off[m] - 8, pl.lag_pts[m] * esz[m]);
      memcpy(out + pl.lag_off[m], in + z.off[m], esz[m]);
    }
    // --- transforms: level k of member m = srs_ifft of size 2^k over its first points, scaled by 1/2^k ---
    const uint32_t tab_log = z.power + 1;
    Fr tab[128];   // omega_N^-(2^b) (N = 2^tab_log) at b < 64, (1/2)^k at 64 + k
    tab[0] = Fr::inv(fr_domain_root<Fr>((int)tab_log));
    tab[64] = Fr::one();
    const Fr half = Fr::inv(fr_from_u64<Fr>(2));
    for (int b = 1; b < 64; b++) { tab[b] = Fr::sqr(tab[b - 1]); tab[64 + b] = Fr::mul(tab[63 + b], half); }
    G16_CUDA(dtab.reserve(sizeof(tab)));
    G16_CUDA(cudaMemcpyAsync(dtab.p, tab, sizeof(tab), cudaMemcpyHostToDevice, st));
    tm.h2d_bytes += sizeof(tab);
    const Fr* dt = dtab.template as<Fr>();
    unsigned long long launches = 0;
    // Levels 1 .. PTAU_SMALL_LEVELS of a member each run on a stream of their own, into their own slice of work and stage
    // (level k at point 2^k - 1, as in the section): they are latency-bound, one thread's scalar multiplication per stage,
    // and together they hold fewer butterflies than one wave.  The larger levels follow one by one on the main stream.
    struct SideStreams {
      cudaStream_t s[PTAU_SMALL_LEVELS] = {};
      cudaEvent_t ev = nullptr;
      ~SideStreams() {
        for (cudaStream_t x : s) if (x) cudaStreamDestroy(x);
        if (ev) cudaEventDestroy(ev);
      }
    } side;
    for (cudaStream_t& x : side.s) G16_CUDA(cudaStreamCreateWithFlags(&x, cudaStreamNonBlocking));
    G16_CUDA(cudaEventCreateWithFlags(&side.ev, cudaEventDisableTiming));
    for (int m = 0; m < PTAU_MEMBERS; m++) {
      const auto t1 = std::chrono::steady_clock::now();
      const uint32_t top = ptau_top_level(m, z.power), small = std::min(top, PTAU_SMALL_LEVELS);
      const uint64_t bytes = z.len[m] * esz[m], pts = ptau_work_points(top);
      for (DevBuf* b : {&din, &work, &stage}) b->release();   // the peak is one member's
      G16_CUDA(din.reserve(bytes));
      G16_CUDA(work.reserve(psz[m] * pts));
      G16_CUDA(stage.reserve(esz[m] * pts));
      G16_CUDA(cudaMemcpyAsync(din.p, in + z.off[m], bytes, cudaMemcpyHostToDevice, st));
      tm.h2d_bytes += bytes;
      // level k on stream s, into the slices at point `at` of work and stage
      auto level = [&](cudaStream_t s, uint32_t k, uint64_t at) -> cudaError_t {
        if (m == PTAU_TAU_G2)
          return srs_ifft<Fq2, Fr>(s, din.template as<A2>(), z.len[m], 0, (int)k, dt + 64 + k, 0, dt, (int)tab_log,
                                   work.template as<P2>() + at, stage.template as<A2>() + at, &launches);
        return srs_ifft<Fq, Fr>(s, din.template as<A1>(), z.len[m], 0, (int)k, dt + 64 + k, 0, dt, (int)tab_log,
                                work.template as<P1>() + at, stage.template as<A1>() + at, &launches);
      };
      if (small) {
        G16_CUDA(cudaEventRecord(side.ev, st));   // the member's points are on the device
        for (uint32_t k = 1; k <= small; k++) {
          G16_CUDA(cudaStreamWaitEvent(side.s[k - 1], side.ev, 0));
          G16_CUDA(level(side.s[k - 1], k, ptau_level_start(k)));
        }
        for (uint32_t k = 1; k <= small; k++) G16_CUDA(cudaStreamSynchronize(side.s[k - 1]));
        const uint64_t cnt = ptau_level_start(small + 1) - 1;   // levels 1 .. small, contiguous as in the section
        G16_CUDA(cudaMemcpyAsync(out + pl.lag_off[m] + esz[m], stage.template as<uint8_t>() + esz[m], cnt * esz[m],
                                 cudaMemcpyDeviceToHost, st));
        tm.d2h_bytes += cnt * esz[m];
      }
      for (uint32_t k = small + 1; k <= top; k++) {
        G16_CUDA(level(st, k, 0));
        const uint64_t cnt = 1ull << k;
        G16_CUDA(cudaMemcpyAsync(out + pl.lag_off[m] + ptau_level_start(k) * esz[m], stage.p, cnt * esz[m],
                                 cudaMemcpyDeviceToHost, st));
        tm.d2h_bytes += cnt * esz[m];
      }
      G16_CUDA(cudaStreamSynchronize(st));
      tm.msm_ms[m] = ms_since(t1);
    }
    tm.launches += launches;
    tm.total_ms = ms_since(t0);
    return G16_OK;
  }
  int pk_export_serialized(uint32_t flags, uint8_t* out, uint64_t cap, uint64_t* len_out) override {
    using Fmt = SerFormat<CP>;
    if (!have_pk || !from_setup) return fail(G16_ERR_BAD_ARGUMENT, "g16_pk_export_serialized needs a key produced by g16_setup");
    if (!len_out) return fail(G16_ERR_BAD_ARGUMENT, "null len_out");
    if (flags & ~(uint32_t)G16_SER_COMPRESSED) return fail(G16_ERR_BAD_ARGUMENT, "export takes G16_SER_COMPRESSED only");
    G16_NOT_BUSY();
    const uint64_t nv = nvars();
    SerItem it[SER_ITEMS];
    ser_items(it);
    it[SER_GAMMA_ABC].len = num_inputs;
    it[SER_A].len = it[SER_B_G1].len = it[SER_B_G2].len = nv;
    it[SER_H].len = h_query_len();
    it[SER_L].len = num_witness;
    const uint64_t size = ser_size(it, Fmt::NB, flags & G16_SER_COMPRESSED, Fmt::G2_NC);
    *len_out = size;
    if (!out) return G16_OK;
    if (cap < size)
      return fail(G16_ERR_BAD_ARGUMENT, "output buffer holds " + std::to_string(cap) + " bytes, the key needs " + std::to_string(size));
    G16_CUDA(cudaSetDevice(device));
    const A1 g1s[SER_ITEMS] = {alpha_g1, {}, {}, {}, {}, beta_g1, delta_g1};
    const A2 g2s[SER_ITEMS] = {{}, beta_g2, gamma_g2, delta_g2};
    const void* src[SER_ITEMS] = {};
    src[SER_GAMMA_ABC] = d_gamma_abc.p; src[SER_A] = full_a.p; src[SER_B_G1] = full_b1.p; src[SER_B_G2] = full_b2.p;
    src[SER_H] = q[M_H].bases.p; src[SER_L] = q[M_L].bases.p;
    DevBuf stage;
    G16_CUDA(stage.reserve((size_t)SER_CHUNK * 4 * Fmt::NB));
    for (int m = 0; m < SER_ITEMS; m++) {
      const SerItem& x = it[m];
      if (!x.vec) {   // a single point: encoded here, with the kernel's own function
        if (x.g2) ser_encode<CP, true>(g2s[m], flags, out + x.off);
        else ser_encode<CP, false>(g1s[m], flags, out + x.off);
        continue;
      }
      for (int k = 0; k < 8; k++) out[x.off - 8 + k] = (uint8_t)(x.len >> (8 * k));
      const size_t esz = x.g2 ? sizeof(A2) : sizeof(A1);
      for (uint64_t f = 0; f < x.len; f += SER_CHUNK) {
        const uint32_t cnt = (uint32_t)std::min<uint64_t>(SER_CHUNK, x.len - f);
        const void* s = (const char*)src[m] + f * esz;
        G16_CUDA((x.g2 ? ser_encode_enqueue<CP, true>(S0.st_main, s, cnt, flags, stage.template as<uint8_t>())
                       : ser_encode_enqueue<CP, false>(S0.st_main, s, cnt, flags, stage.template as<uint8_t>())));
        G16_CUDA(cudaMemcpyAsync(out + x.off + f * x.psize, stage.p, (size_t)cnt * x.psize, cudaMemcpyDeviceToHost, S0.st_main));
        G16_CUDA(cudaStreamSynchronize(S0.st_main));
      }
    }
    return G16_OK;
  }

  // ---- proving ----
  // enqueue on sl.st_main: upload z, row evaluation, witness map
  // count > 1 (batch proving): `count` assignments, nv elements apart, and as many witness maps
  int enqueue_witness_map(Slot& sl, const uint64_t* z, uint32_t flags, uint32_t count = 1) {
    const uint64_t nv = nvars();
    int rc = ensure_circuit_domain();   // no-op unless something rebuilt `dom` for another size
    if (rc) return rc;
    if ((rc = ensure_slot_buffers(sl, L, count))) return rc;
    G16_CUDA(sl.d_z.reserve((size_t)nv * sizeof(Fr) * count));
    sl.tm.h2d_bytes = 0;
    G16_CUDA(cudaEventRecord(sl.ev_start, sl.st_main));
    if (flags & G16_ASSIGNMENT_ON_DEVICE) {
      G16_CUDA(cudaMemcpyAsync(sl.d_z.p, z, nv * sizeof(Fr) * count, cudaMemcpyDeviceToDevice, sl.st_main));
    } else {
      G16_CUDA(cudaMemcpyAsync(sl.d_z.p, z, nv * sizeof(Fr) * count, cudaMemcpyHostToDevice, sl.st_main));
      sl.tm.h2d_bytes = nv * sizeof(Fr) * count;
    }
    G16_CUDA(cudaEventRecord(sl.ev_z, sl.st_main));
    const uint32_t n = 1u << L;
    CsrDev cs[3];
    csr_dev(cs);
    sl.check = (flags & G16_CHECK_WITNESS) != 0;
    if (sl.check) {   // on the main stream only: the MSMs, which wait for ev_z, run beside it
      const size_t bytes = (size_t)count * 3 * sizeof(uint32_t);
      G16_CUDA(sl.d_check.reserve(bytes));
      if (sl.h_check_cap < bytes) {
        if (sl.h_check) cudaFreeHost(sl.h_check);
        sl.h_check = nullptr;
        sl.h_check_cap = 0;
        G16_CUDA(cudaMallocHost(&sl.h_check, bytes));
        sl.h_check_cap = bytes;
      }
      G16_CUDA(r1cs_check<Fr>(sl.st_main, cs, sl.d_z.template as<Fr>(), num_constraints, (uint32_t)nv, count,
                              sl.d_check.template as<uint32_t>(), &ntt_launches));
    }
    r1cs_matvec<Fr>(sl.st_main, cs, sl.d_z.template as<Fr>(), num_constraints, num_inputs, n, sl.d_a.template as<Fr>(),
                    sl.d_b.template as<Fr>(), sl.d_c.template as<Fr>(), count, (uint32_t)nv, qap == G16_QAP_LIBSNARK);
    ntt_launches++;
    if (sl.split_wm && nccl_comm_wm) {
      if ((rc = witness_map_split(sl))) return rc;
    } else if (qap == G16_QAP_CIRCOM) {
      witness_map_device_circom(sl, dom, count);
    } else {
      witness_map_device(sl, dom, count);
    }
    G16_CUDA(cudaGetLastError());
    G16_CUDA(cudaEventRecord(sl.ev_h, sl.st_main));
    if (sl.check)   // after ev_h: the H MSM does not wait for the copy
      G16_CUDA(cudaMemcpyAsync(sl.h_check, sl.d_check.p, (size_t)count * 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, sl.st_main));
    return G16_OK;
  }
  void csr_dev(CsrDev cs[3]) const {
    for (int m = 0; m < 3; m++) cs[m] = CsrDev{csr_rp[m].template as<uint32_t>(), csr_col[m].template as<uint32_t>(), csr_val[m].p};
  }
  // One r1cs_check record (lowest unsatisfied row, ~count, lowest malformed element) as the ABI reports it: a malformed
  // element leaves the rows unevaluated
  static g16_witness_report report_of(const uint32_t* x) {
    g16_witness_report w;
    w.first_malformed = x[2] == UINT32_MAX ? G16_NONE : x[2];
    const bool rows = w.first_malformed == G16_NONE;
    w.first_unsatisfied = rows && x[0] != UINT32_MAX ? x[0] : G16_NONE;
    w.num_unsatisfied = rows ? (uint32_t)~x[1] : 0;
    return w;
  }
  static bool report_ok(const g16_witness_report& w) { return w.first_malformed == G16_NONE && w.num_unsatisfied == 0; }
  static std::string report_reason(const g16_witness_report& w) {
    if (w.first_malformed == 0) return "assignment element 0 is not One";
    if (w.first_malformed != G16_NONE)
      return "assignment element " + std::to_string(w.first_malformed) + " is not a canonical Fr";
    return "constraint " + std::to_string(w.first_unsatisfied) + " unsatisfied (" + std::to_string(w.num_unsatisfied) + " in all)";
  }
  // The verdict of a single-proof submission, once its main stream has drained: G16_OK, or G16_ERR_UNSATISFIED naming why
  int slot_verdict(const Slot& sl) const {
    if (!sl.check) return G16_OK;
    const g16_witness_report w = report_of(sl.h_check);
    return report_ok(w) ? G16_OK : fail(G16_ERR_UNSATISFIED, report_reason(w));
  }
  // g16_check_witness: slot 0's main stream, one launch per chunk of at most R1CS_CHECK_MAX_Y assignments; host assignments
  // go up chunk by chunk, each chunk at most half the free device memory
  int check_witness(uint32_t count, const uint64_t* z, uint32_t flags, g16_witness_report* out) override {
    if (count == 0) return G16_OK;
    if (flags & ~(uint32_t)G16_ASSIGNMENT_ON_DEVICE) return fail(G16_ERR_BAD_ARGUMENT, "g16_check_witness takes G16_ASSIGNMENT_ON_DEVICE only");
    if (!z || !out) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    if (!have_circuit) return fail(G16_ERR_BAD_ARGUMENT, "no circuit resident");
    if (S0.busy) return fail(G16_ERR_BAD_ARGUMENT, "slot 0 has a proof in flight");
    G16_CUDA(cudaSetDevice(device));
    const bool on_device = (flags & G16_ASSIGNMENT_ON_DEVICE) != 0;
    const uint64_t nv = nvars();
    const size_t zb = (size_t)nv * sizeof(Fr);
    uint64_t chunk = std::min<uint64_t>(count, R1CS_CHECK_MAX_Y);
    DevBuf dz, dres;
    if (!on_device) {
      size_t free_b = 0, total_b = 0;
      G16_CUDA(cudaMemGetInfo(&free_b, &total_b));
      chunk = std::max<uint64_t>(1, std::min<uint64_t>(chunk, free_b / 2 / zb));
      G16_CUDA(dz.reserve(chunk * zb));
    }
    G16_CUDA(dres.reserve(chunk * 3 * sizeof(uint32_t)));
    std::vector<uint32_t> res(chunk * 3);
    CsrDev cs[3];
    csr_dev(cs);
    cudaStream_t st = S0.st_main;
    for (uint64_t first = 0; first < count; first += chunk) {
      const uint32_t k = (uint32_t)std::min<uint64_t>(chunk, count - first);
      const uint64_t* src = z + first * nv * FR64;
      if (!on_device) G16_CUDA(cudaMemcpyAsync(dz.p, src, k * zb, cudaMemcpyHostToDevice, st));
      const Fr* zk = on_device ? reinterpret_cast<const Fr*>(src) : dz.template as<Fr>();
      G16_CUDA(r1cs_check<Fr>(st, cs, zk, num_constraints, (uint32_t)nv, k, dres.template as<uint32_t>(), &ntt_launches));
      G16_CUDA(cudaMemcpyAsync(res.data(), dres.p, (size_t)k * 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
      G16_CUDA(cudaStreamSynchronize(st));
      for (uint32_t i = 0; i < k; i++) out[first + i] = report_of(&res[3 * (size_t)i]);
    }
    return G16_OK;
  }
  int witness_map(const uint64_t* z, uint32_t flags, uint64_t* h) override {
    if (!have_circuit) return fail(G16_ERR_BAD_ARGUMENT, "no circuit resident");
    if (!z || !h) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    if (S0.busy) return fail(G16_ERR_BAD_ARGUMENT, "slot 0 has a proof in flight");
    G16_CUDA(cudaSetDevice(device));
    int rc = enqueue_witness_map(S0, z, flags);
    if (rc) return rc;
    if (S0.check) {   // a rejected assignment writes nothing to h
      G16_CUDA(cudaStreamSynchronize(S0.st_main));
      if ((rc = slot_verdict(S0))) return rc;
    }
    G16_CUDA(cudaMemcpyAsync(h, S0.d_h.p, sizeof(Fr) << L, cudaMemcpyDeviceToHost, S0.st_main));
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    return G16_OK;
  }

  // The five MSMs of the slot's proof or group on its streams, with the geometry sl.geom[] and the flags sl.run[] the
  // caller set.  Proof k of a batched geometry reads its scalars k times one proof's vector length further on.
  int enqueue_msms(Slot& sl) {
    const uint64_t nv = nvars(), n = 1ull << L;
    const uint32_t* zs = sl.d_z.template as<uint32_t>();
    const uint32_t* hs = sl.d_h.template as<uint32_t>();
    // scalar sources (prover.rs:63-85): H <- h ; L <- aux ; A, B1, B2 <- input[1..] ++ aux
    constexpr int W = Fr::N;   // 32-bit words per scalar
    const uint32_t* src[5] = {hs, zs + (size_t)num_inputs * W, zs + W, zs + W, zs + W};
    const uint64_t stride[5] = {n * W, nv * W, nv * W, nv * W, nv * W};   // 32-bit words between two proofs' scalars
    // B in G1 and B in G2 run over the same scalars and identity pattern: one counting sort serves both.  B2 sorts
    // (its stream has the higher priority and its tail is the longest), B1 borrows the list.
    const bool share = share_b_sort && sl.run[M_B1] && sl.run[M_B2];
    // "witness map first" (option, off by default): the MSMs that do not need h sort their entries at once but start
    // accumulating only when the witness map is done, so that their register-heavy blocks do not slow the NTT kernels.
    const bool wm_first = !sl.serial && (tune.wm_first > 0 || (tune.wm_first < 0 && world > 1));
    for (int m : {M_L, M_A, M_B2, M_B1, M_H}) {   // H last: it waits for the witness map; B1 borrows B2's sorted list
      NvtxSpan span_msm(span_of(m));
      cudaStream_t st = sl.serial ? sl.st_main : sl.st_msm[m];
      if (!sl.serial) G16_CUDA(cudaStreamWaitEvent(st, m == M_H ? sl.ev_h : sl.ev_z, 0));
      G16_CUDA(cudaEventRecord(sl.ev_m0[m], st));
      if (sl.run[m]) {
        const uint32_t* sc = src[m] + q[m].lo * W;   // first owned scalar; the digit kernel strides by `world`
        cudaEvent_t gate = (wm_first && m != M_H) ? sl.ev_h : nullptr;
        cudaError_t e;
        if (m == M_B2 && share) { sl.b_sorted = MsmSorted{}; sl.b_sorted.ready = sl.ev_bsort; }
        if (m == M_B2) e = msm_enqueue<Fq2, Fr>(st, sl.ws2, sl.geom[m], q[m].bases.template as<A2>(), q[m].mask.template as<uint8_t>(), sc, world, true, &ctr, sl.ev_a0[m], sl.ev_a1[m], share ? &sl.b_sorted : nullptr, nullptr, gate, stride[m]);
        else e = msm_enqueue<Fq, Fr>(st, sl.ws1[m], sl.geom[m], q[m].bases.template as<A1>(), q[m].mask.template as<uint8_t>(), sc, world, true, &ctr, sl.ev_a0[m], sl.ev_a1[m], nullptr, (m == M_B1 && share) ? &sl.b_sorted : nullptr, gate, stride[m]);
        if (e != cudaSuccess) return fail(G16_ERR_CUDA, std::string("msm_enqueue: ") + cudaGetErrorString(e));
      }
      G16_CUDA(cudaEventRecord(sl.ev_m1[m], st));
    }
    return G16_OK;
  }
  // Asynchronous half of a proof: everything is enqueued on the slot's streams, nothing is waited for.
  // s may be null (partial proof: the key products are skipped).
  int submit(Slot& sl, const uint64_t* r, const uint64_t* s, const uint64_t* z, uint32_t flags) {
    if (!have_circuit || !have_pk) return fail(G16_ERR_BAD_ARGUMENT, "circuit and proving key must be resident");
    if (!r || !z) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    if (sl.busy) return fail(G16_ERR_BAD_ARGUMENT, "slot already has a proof in flight (g16_prove_wait first)");
    G16_CUDA(cudaSetDevice(device));
    NvtxSpan span_prover(SPAN_PROVER);
    sl.launches0 = ctr.launches + ntt_launches;
    sl.serial = (flags & G16_SERIAL_MSMS) != 0;
    sl.r = load_fr(r);
    sl.have_s = s != nullptr;
    if (s) sl.s = load_fr(s);
    if (sl.have_s) {
      if (sl.helper) sl.helper->wait();
      if (sl.helper2) sl.helper2->wait();
      sl.helper = pool->submit([this, &sl]() { key_products_a(sl.r, sl.s, sl.kp); });
      sl.helper2 = pool->submit([this, &sl]() { key_products_b(sl.r, sl.s, sl.kp); });
    }
    int rc;
    {
      NvtxSpan span_wm(SPAN_WITNESS_MAP);
      rc = enqueue_witness_map(sl, z, flags);
    }
    if (rc) return rc;
    for (int m = 0; m < 5; m++) {
      const uint64_t cnt = q[m].hi - q[m].lo;
      sl.geom[m] = q[m].geom;
      sl.run[m] = cnt > 0 && !(m == M_B1 && sl.r.is_zero());             // prover.rs:98: B in G1 skipped when r == 0
      sl.tm.msm_pairs[m] = sl.run[m] ? cnt : 0;
    }
    if ((rc = enqueue_msms(sl))) return rc;
    sl.launches0 = ctr.launches + ntt_launches - sl.launches0;   // kernels launched for this proof
    sl.busy = true;
    return G16_OK;
  }
  // Adds the slot's CUDA events and counts to `t`: spans, their timeline measured from `origin`, entries, pairs and bytes.
  // The first group of a call sets the MSMs' begin times, later groups can only lower them.
  void add_timings(const Slot& sl, cudaEvent_t origin, bool first_group, g16_timings& t) const {
    float ms = 0;
    cudaEventElapsedTime(&ms, sl.ev_start, sl.ev_z); t.h2d_ms += ms;
    cudaEventElapsedTime(&ms, sl.ev_z, sl.ev_h); t.witness_map_ms += ms;
    cudaEventElapsedTime(&ms, origin, sl.ev_h);
    t.total_ms = std::max(t.total_ms, ms);
    t.h2d_bytes += sl.tm.h2d_bytes;
    for (int m = 0; m < 5; m++) {
      t.msm_pairs[m] += sl.tm.msm_pairs[m];
      cudaEventElapsedTime(&ms, sl.ev_m0[m], sl.ev_m1[m]); t.msm_ms[m] += ms;
      cudaEventElapsedTime(&ms, origin, sl.ev_m0[m]);
      t.msm_begin_ms[m] = first_group ? ms : std::min(t.msm_begin_ms[m], ms);
      cudaEventElapsedTime(&ms, origin, sl.ev_m1[m]);
      t.msm_end_ms[m] = std::max(t.msm_end_ms[m], ms);
      t.total_ms = std::max(t.total_ms, ms);
      if (!sl.run[m]) continue;
      cudaEventElapsedTime(&ms, sl.ev_a0[m], sl.ev_a1[m]); t.msm_accum_ms[m] += ms;
      t.msm_entries[m] += m == M_B2 ? *sl.ws2.h_total : *sl.ws1[m].h_total;
      t.d2h_bytes += (m == M_B2 ? sl.ws2.plan.leaf_pts * sizeof(P2) : sl.ws1[m].plan.leaf_pts * sizeof(P1)) * sl.geom[m].sets();
    }
  }
  // Synchronous half: wait for the slot's streams, finish every MSM on the host (leaf sums of the bucket reduction,
  // Horner) as soon as its stream drains, one host thread per MSM.
  int wait_partials(Slot& sl, Partials& out) {
    if (!sl.busy) return fail(G16_ERR_BAD_ARGUMENT, "no proof in flight in this slot");
    G16_CUDA(cudaSetDevice(device));
    sl.busy = false;
    auto t0 = std::chrono::steady_clock::now();
    if (sl.serial) G16_CUDA(cudaStreamSynchronize(sl.st_main));
    {
      cudaError_t errs[5] = {cudaSuccess, cudaSuccess, cudaSuccess, cudaSuccess, cudaSuccess};
      P1* outs1[4] = {&out.h, &out.l, &out.a, &out.b1};
      std::shared_ptr<HostPool::Ticket> tk[5];
      for (int m = 0; m < 5; m++) {
        tk[m] = pool->submit([&, m]() {
          cudaSetDevice(device);
          if (!sl.serial) errs[m] = cudaStreamSynchronize(sl.st_msm[m]);
          if (errs[m] != cudaSuccess) return;
          if (m == M_B2) out.b2 = sl.run[m] ? msm_finish<Fq2>(sl.ws2, sl.geom[m]) : P2::inf();
          else *outs1[m] = sl.run[m] ? msm_finish<Fq>(sl.ws1[m], sl.geom[m]) : P1::inf();
          if (sl.have_s && (m == M_A || m == M_B1)) {       // prover.rs:94 / :114, distributed over the MSM result
            uint32_t k[Fr::N];
            fr_to_canon(m == M_A ? sl.s : sl.r, k);
            if (m == M_A) out.sa = out.a.mul_u32(k, Fr::N);
            else out.rb1 = out.b1.mul_u32(k, Fr::N);
          }
        });
      }
      for (auto& t : tk) t->wait();
      out.scaled = sl.have_s;
      for (int m = 0; m < 5; m++)
        if (errs[m] != cudaSuccess) return fail(G16_ERR_CUDA, std::string("msm stream sync: ") + cudaGetErrorString(errs[m]));
      G16_CUDA(cudaStreamSynchronize(sl.st_main));
    }
    g16_timings t{};
    t.host_finish_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    add_timings(sl, sl.ev_start, true, t);
    t.launches = sl.launches0;
    sl.tm = tm = t;
    return G16_OK;
  }
  void store_partials(uint64_t* p, const Partials& x) {
    store_a1(p, x.h.to_affine());
    store_a1(p + 2 * NQ64, x.l.to_affine());
    store_a1(p + 4 * NQ64, x.a.to_affine());
    store_a1(p + 6 * NQ64, x.b1.to_affine());
    store_a2(p + 8 * NQ64, x.b2.to_affine());
  }
  int prove_partial(const uint64_t* r, const uint64_t* z, uint32_t flags, uint64_t* partial) override {
    if (!partial) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    int rc = submit(S0, r, nullptr, z, flags);
    if (rc) return rc;
    Partials x;
    if ((rc = wait_partials(S0, x)) || (rc = slot_verdict(S0))) return rc;
    store_partials(partial, x);
    return G16_OK;
  }
  int partial_submit(int slot, const uint64_t* r, const uint64_t* z, uint32_t flags) override {
    if (slot < 0 || slot >= NSLOTS) return fail(G16_ERR_BAD_ARGUMENT, "bad slot");
    return submit(slots[slot], r, nullptr, z, flags);
  }
  int partial_wait(int slot, uint64_t* partial) override {
    if (slot < 0 || slot >= NSLOTS || !partial) return fail(G16_ERR_BAD_ARGUMENT, "bad slot / null buffer");
    Partials x;
    int rc = wait_partials(slots[slot], x);
    if (rc || (rc = slot_verdict(slots[slot]))) return rc;
    store_partials(partial, x);
    return G16_OK;
  }
  // The five key products of the proof tail (batch.cuh), for the single-proof paths: computed on the host by two pool
  // threads while the GPU works, split into halves of similar cost (a G2 product costs about three G1 products).
  void key_products_a(const Fr& r, const Fr& s, Products& p) const {
    uint32_t rk[Fr::N], sk[Fr::N], rsk[Fr::N];
    fr_to_canon(r, rk);
    fr_to_canon(s, sk);
    fr_to_canon(Fr::mul(r, s), rsk);
    const P1 d1 = P1::from_affine(delta_g1);
    p.r_d1 = d1.mul_u32(rk, Fr::N);
    p.rs_d1 = d1.mul_u32(rsk, Fr::N);
    p.s_pa = P1::from_affine(p_a).mul_u32(sk, Fr::N);
  }
  void key_products_b(const Fr& r, const Fr& s, Products& p) const {
    uint32_t rk[Fr::N], sk[Fr::N];
    fr_to_canon(r, rk);
    fr_to_canon(s, sk);
    p.r_pb = P1::from_affine(p_b).mul_u32(rk, Fr::N);   // the identity when r == 0
    p.s_d2 = P2::from_affine(delta_g2).mul_u32(sk, Fr::N);
  }
  Products key_products(const Fr& r, const Fr& s) const {
    Products p;
    key_products_a(r, s, p);
    key_products_b(r, s, p);
    return p;
  }
  // this rank's contribution to g_c that depends on its MSM results: s A + r B1 + L + H
  P1 c_part(const Fr& r, const Fr& s, const Partials& x) const {
    uint32_t k[Fr::N];
    P1 c = x.scaled ? x.sa : (fr_to_canon(s, k), x.a.mul_u32(k, Fr::N));
    if (!r.is_zero()) c.add(x.scaled ? x.rb1 : (fr_to_canon(r, k), x.b1.mul_u32(k, Fr::N)));
    c.add(x.l);
    c.add(x.h);
    return c;
  }
  // a, b2: the A and B-in-G2 MSM results; c = c_part (each summed over the ranks when the key is sharded)
  void store_proof(uint64_t* proof, const Products& kp, const P1& a, const P2& b2, const P1& c) const {
    NvtxSpan span_finish(SPAN_FINISH_C);
    const ProofPoints<Fq, Fq2> pf = proof_tail(kp, p_a, p_2, a, b2, c);
    store_a1(proof, pf.g_a.to_affine());   // prover.rs:127-131
    store_a2(proof + 2 * NQ64, pf.g2_b.to_affine());
    store_a1(proof + 2 * NQ64 + G2_64, pf.g_c.to_affine());
  }
  int prove_submit(int slot, const uint64_t* r, const uint64_t* s, const uint64_t* z, uint32_t flags) override {
    if (slot < 0 || slot >= NSLOTS) return fail(G16_ERR_BAD_ARGUMENT, "bad slot");
    if (!s) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    if (world != 1) return fail(G16_ERR_BAD_ARGUMENT, "key is sharded: use g16_prove_partial + g16_prove_assemble");
    return submit(slots[slot], r, s, z, flags);
  }
  // the MSM results and key products of a whole proof (not a partial one) in the slot
  int wait_proof(Slot& sl, Partials& x) {
    int rc = wait_partials(sl, x);
    if (sl.helper) { sl.helper->wait(); sl.helper.reset(); }
    if (sl.helper2) { sl.helper2->wait(); sl.helper2.reset(); }
    if (rc) return rc;
    if (!sl.have_s) return fail(G16_ERR_BAD_ARGUMENT, "slot holds a partial proof (use g16_prove_partial_wait)");
    return G16_OK;
  }
  int prove_wait(int slot, uint64_t* proof) override {
    if (slot < 0 || slot >= NSLOTS || !proof) return fail(G16_ERR_BAD_ARGUMENT, "bad slot / null buffer");
    Slot& sl = slots[slot];
    Partials x;
    int rc = wait_proof(sl, x);
    if (rc || (rc = slot_verdict(sl))) return rc;
    auto t0 = std::chrono::steady_clock::now();
    store_proof(proof, sl.kp, x.a, x.b2, c_part(sl.r, sl.s, x));
    sl.tm.host_finish_ms += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    sl.tm.d2h_bytes += PROOF64 * 8;
    tm = sl.tm;
    return G16_OK;
  }
  int prove(const uint64_t* r, const uint64_t* s, const uint64_t* z, uint32_t flags, uint64_t* proof) override {
    if (!proof) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    int rc = prove_submit(0, r, s, z, flags);
    if (rc) return rc;
    return prove_wait(0, proof);
  }

  // ---- batch proving (g16_prove_batch) ----
  // The proofs of a group share every launch: proof k owns bucket sets k*ne .. k*ne+ne-1 of each MSM over the same resident
  // bases (msm_digits, blockIdx.y = k), so one sort, one set of batched-affine rounds and one bucket reduction per MSM
  // serve the group, and the group's 7 transforms are one launch per NTT pass.  Groups alternate between the two proof
  // slots (proof_slots = 2): the host tail of group g overlaps the GPU work of group g + 1.
  cudaEvent_t ev_batch = nullptr;   // start of the current g16_prove_batch call (timings)
  // padded sorted entries of the largest MSM of one proof, at the largest bucket padding the rounds can ask for
  uint64_t batch_entries_per_proof() const {
    uint64_t e = 0;
    for (const Query& x : q)
      if (x.hi > x.lo) e = std::max<uint64_t>(e, x.geom.max_entries + (uint64_t)x.geom.nkeys * ((1u << MSM_BA_MAX_ROUNDS) - 1));
    return e;
  }
  // device workspace of one proof of a group (upper bound): work vectors, the fixed-base scalars and products, and every
  // MSM's workspace (msm_batch_bytes_per_proof) at the smallest k0 with_k0 can pick under the current knobs (acc_k0 4 .. 7
  // goes below the automatic floor), any round count and, for the B MSMs sharing one sorted list, any padding
  uint64_t batch_bytes_per_proof() const {
    const uint64_t n = 1ull << L;
    uint64_t b = nvars() * sizeof(Fr) + 5 * n * sizeof(Fr) + 3 * sizeof(Fr) + 4 * sizeof(A1) + sizeof(A2);
    for (int m = 0; m < 5; m++) {
      if (q[m].hi <= q[m].lo) continue;
      const bool g2 = m == M_B2;
      const int k0_min = msm_k0_floor(g2, g2 ? tune.k0_g2 : tune.k0_g1);
      const bool shared = share_b_sort && (m == M_B1 || m == M_B2);
      b += g2 ? msm_batch_bytes_per_proof<Fq2>(q[m].geom, k0_min, shared) : msm_batch_bytes_per_proof<Fq>(q[m].geom, k0_min, shared);
    }
    return b;
  }
  // geometry of `count` proofs' MSMs in one pass: the single proof's windows, k0 and rounds re-derived from the entry count
  void batch_geoms(uint32_t count, bool share, MsmGeom* gb) const {
    for (int m = 0; m < 5; m++) {
      gb[m] = with_k0(msm_geom_batch(q[m].geom, count), m == M_B2, m);
      gb[m].ba_pad = gb[m].ba;
    }
    if (share) gb[M_B1].ba_pad = gb[M_B2].ba_pad = std::max(gb[M_B1].ba, gb[M_B2].ba);   // one padding for the shared list
  }
  int ensure_tail_tables() {
    if (tail_ready) return G16_OK;
    const A1 gens[3] = {delta_g1, p_a, p_b};   // TAB_D1, TAB_PA, TAB_PB
    for (int t = 0; t < 3; t++) {
      G16_CUDA(tail_tab[t].reserve((size_t)fb_windows<Fr>() * 255 * sizeof(P1)));
      G16_CUDA((fb_batch_mul<Fq, Fr>(S0.st_main, gens[t], nullptr, 0, nullptr, tail_tab[t].template as<P1>())));
    }
    G16_CUDA(tail_tab[TAB_D2].reserve((size_t)fb_windows<Fr>() * 255 * sizeof(P2)));
    G16_CUDA((fb_batch_mul<Fq2, Fr>(S0.st_main, delta_g2, nullptr, 0, nullptr, tail_tab[TAB_D2].template as<P2>())));
    ctr.launches += 4;
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    tail_ready = true;
    return G16_OK;
  }
  static size_t tail_scalar_bytes(uint32_t count) { return (size_t)3 * count * sizeof(Fr); }
  static size_t tail_point_bytes(uint32_t count) { return (size_t)count * (4 * sizeof(A1) + sizeof(A2)); }
  // enqueue proofs first .. first + count - 1 on the slot's streams
  int batch_submit(Slot& sl, uint32_t first, uint32_t count, const uint64_t* r, const uint64_t* s, const uint64_t* z, uint32_t flags) {
    const uint64_t nv = nvars();
    sl.serial = (flags & G16_SERIAL_MSMS) != 0;
    sl.batch_first = first;
    sl.batch_count = count;
    const size_t sc_bytes = tail_scalar_bytes(count), pt_bytes = tail_point_bytes(count);
    G16_CUDA(sl.d_tail.reserve(sc_bytes + pt_bytes));
    if (sl.h_tail_cap < sc_bytes + pt_bytes) {
      if (sl.h_tail) cudaFreeHost(sl.h_tail);
      sl.h_tail = nullptr;
      sl.h_tail_cap = 0;
      G16_CUDA(cudaMallocHost(&sl.h_tail, sc_bytes + pt_bytes));
      sl.h_tail_cap = sc_bytes + pt_bytes;
    }
    Fr* hsc = reinterpret_cast<Fr*>(sl.h_tail);   // r[count], s[count], (r s)[count]
    for (uint32_t k = 0; k < count; k++) {
      hsc[k] = load_fr(r + FR64 * (size_t)(first + k));
      hsc[count + k] = load_fr(s + FR64 * (size_t)(first + k));
      hsc[2 * count + k] = Fr::mul(hsc[k], hsc[count + k]);
    }
    int rc;
    {
      NvtxSpan span_wm(SPAN_WITNESS_MAP);
      rc = enqueue_witness_map(sl, z + (size_t)first * nv * FR64, flags, count);
    }
    if (rc) return rc;
    // the five fixed-base products of every proof, after the witness map on its stream (the H MSM waits for ev_h only)
    cudaStream_t st = sl.st_main;
    G16_CUDA(cudaMemcpyAsync(sl.d_tail.p, sl.h_tail, sc_bytes, cudaMemcpyHostToDevice, st));
    const Fr* d_r = sl.d_tail.template as<Fr>();
    const Fr* d_s = d_r + count;
    const Fr* d_rs = d_r + 2 * count;
    A1* o1 = reinterpret_cast<A1*>(sl.d_tail.template as<char>() + sc_bytes);   // r d1, (r s) d1, s P_a, r P_b
    A2* o2 = reinterpret_cast<A2*>(o1 + 4 * (size_t)count);                       // s d2
    G16_CUDA((fb_mul<Fq, Fr>(st, tail_tab[TAB_D1].template as<P1>(), d_r, count, o1)));
    G16_CUDA((fb_mul<Fq, Fr>(st, tail_tab[TAB_D1].template as<P1>(), d_rs, count, o1 + count)));
    G16_CUDA((fb_mul<Fq, Fr>(st, tail_tab[TAB_PA].template as<P1>(), d_s, count, o1 + 2 * (size_t)count)));
    G16_CUDA((fb_mul<Fq, Fr>(st, tail_tab[TAB_PB].template as<P1>(), d_r, count, o1 + 3 * (size_t)count)));
    G16_CUDA((fb_mul<Fq2, Fr>(st, tail_tab[TAB_D2].template as<P2>(), d_s, count, o2)));
    ctr.launches += 5;
    G16_CUDA(cudaMemcpyAsync(sl.h_tail + sc_bytes / 8, o1, pt_bytes, cudaMemcpyDeviceToHost, st));
    for (int m = 0; m < 5; m++) {
      sl.run[m] = q[m].hi > q[m].lo;
      sl.tm.msm_pairs[m] = sl.run[m] ? (q[m].hi - q[m].lo) * count : 0;
    }
    batch_geoms(count, share_b_sort && sl.run[M_B1] && sl.run[M_B2], sl.geom);
    return enqueue_msms(sl);
  }
  // wait for the slot's group, then finish its proofs on the pool (one proof per task); adds the group to `acc`.  Under
  // G16_CHECK_WITNESS a rejected proof is written as all-zero limbs, and the first one of the call is kept in *rejected
  // (index, reason)
  int batch_finish(Slot& sl, const uint64_t* r, const uint64_t* s, uint64_t* proofs, g16_timings& acc, float* host_ms,
                   std::pair<int64_t, std::string>* rejected) {
    const uint32_t count = sl.batch_count, first = sl.batch_first;
    sl.batch_count = 0;
    for (int m = 0; m < 5 && !sl.serial; m++) G16_CUDA(cudaStreamSynchronize(sl.st_msm[m]));
    G16_CUDA(cudaStreamSynchronize(sl.st_main));
    const auto t0 = std::chrono::steady_clock::now();
    const A1* o1 = reinterpret_cast<const A1*>(sl.h_tail + tail_scalar_bytes(count) / 8);
    const A2* o2 = reinterpret_cast<const A2*>(o1 + 4 * (size_t)count);
    std::vector<std::shared_ptr<HostPool::Ticket>> tk(count);
    for (uint32_t k = 0; k < count; k++) {
      if (sl.check) {
        const g16_witness_report w = report_of(sl.h_check + 3 * (size_t)k);
        if (!report_ok(w)) {
          memset(proofs + (size_t)(first + k) * PROOF64, 0, PROOF64 * sizeof(uint64_t));   // three identity points
          if (rejected->first < 0) *rejected = {(int64_t)(first + k), report_reason(w)};   // groups finish in order
          continue;
        }
      }
      tk[k] = pool->submit([&, k]() {
        const Products kp{P1::from_affine(o1[k]), P1::from_affine(o1[count + k]), P1::from_affine(o1[2 * (size_t)count + k]),
                          P1::from_affine(o1[3 * (size_t)count + k]), P2::from_affine(o2[k])};
        Partials x;
        P1* outs[4] = {&x.h, &x.l, &x.a, &x.b1};
        for (int m = 0; m < 4; m++) *outs[m] = sl.run[m] ? msm_finish<Fq>(sl.ws1[m], sl.geom[m], k) : P1::inf();
        x.b2 = sl.run[M_B2] ? msm_finish<Fq2>(sl.ws2, sl.geom[M_B2], k) : P2::inf();
        const Fr rk = load_fr(r + FR64 * (size_t)(first + k)), sk = load_fr(s + FR64 * (size_t)(first + k));
        store_proof(proofs + (size_t)(first + k) * PROOF64, kp, x.a, x.b2, c_part(rk, sk, x));
      });
    }
    for (auto& t : tk) if (t) t->wait();
    *host_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    add_timings(sl, ev_batch, first == 0, acc);
    acc.d2h_bytes += tail_point_bytes(count);
    return G16_OK;
  }
  int prove_batch(uint32_t count, const uint64_t* r, const uint64_t* s, const uint64_t* z, uint32_t group, uint32_t flags,
                  uint64_t* proofs) override {
    if (count == 0) return G16_OK;
    if (!r || !s || !z || !proofs) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    if (!have_circuit || !have_pk) return fail(G16_ERR_BAD_ARGUMENT, "circuit and proving key must be resident");
    if (world != 1) return fail(G16_ERR_BAD_ARGUMENT, "key is sharded: batch proving needs the whole key (world 1)");
    G16_NOT_BUSY();
    G16_CUDA(cudaSetDevice(device));
    NvtxSpan span(SPAN_PROVER);
    int rc = ensure_tail_tables();
    if (rc) return rc;
    size_t free_b = 0, total_b = 0;
    G16_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const uint32_t nslots = (uint32_t)tune.proof_slots;
    const uint32_t G = batch_group_size(count, group, batch_entries_per_proof(), batch_bytes_per_proof(), free_b, nslots);
    const unsigned long long launches0 = ctr.launches + ntt_launches;
    if (!ev_batch) G16_CUDA(cudaEventCreate(&ev_batch));
    G16_CUDA(cudaEventRecord(ev_batch, slots[0].st_main));
    g16_timings acc{};
    float host_ms = 0;
    std::pair<int64_t, std::string> rejected{-1, std::string()};   // lowest proof rejected by G16_CHECK_WITNESS
    int order[NSLOTS] = {-1, -1};   // slots holding a group, oldest first
    auto finish_oldest = [&]() -> int {
      const int si = order[0];
      order[0] = order[1];
      order[1] = -1;
      return batch_finish(slots[si], r, s, proofs, acc, &host_ms, &rejected);
    };
    for (uint32_t first = 0, gi = 0; first < count && !rc; first += G, gi++) {
      const int si = nslots > 1 ? (int)(gi & 1) : 0;
      if (slots[si].batch_count) rc = finish_oldest();   // the slot's previous group (with one slot: the only one)
      if (!rc) rc = batch_submit(slots[si], first, std::min(G, count - first), r, s, z, flags);
      if (!rc) order[order[0] < 0 ? 0 : 1] = si;
    }
    while (!rc && order[0] >= 0) rc = finish_oldest();
    if (rc) {   // leave no group half-finished behind
      cudaDeviceSynchronize();
      for (Slot& sl : slots) sl.batch_count = 0;
      return rc;
    }
    acc.host_finish_ms = host_ms;   // host work after the last group's GPU work
    acc.launches = ctr.launches + ntt_launches - launches0;
    tm = acc;
    if (rejected.first >= 0) return fail(G16_ERR_UNSATISFIED, "proof " + std::to_string(rejected.first) + ": " + rejected.second);
    return G16_OK;
  }
  // ---- sharded proof with the exchange inside the library (g16_comm_init + g16_prove_sharded*) ----
  // Every rank holds pair i of every MSM with i mod world == rank.  Per proof a rank contributes THREE points:
  //   A_k (its share of the A MSM), B2_k (its share of B in G2) and C_k = s A_k + r B1_k + L_k + H_k,
  // in XYZZ coordinates (no inversion on the exchange path): 2 * 4 * Fq + 4 * Fq2 limbs = 768 B on BLS12-381.  One
  // ncclAllGather of that record on a dedicated high-priority stream, then every rank adds the records in rank order and
  // finishes the same proof (EC addition is exactly associative and commutative: bit-identical for any world size).
  void* nccl_comm = nullptr;      // all-gather of the partial proof points (stream st_comm)
  void* nccl_comm_wm = nullptr;   // witness-map exchange (send / recv / broadcast on the proof slot's main stream)
  uint32_t comm_rank = 0, comm_world = 0;
  cudaStream_t st_comm = nullptr;
  DevBuf d_comm_send, d_comm_recv;
  uint64_t* h_comm_send = nullptr;   // pinned
  uint64_t* h_comm_recv = nullptr;   // pinned, world records
  static constexpr size_t REC_LIMBS = 2 * 4 * (size_t)NQ64 + sizeof(P2) / 8;   // A_k, C_k (XYZZ G1), B2_k (XYZZ G2)
  void comm_release() {
    if (nccl_comm && nccl_api().CommDestroy) nccl_api().CommDestroy(nccl_comm);
    if (nccl_comm_wm && nccl_api().CommDestroy) nccl_api().CommDestroy(nccl_comm_wm);
    nccl_comm = nccl_comm_wm = nullptr;
    if (h_comm_send) cudaFreeHost(h_comm_send);
    if (h_comm_recv) cudaFreeHost(h_comm_recv);
    h_comm_send = h_comm_recv = nullptr;
    d_comm_send.release();
    d_comm_recv.release();
    if (st_comm) cudaStreamDestroy(st_comm);
    st_comm = nullptr;
  }
  int comm_init(const uint8_t* id128, uint32_t rk, uint32_t wd) override {   // id128: TWO NCCL unique ids (256 bytes)
    if (!id128 || wd == 0 || rk >= wd) return fail(G16_ERR_BAD_ARGUMENT, "bad unique id / rank / world");
    G16_NOT_BUSY();
    NcclApi& api = nccl_api();
    if (!api.load()) return fail(G16_ERR_CUDA, "NCCL is not available: " + api.err);
    G16_CUDA(cudaSetDevice(device));
    comm_release();
    NcclUniqueId id;
    memcpy(id.internal, id128, 128);
    int rc = api.CommInitRank(&nccl_comm, (int)wd, id, (int)rk);
    if (rc != 0) { nccl_comm = nullptr; return fail(G16_ERR_CUDA, std::string("ncclCommInitRank: ") + api.GetErrorString(rc)); }
    memcpy(id.internal, id128 + 128, 128);
    rc = api.CommInitRank(&nccl_comm_wm, (int)wd, id, (int)rk);
    if (rc != 0) { nccl_comm_wm = nullptr; return fail(G16_ERR_CUDA, std::string("ncclCommInitRank (witness map): ") + api.GetErrorString(rc)); }
    comm_rank = rk;
    comm_world = wd;
    int prio_lo = 0, prio_hi = 0;
    G16_CUDA(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
    G16_CUDA(cudaStreamCreateWithPriority(&st_comm, cudaStreamNonBlocking, prio_hi));
    nvtxNameCudaStreamA(st_comm, "NCCL all-gather of the partial proof points");
    G16_CUDA(d_comm_send.reserve(REC_LIMBS * 8));
    G16_CUDA(d_comm_recv.reserve(REC_LIMBS * 8 * wd));
    G16_CUDA(cudaMallocHost(&h_comm_send, REC_LIMBS * 8));
    G16_CUDA(cudaMallocHost(&h_comm_recv, REC_LIMBS * 8 * wd));
    // one warm-up exchange: NCCL builds its channels on first use (tens of ms), keep that out of the first proof
    G16_CUDA(cudaMemsetAsync(d_comm_send.p, 0, REC_LIMBS * 8, st_comm));
    rc = api.AllGather(d_comm_send.p, d_comm_recv.p, REC_LIMBS * 8, /*ncclUint8*/ 1, nccl_comm, st_comm);
    if (rc != 0) return fail(G16_ERR_CUDA, std::string("ncclAllGather (warm-up): ") + api.GetErrorString(rc));
    G16_CUDA(cudaStreamSynchronize(st_comm));
    return G16_OK;
  }
  int sharded_submit(int slot, const uint64_t* r, const uint64_t* s, const uint64_t* z, uint32_t flags) override {
    if (slot < 0 || slot >= NSLOTS) return fail(G16_ERR_BAD_ARGUMENT, "bad slot");
    if (!s) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    if (!nccl_comm) return fail(G16_ERR_BAD_ARGUMENT, "g16_comm_init must precede g16_prove_sharded");
    if (comm_world != world || comm_rank != rank) return fail(G16_ERR_BAD_ARGUMENT, "the key's (rank, world) differs from the communicator's");
    slots[slot].split_wm = tune.wm_split && comm_world > 1;
    const int rc = submit(slots[slot], r, s, z, flags);
    slots[slot].split_wm = false;
    return rc;
  }
  template <class PT>
  static uint64_t* put_xyzz(uint64_t* p, const PT& x) { memcpy(p, &x, sizeof(PT)); return p + sizeof(PT) / 8; }
  template <class PT>
  static const uint64_t* get_xyzz(const uint64_t* p, PT& x) { memcpy(&x, p, sizeof(PT)); return p + sizeof(PT) / 8; }
  int sharded_wait(int slot, uint64_t* proof) override {
    if (slot < 0 || slot >= NSLOTS || !proof) return fail(G16_ERR_BAD_ARGUMENT, "bad slot / null buffer");
    if (!nccl_comm) return fail(G16_ERR_BAD_ARGUMENT, "g16_comm_init must precede g16_prove_sharded");
    Slot& sl = slots[slot];
    Partials x;
    int rc = wait_proof(sl, x);
    if (rc) return rc;
    auto t0 = std::chrono::steady_clock::now();
    static_assert(sizeof(P1) == 4 * sizeof(Fq) && sizeof(P2) == 4 * sizeof(Fq2), "XYZZ records are packed");
    uint64_t* w = h_comm_send;
    w = put_xyzz(w, x.a);
    w = put_xyzz(w, c_part(sl.r, sl.s, x));
    w = put_xyzz(w, x.b2);
    NcclApi& api = nccl_api();
    G16_CUDA(cudaMemcpyAsync(d_comm_send.p, h_comm_send, REC_LIMBS * 8, cudaMemcpyHostToDevice, st_comm));
    rc = api.AllGather(d_comm_send.p, d_comm_recv.p, REC_LIMBS * 8, /*ncclUint8*/ 1, nccl_comm, st_comm);
    if (rc != 0) return fail(G16_ERR_CUDA, std::string("ncclAllGather: ") + api.GetErrorString(rc));
    G16_CUDA(cudaMemcpyAsync(h_comm_recv, d_comm_recv.p, REC_LIMBS * 8 * comm_world, cudaMemcpyDeviceToHost, st_comm));
    G16_CUDA(cudaStreamSynchronize(st_comm));
    // every rank checked the same assignment and reaches the same verdict, but only after its part of every exchange: a
    // rank that left one out would leave the others waiting
    if ((rc = slot_verdict(sl))) return rc;
    P1 a_sum = P1::inf(), c_sum = P1::inf();
    P2 b2_sum = P2::inf();
    for (uint32_t k = 0; k < comm_world; k++) {           // fixed rank order; the sum is order-independent anyway
      const uint64_t* p = h_comm_recv + (size_t)k * REC_LIMBS;
      P1 a, c;
      P2 b2;
      p = get_xyzz(p, a);
      p = get_xyzz(p, c);
      p = get_xyzz(p, b2);
      a_sum.add(a);
      c_sum.add(c);
      b2_sum.add(b2);
    }
    store_proof(proof, sl.kp, a_sum, b2_sum, c_sum);
    sl.tm.host_finish_ms += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    sl.tm.d2h_bytes += REC_LIMBS * 8 * comm_world;
    tm = sl.tm;
    return G16_OK;
  }

  // Sharded path: the key products can be started before the partial sums exist
  // (g16_prove_assemble_prepare), so that they overlap the GPU work and the gather; prove_assemble picks them up.
  Fr asm_r, asm_s;
  Products asm_kp;
  bool asm_valid = false;   // asm_kp belongs to (asm_r, asm_s) under the resident key
  std::shared_ptr<HostPool::Ticket> asm_helper;
  int assemble_prepare(const uint64_t* r, const uint64_t* s) override {
    if (!have_pk) return fail(G16_ERR_BAD_ARGUMENT, "no proving key resident");
    if (!r || !s) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    if (asm_helper) asm_helper->wait();
    asm_r = load_fr(r);
    asm_s = load_fr(s);
    asm_valid = true;
    asm_helper = pool->submit([this]() { asm_kp = key_products(asm_r, asm_s); });
    return G16_OK;
  }
  int prove_assemble(const uint64_t* r, const uint64_t* s, const uint64_t* partials, uint32_t nparts, uint64_t* proof) override {
    if (!have_pk) return fail(G16_ERR_BAD_ARGUMENT, "no proving key resident");
    if (!r || !s || !partials || !proof || nparts == 0) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    if (asm_helper) { asm_helper->wait(); asm_helper.reset(); }
    Partials x{P1::inf(), P1::inf(), P1::inf(), P1::inf(), P2::inf()};
    const int pl = partial_limbs();
    for (uint32_t i = 0; i < nparts; i++) {   // fixed rank order; the sum is order-independent anyway
      const uint64_t* p = partials + (size_t)i * pl;
      x.h.madd(load_a1(p));
      x.l.madd(load_a1(p + 2 * NQ64));
      x.a.madd(load_a1(p + 4 * NQ64));
      x.b1.madd(load_a1(p + 6 * NQ64));
      x.b2.madd(load_a2(p + 8 * NQ64));
    }
    const Fr rr = load_fr(r), ss = load_fr(s);
    const bool prepared = asm_valid && rr == asm_r && ss == asm_s;
    store_proof(proof, prepared ? asm_kp : key_products(rr, ss), x.a, x.b2, c_part(rr, ss, x));
    return G16_OK;
  }
};

// extern-template declarations for one curve: put before make_engine<CP> is instantiated (engine_<curve>.cu)
#define G16_CURVE_KERNELS(X, CP)                                                                  \
  G16_NTT_TEMPLATES(X, Fp<CP::FrP>)                                                               \
  G16_MSM_TEMPLATES(X, Fp<CP::FqP>, Fp<CP::FrP>)                                                  \
  G16_MSM_TEMPLATES(X, G16_FQ2(CP), Fp<CP::FrP>)                                                  \
  G16_SER_TEMPLATES(X, CP)                                                                        \
  G16_SRS_TEMPLATES(X, CP)                                                                        \
  G16_SRS_POINT_TEMPLATES(X, G16_FQ2(CP), Fp<CP::FrP>)
#define G16_FQ2(CP) CP::G2F

template <class CP>
IEngine* make_engine(int device, int* rc) {
  auto* e = new Engine<CP>();
  *rc = e->init(device);
  if (*rc) { delete e; return nullptr; }
  return e;
}

}  // namespace g16
