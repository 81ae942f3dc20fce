// engine.cuh -- per-curve host orchestration of the proving hot path behind the C ABI (include/g16b200.h).
//
// Mirrors, function by function, what /root/reference does between `create_proof_with_reduction_and_matrices`
// (prover.rs:26-51) and `Proof{a,b,c}` (prover.rs:127-131); the heavy steps are the CUDA kernels of ntt.cuh and
// msm.cuh, the O(1) tail (six scalar multiplications, sums, into_affine) runs on the host with the same field code.
#pragma once
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>       // header-only NVTX v3: no-ops unless a profiler injects itself
#include <nvtx3/nvToolsExtCudaRt.h>
#include <algorithm>
#include <chrono>
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
#include "ec.cuh"
#include "msm.cuh"
#include "ntt_tma.cuh"

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
  virtual int partial_limbs() const = 0;
  virtual int ntt(uint32_t log_n, int inverse, int coset, uint64_t* inout) = 0;
  virtual int witness_map_evals(uint32_t log_n, const uint64_t* a, const uint64_t* b, const uint64_t* c, uint64_t* h) = 0;
  virtual int msm_g1(const uint64_t* bases, const uint64_t* scalars, uint64_t n, uint64_t* out) = 0;
  virtual int msm_g2(const uint64_t* bases, const uint64_t* scalars, uint64_t n, uint64_t* out) = 0;
  virtual int circuit_load(uint32_t ni, uint32_t nc, uint32_t nw, const g16_csr* a, const g16_csr* b, const g16_csr* c) = 0;
  virtual int pk_load(const g16_pk_desc* pk, uint32_t rank, uint32_t world) = 0;
  virtual int setup(const uint64_t* alpha, const uint64_t* beta, const uint64_t* gamma, const uint64_t* delta,
                    const uint64_t* tau, const uint64_t* g1, const uint64_t* g2) = 0;
  virtual int pk_export(const g16_pk_export_desc* out) = 0;
  virtual int prove(const uint64_t* r, const uint64_t* s, const uint64_t* z, uint32_t flags, uint64_t* proof) = 0;
  virtual int prove_partial(const uint64_t* r, const uint64_t* z, uint32_t flags, uint64_t* partial) = 0;
  virtual int prove_assemble(const uint64_t* r, const uint64_t* s, const uint64_t* partials, uint32_t nparts, uint64_t* proof) = 0;
  virtual int assemble_prepare(const uint64_t* r, const uint64_t* s) = 0;
  virtual int prove_submit(int slot, const uint64_t* r, const uint64_t* s, const uint64_t* z, uint32_t flags) = 0;
  virtual int prove_wait(int slot, uint64_t* proof) = 0;
  virtual int partial_submit(int slot, const uint64_t* r, const uint64_t* z, uint32_t flags) = 0;
  virtual int partial_wait(int slot, uint64_t* partial) = 0;
  virtual int witness_map(const uint64_t* z, uint32_t flags, uint64_t* h) = 0;
  virtual uint32_t domain_log() const = 0;
  virtual int comm_init(const uint8_t* id128, uint32_t rank, uint32_t world) = 0;
  virtual int sharded_submit(int slot, const uint64_t* r, const uint64_t* s, const uint64_t* z, uint32_t flags) = 0;
  virtual int sharded_wait(int slot, uint64_t* proof) = 0;
  virtual int set_option(const char* key, long long value) = 0;
  virtual int get_config(g16_config* out) const = 0;
  g16_timings tm{};
};

// ------------------------------------------------------------------------------------------------
template <class CP>
struct Engine : IEngine {
  using Fr = Fp<typename CP::FrP>;
  using Fq = Fp<typename CP::FqP>;
  using Fq2 = Fp2<typename CP::FqP, CP::FQ2_NONRESIDUE_NEG>;
  using A1 = Affine<Fq>;
  using A2 = Affine<Fq2>;
  using P1 = XYZZ<Fq>;
  using P2 = XYZZ<Fq2>;
  static constexpr int NQ64 = Fq::N / 2;
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
  // (r, s, key)-only parts of the proof, computed on pool threads while the GPU works (prover.rs:76,90-92,100-101,112-113):
  //   ga0 = r*delta_g1 + a_query[0] + alpha_g1        s_ga0 = s * ga0            neg_rs_d1 = -(r*s) * delta_g1
  //   r_gb0 = r * (s*delta_g1 + b_g1_query[0] + beta_g1)   (identity when r == 0)   gb2_0 = s*delta_g2 + b_g2_query[0] + beta_g2
  struct FixedMuls { P1 ga0, s_ga0, r_gb0, neg_rs_d1; P2 gb2_0; };
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
    FixedMuls fx;
    std::shared_ptr<HostPool::Ticket> helper, helper2;   // (r, s)-only scalar multiplications in flight on the pool
    unsigned long long launches0 = 0;
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
  uint32_t num_inputs = 0, num_constraints = 0, num_witness = 0;
  int L = 0;
  DevBuf csr_rp[3], csr_col[3], csr_val[3];
  std::vector<uint32_t> h_rp[3], h_col[3];   // host copies kept for g16_setup
  std::vector<Fr> h_val[3];

  // resident proving key (this rank's shard)
  bool have_pk = false;
  uint32_t rank = 0, world = 1;
  struct Query {
    DevBuf bases, mask;   // bases: geom.copies * (hi - lo) affine points, copy-major (copy j = 2^(c*ne*j) * P)
    uint64_t pairs = 0;   // full MSM length
    uint64_t lo = 0, hi = 0;   // this rank owns pairs lo, lo + world, lo + 2 world, ... : hi - lo of them (lo = rank)
    MsmGeom geom{};
  } q[5];
  // MSM tuning knobs: defaults below, overridden at context creation by the environment (G16_MSM_C, G16_MSM_NE,
  // G16_MSM_MAXCOPIES, G16_MSM_BA, G16_MSM_BA_G2, G16_BA_M, G16_BA_G, G16_BA_INV_GCD, G16_ACC_K0_G1, G16_ACC_K0_G2,
  // G16_ACC_BLOCK) and at run time by g16_set_option (same names, lower case, without the G16_ prefix).
  int cfg_c = 0;          // 0 = pick from n
  int cfg_ne = 1;         // effective windows with precomputed bases; 0 = no precomputation
  int cfg_maxcopies = MSM_MAX_COPIES;
  struct Tune {
    // defaults from sweeps of a full proof at 2^20 (tools/sweep.py)
    int ba_g1 = 4;        // batched-affine rounds before the XYZZ accumulation, G1 MSMs with >= 2^18 entries
    int ba_g2 = 4;        // same for the G2 MSM (on an H100 a fifth round costs more than it saves)
    int ba_m = 32;        // additions per thread and round
    int ba_G = 16;        // thread products per inversion
    int ba_gcd = 1;       // safegcd inversion
    int k0_g1 = 0;        // sorted entries per accumulation thread (0 = automatic)
    int k0_g2 = 0;
    int acc_block = 128;
    int ba_occ_g2 = 0;    // != 0: register-lean Fq2 round kernels, 3 resident blocks per SM (168 registers; msm_ba.cuh)
    int ba_occ_g1 = 0;    // != 0: register-lean G1 round kernels, 5 resident blocks per SM
    int ba_cap_fwd_g1 = 0, ba_cap_bwd_g1 = 0;   // blocks per SM of a forward / backward round launch (0 = one block per tile)
    int ba_cap_fwd_g2 = 0, ba_cap_bwd_g2 = 0;
    // Smallest MSM (in bucket entries) that runs the rounds, and how many: a round halves a list whose buckets hold
    // `entries / buckets` slots on average and pads every bucket to 2^R slots, so R is the smallest value with
    // 11 * 2^R >= that average, capped by ba_g1 / ba_g2 (4 / 4 at
    // 2^20 pairs on one GPU, 3 on the 2.1 M-entry shards of an 8-way proof, 2 on its 1.0 M-entry A / B shards).
    long long ba_min_g1 = 1ll << 19;
    long long ba_min_g2 = 1ll << 19;
    int ba_adaptive = 1;  // 0: exactly ba_g1 / ba_g2 rounds whatever the bucket occupancy (tests)
  } tune;
  MsmGeom pick_geom(uint64_t cnt) const {
    if (cfg_ne <= 0) return msm_geom(cnt, FR_BITS, cfg_c, 0);
    // with all windows sharing one bucket set the bucket count is 2^(c-1) whatever the size: c = 16 from 2^16 pairs up
    // (also for the per-rank shards of a multi-GPU run), the size-based rule below that
    const int c = cfg_c > 0 ? cfg_c : (cnt >= (1u << 16) ? 16 : 0);
    MsmGeom g = msm_geom(cnt, FR_BITS, c, cfg_ne);
    int ne = cfg_ne;
    while (g.copies > cfg_maxcopies) g = msm_geom(cnt, FR_BITS, c, ++ne);
    return g;
  }
  // entries per level-0 thread, from the number of resident accumulation threads of this device
  int sm_count = 132;
  int proof_slots = NSLOTS;   // slots the caller will use (g16_set_option "proof_slots" 1 halves the workspace the key must leave room for)
  bool ba_allowed = true;   // cleared by pk_load / setup when the rounds' work lists would not fit in device memory
  uint32_t ba_allowed_mask = 0x1f;   // per MSM (bit m): the work lists of MSM m fit next to the key and the other MSMs' lists
  MsmGeom with_k0(MsmGeom g, bool g2, int m = -1) const {
    g.k0 = msm_pick_k0(g.max_entries, (uint64_t)sm_count * 128 * (g2 ? 2 : 3), g2 ? 16 : 8);
    // G2 additions are ~3x longer: 32 entries per thread (twice the thread count) shortens the last partial wave (-13 %)
    if (g2 && g.k0 > 32) g.k0 = 32;
    const int k = g2 ? tune.k0_g2 : tune.k0_g1;
    if (k >= 4 && k <= 1024) g.k0 = k;
    // batched-affine pre-reduction (msm_ba.cuh) for MSMs with at least 2^18 entries
    const int r = g2 ? tune.ba_g2 : tune.ba_g1;
    const bool allowed = ba_allowed && (m < 0 || ((ba_allowed_mask >> m) & 1));
    const uint64_t min_entries = (uint64_t)std::max(1ll << 18, g2 ? tune.ba_min_g2 : tune.ba_min_g1);
    int r_fit = 0;   // smallest R with 11 * 2^R >= average entries per bucket
    for (uint64_t per_bucket = g.max_entries / std::max<uint64_t>(1, g.nkeys); (11ull << r_fit) < per_bucket; r_fit++) {}
    if (!tune.ba_adaptive) r_fit = r;
    g.ba = (allowed && r > 0 && g.max_entries >= min_entries) ? std::min(std::min(r, r_fit), (int)MSM_BA_MAX_ROUNDS) : 0;
    g.ba_m = tune.ba_m;
    g.ba_G = tune.ba_G;
    g.ba_gcd = tune.ba_gcd;
    g.acc_block = tune.acc_block;
    g.ba_occ = g2 ? tune.ba_occ_g2 : tune.ba_occ_g1;
    g.ba_grid_fwd = sm_count * (g2 ? tune.ba_cap_fwd_g2 : tune.ba_cap_fwd_g1);
    g.ba_grid_bwd = sm_count * (g2 ? tune.ba_cap_bwd_g2 : tune.ba_cap_bwd_g1);
    return g;
  }
  int wm_first_opt = 0;        // g16_set_option "wm_first": 1 / 0 / -1 = automatic (sharded keys).  Off: with enough hardware work
                               // queues (CUDA_DEVICE_MAX_CONNECTIONS, see api.cu) the witness map is not held up, and delaying the
                               // other accumulations then only idles the GPU
  bool share_b_sort = false;   // set when a key is made resident: b_g1_query and b_g2_query have the same identity pattern
  bool share_b_sort_wanted = true;
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
    if (share_b_sort_wanted && cnt > 0 && cnt == y.hi - y.lo && x.lo == y.lo && x.geom.c == y.geom.c && x.geom.ne == y.geom.ne &&
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
      if ((uint64_t)proof_slots * (plain + used + need) + margin <= fr) { used += need; mask |= 1u << m; }
    }
    ba_allowed_mask = mask;
    refresh_geoms();
  }
  int set_option(const char* key, long long v) override {
    if (any_busy()) return fail(G16_ERR_BAD_ARGUMENT, "a proof is in flight");
    const std::string k(key ? key : "");
    if (k == "msm_ba") tune.ba_g1 = (int)v;
    else if (k == "msm_ba_g2") tune.ba_g2 = (int)v;
    else if (k == "ba_m") tune.ba_m = (int)std::max(1ll, std::min(v, 256ll));
    else if (k == "ba_g") tune.ba_G = (int)std::max(1ll, std::min(v, 4096ll));
    else if (k == "ba_inv_gcd") tune.ba_gcd = v ? 1 : 0;
    else if (k == "acc_k0_g1") tune.k0_g1 = (int)v;
    else if (k == "acc_k0_g2") tune.k0_g2 = (int)v;
    else if (k == "acc_block") tune.acc_block = (int)v;
    else if (k == "ba_occ_g2") tune.ba_occ_g2 = v != 0 ? 3 : 0;
    else if (k == "ba_occ_g1") tune.ba_occ_g1 = v != 0 ? 5 : 0;
    else if (k == "ba_cap_fwd_g1") tune.ba_cap_fwd_g1 = (int)std::max(0ll, std::min(v, 16ll));
    else if (k == "ba_cap_bwd_g1") tune.ba_cap_bwd_g1 = (int)std::max(0ll, std::min(v, 16ll));
    else if (k == "ba_cap_fwd_g2") tune.ba_cap_fwd_g2 = (int)std::max(0ll, std::min(v, 16ll));
    else if (k == "ba_cap_bwd_g2") tune.ba_cap_bwd_g2 = (int)std::max(0ll, std::min(v, 16ll));
    else if (k == "ba_adaptive") tune.ba_adaptive = v ? 1 : 0;
    else if (k == "ba_min_entries_g1") tune.ba_min_g1 = std::max(0ll, v);
    else if (k == "ba_min_entries_g2") tune.ba_min_g2 = std::max(0ll, v);
    else if (k == "ntt_tma") { use_ntt_tma = v < 0 ? -1 : (v != 0 ? 1 : 0); return G16_OK; }
    else if (k == "wm_first") { wm_first_opt = v < 0 ? -1 : (v ? 1 : 0); return G16_OK; }
    else if (k == "wm_split") { split_wm_wanted = v != 0; return G16_OK; }
    else if (k == "proof_slots") { proof_slots = v <= 1 ? 1 : NSLOTS; if (have_pk) decide_ba_memory(); return G16_OK; }
    // residency knobs: take effect at the NEXT g16_pk_load / g16_setup (they decide how many precomputed multiples a key keeps)
    else if (k == "msm_ne") { cfg_ne = (int)std::max(0ll, std::min(v, 32ll)); return G16_OK; }
    else if (k == "msm_c") { cfg_c = (v < 0 || v > 24) ? 0 : (int)v; return G16_OK; }
    else if (k == "msm_maxcopies") { cfg_maxcopies = (int)std::max(1ll, std::min(v, (long long)MSM_MAX_COPIES)); return G16_OK; }
    else if (k == "share_b_sort") { share_b_sort_wanted = v != 0; if (have_pk) { int rc = decide_b_sort_sharing(); if (rc) return rc; } }
    else return fail(G16_ERR_BAD_ARGUMENT, "unknown option: " + k);
    refresh_geoms();
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
    o->ba_m = tune.ba_m; o->ba_g = tune.ba_G; o->ba_inv_gcd = tune.ba_gcd; o->acc_block = tune.acc_block;
    o->sm_count = sm_count;
    o->world = (int32_t)world; o->rank = (int32_t)rank;
    o->ba_lean_g1 = g1.ba_occ != 0; o->ba_lean_g2 = g2.ba_occ != 0;
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
  A1 a0, b1_0, alpha_g1, beta_g1, delta_g1;
  A2 b2_0, beta_g2, delta_g2;
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
    pool.reset(new HostPool(7));
    if (const char* v = getenv("G16_MSM_C")) cfg_c = atoi(v);
    if (const char* v = getenv("G16_MSM_NE")) cfg_ne = atoi(v);
    if (const char* v = getenv("G16_MSM_MAXCOPIES")) cfg_maxcopies = std::max(1, std::min(atoi(v), (int)MSM_MAX_COPIES));
    auto env_int = [](const char* name, int& dst, int lo, int hi) {
      if (const char* v = getenv(name)) { const int x = atoi(v); if (x >= lo && x <= hi) dst = x; }
    };
    env_int("G16_MSM_BA", tune.ba_g1, 0, MSM_BA_MAX_ROUNDS);
    env_int("G16_MSM_BA_G2", tune.ba_g2, 0, MSM_BA_MAX_ROUNDS);
    env_int("G16_BA_M", tune.ba_m, 1, 256);
    env_int("G16_BA_G", tune.ba_G, 1, 4096);
    env_int("G16_BA_INV_GCD", tune.ba_gcd, 0, 1);
    env_int("G16_ACC_K0_G1", tune.k0_g1, 4, 1024);
    env_int("G16_ACC_K0_G2", tune.k0_g2, 4, 1024);
    env_int("G16_ACC_BLOCK", tune.acc_block, 32, 128);
    env_int("G16_BA_OCC_G2", tune.ba_occ_g2, 0, 3);
    env_int("G16_BA_OCC_G1", tune.ba_occ_g1, 0, 5);
    env_int("G16_BA_CAP_FWD_G1", tune.ba_cap_fwd_g1, 0, 16);
    env_int("G16_BA_CAP_BWD_G1", tune.ba_cap_bwd_g1, 0, 16);
    env_int("G16_BA_CAP_FWD_G2", tune.ba_cap_fwd_g2, 0, 16);
    env_int("G16_BA_CAP_BWD_G2", tune.ba_cap_bwd_g2, 0, 16);
    if (cfg_c < 0 || cfg_c > 24) cfg_c = 0;
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
  ~Engine() override {
    cudaSetDevice(device);
    for (Slot& sl : slots) {
      if (sl.helper) sl.helper->wait();
      if (sl.helper2) sl.helper2->wait();
    }
    if (asm_helper) asm_helper->wait();
    comm_release();
    pool.reset();
    cudaDeviceSynchronize();
    dom.release();
    dom_api.release();
    for (Slot& sl : slots) {
      sl.d_z.release(); sl.d_a.release(); sl.d_b.release(); sl.d_c.release(); sl.d_t.release(); sl.d_h.release();
      for (auto& w : sl.ws1) w.release();
      sl.ws2.release();
      if (sl.st_main) cudaStreamDestroy(sl.st_main);
      for (auto s : sl.st_msm) if (s) cudaStreamDestroy(s);
      auto kill = [](cudaEvent_t ev) { if (ev) cudaEventDestroy(ev); };
      kill(sl.ev_start); kill(sl.ev_z); kill(sl.ev_h); kill(sl.ev_bsort);
      for (int i = 0; i < 5; i++) { kill(sl.ev_m0[i]); kill(sl.ev_m1[i]); kill(sl.ev_a0[i]); kill(sl.ev_a1[i]); }
    }
    for (int m = 0; m < 3; m++) { csr_rp[m].release(); csr_col[m].release(); csr_val[m].release(); }
    for (auto& x : q) { x.bases.release(); x.mask.release(); }
    d_gamma_abc.release(); full_a.release(); full_b1.release(); full_b2.release();
  }
  int fq_limbs() const override { return NQ64; }
  int partial_limbs() const override { return 4 * 2 * NQ64 + 4 * NQ64; }
  uint32_t domain_log() const override { return (uint32_t)L; }

  bool any_busy() const { return slots[0].busy || slots[1].busy; }
#define G16_NOT_BUSY() \
  if (any_busy()) return fail(G16_ERR_BAD_ARGUMENT, "a proof is in flight (g16_prove_wait / g16_prove_partial_wait it first)")

  // ---- small host helpers ----
  static Fr load_fr(const uint64_t* p) { Fr r; memcpy(r.v, p, sizeof(r.v)); return r; }
  static A1 load_a1(const uint64_t* p) { A1 r; memcpy(&r.x, p, sizeof(Fq)); memcpy(&r.y, p + NQ64, sizeof(Fq)); return r; }
  static A2 load_a2(const uint64_t* p) {
    A2 r;
    memcpy(&r.x.c0, p, sizeof(Fq)); memcpy(&r.x.c1, p + NQ64, sizeof(Fq));
    memcpy(&r.y.c0, p + 2 * NQ64, sizeof(Fq)); memcpy(&r.y.c1, p + 3 * NQ64, sizeof(Fq));
    return r;
  }
  static void store_a1(uint64_t* p, const A1& a) { memcpy(p, &a.x, sizeof(Fq)); memcpy(p + NQ64, &a.y, sizeof(Fq)); }
  static void store_a2(uint64_t* p, const A2& a) {
    memcpy(p, &a.x.c0, sizeof(Fq)); memcpy(p + NQ64, &a.x.c1, sizeof(Fq));
    memcpy(p + 2 * NQ64, &a.y.c0, sizeof(Fq)); memcpy(p + 3 * NQ64, &a.y.c1, sizeof(Fq));
  }
  // Jacobian normalised to Z = 1 (identity: (1,1,0) like ark)
  template <class F, class PT>
  static void store_proj(uint64_t* p, const PT& pt) {
    Affine<F> a = pt.to_affine();
    F one = F::one(), zero = F::zero();
    const size_t w = sizeof(F) / 8;
    if (pt.is_inf()) { memcpy(p, &one, sizeof(F)); memcpy(p + w, &one, sizeof(F)); memcpy(p + 2 * w, &zero, sizeof(F)); }
    else { memcpy(p, &a.x, sizeof(F)); memcpy(p + w, &a.y, sizeof(F)); memcpy(p + 2 * w, &one, sizeof(F)); }
  }
  static void fr_to_canon(const Fr& m, uint32_t out[8]) {
    Fr c = Fr::from_mont(m);
    memcpy(out, c.v, 32);
  }
  static int check_log(uint32_t log_n) {
    if ((int)log_n > CP::FrP::TWO_ADICITY) return fail(G16_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "domain size exceeds the field's two-adicity (PolynomialDegreeTooLarge)");
    if (log_n > 28) return fail(G16_ERR_BAD_ARGUMENT, "log_n > 28 unsupported");
    return G16_OK;
  }

  // ---- domain + buffers ----
  int ensure_slot_buffers(Slot& sl, int Ln) {
    const size_t bytes = (size_t)sizeof(Fr) << Ln;
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
  // the resident circuit's domain must be the one the prover / setup run with
  int ensure_circuit_domain() { return ensure_domain(dom, L); }
  // stand-alone transforms: the circuit's tables when the size matches, a separate domain otherwise
  NttDomain<Fr>* api_domain(int Ln, int* rc) {
    NttDomain<Fr>* d = (have_circuit && Ln == L) ? &dom : &dom_api;
    *rc = ensure_domain(*d, Ln);
    return d;
  }

  // One transform: the TMA-tiled passes (ntt_tma.cuh) from 2^14 points up, the generic passes (ntt.cuh) below that or
  // when the tensor-map encoder is unavailable / switched off (g16_set_option "ntt_tma" 0).
  // Measured on an H100 (tools/sweep.py, BLS12-381 at 2^20): the TMA plan halves the passes' DRAM traffic but loses on
  // time -- its 128 KB tiles are only 256 CTAs for 132 SMs (1.9 waves, one CTA per SM, no overlap of load / butterflies /
  // store): witness map 2.61 ms against 2.30 ms with the generic passes.  It is therefore OFF by default and selectable
  // (g16_set_option "ntt_tma" 1) -- DESIGN.md section 3 has the analysis.  1 = from 2^14 points, 0 / -1 = generic passes.
  int use_ntt_tma = 0;
  void ntt_any(cudaStream_t st, const NttDomain<Fr>& d, bool inverse, const Fr* src, Fr* work, Fr* dst, int load_mode, const Fr* ltab,
               const Fr* in_b, const Fr* in_c, const Fr& load_cst, int store_mode, const Fr* stab, const Fr& store_cst) {
    const bool tma = use_ntt_tma > 0;
    if (tma && ntt2_run<Fr>(st, d, inverse, src, work, dst, load_mode, ltab, in_b, in_c, load_cst, store_mode, stab, store_cst, &ntt_launches))
      return;
    ntt_run<Fr>(st, d, inverse, src, work, dst, load_mode, ltab, in_b, in_c, load_cst, store_mode, stab, store_cst, &ntt_launches);
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
  void witness_map_device(Slot& sl, const NttDomain<Fr>& dom) {
    cudaStream_t st = sl.st_main;
    Fr* A = sl.d_a.template as<Fr>(); Fr* B = sl.d_b.template as<Fr>(); Fr* C = sl.d_c.template as<Fr>(); Fr* T = sl.d_t.template as<Fr>(); Fr* H = sl.d_h.template as<Fr>();
    const Fr zero = Fr::zero();
    for (Fr* X : {A, B, C}) {
      // domain.ifft_in_place (r1cs_to_qap.rs:201-202,220) followed by coset_domain.fft_in_place (:204-207,221): the inverse
      // transform's n^-1 and the coset pre-scaling g^i are one multiplication by the table n^-1 g^i at the second load
      ntt_any(st, dom, true, X, X, T, NTT_LOAD_PLAIN, nullptr, nullptr, nullptr, zero, NTT_STORE_PLAIN, nullptr, zero);
      ntt_any(st, dom, false, T, T, X, NTT_LOAD_MUL_TABLE, dom.coset_fwd_ninv, nullptr, nullptr, zero, NTT_STORE_PLAIN, nullptr, zero);
    }
    // (a*b - c) * Z^-1 fused into the load of coset_domain.ifft_in_place (r1cs_to_qap.rs:209,223-232)
    ntt_any(st, dom, true, A, T, H, NTT_LOAD_AB_MINUS_C, nullptr, B, C, dom.z_inv, NTT_STORE_MUL_TABLE, dom.coset_inv, zero);
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
    for (int v = 0; v < 3; v++) {
      if (v % w != me) continue;
      ntt_any(st, dom, true, V[v], V[v], T, NTT_LOAD_PLAIN, nullptr, nullptr, nullptr, zero, NTT_STORE_PLAIN, nullptr, zero);
      ntt_any(st, dom, false, T, T, V[v], NTT_LOAD_MUL_TABLE, dom.coset_fwd_ninv, nullptr, nullptr, zero, NTT_STORE_PLAIN, nullptr, zero);
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
    if (me == fin)
      ntt_any(st, dom, true, V[0], T, H, NTT_LOAD_AB_MINUS_C, nullptr, V[1], V[2], dom.z_inv, NTT_STORE_MUL_TABLE, dom.coset_inv, zero);
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
  int msm_host(WS& ws, const uint64_t* bases, const uint64_t* scalars, uint64_t n, uint64_t* out) {
    if (!out || (n && (!bases || !scalars))) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    if (n >= (1ull << 27)) return fail(G16_ERR_BAD_ARGUMENT, "n too large");
    G16_NOT_BUSY();
    G16_CUDA(cudaSetDevice(device));
    XYZZ<F> res = XYZZ<F>::inf();
    if (n) {
      DevBuf db, ds, dm;
      G16_CUDA(db.reserve(n * sizeof(Affine<F>)));
      G16_CUDA(ds.reserve(n * 32));
      G16_CUDA(dm.reserve(n));
      G16_CUDA(cudaMemcpyAsync(db.p, bases, n * sizeof(Affine<F>), cudaMemcpyHostToDevice, S0.st_main));
      G16_CUDA(cudaMemcpyAsync(ds.p, scalars, n * 32, cudaMemcpyHostToDevice, S0.st_main));
      G16_CUDA(msm_prepare_query<F>(S0.st_main, db.template as<Affine<F>>(), (uint32_t)n, 1, 0, dm.template as<uint8_t>()));
      const MsmGeom g = with_k0(msm_geom(n, FR_BITS, cfg_c, 0), sizeof(F) > 48);   // caller-supplied bases: no precomputed copies
      cudaError_t e = msm_enqueue<F, Fr>(S0.st_main, ws, g, db.template as<Affine<F>>(), dm.template as<uint8_t>(), ds.template as<uint32_t>(), 1, false, &ctr, nullptr, nullptr, nullptr, nullptr, nullptr);
      if (e != cudaSuccess) { db.release(); ds.release(); dm.release(); return fail(G16_ERR_CUDA, std::string("msm_enqueue: ") + cudaGetErrorString(e)); }
      e = cudaStreamSynchronize(S0.st_main);
      db.release(); ds.release(); dm.release();
      if (e != cudaSuccess) return fail(G16_ERR_CUDA, std::string("msm sync: ") + cudaGetErrorString(e));
      res = msm_finish<F>(ws, g);
    }
    store_proj<F>(out, res);
    return G16_OK;
  }
  int msm_g1(const uint64_t* bases, const uint64_t* scalars, uint64_t n, uint64_t* out) override { return msm_host<Fq>(S0.ws1[0], bases, scalars, n, out); }
  int msm_g2(const uint64_t* bases, const uint64_t* scalars, uint64_t n, uint64_t* out) override { return msm_host<Fq2>(S0.ws2, bases, scalars, n, out); }

  // ---- circuit ----
  int circuit_load(uint32_t ni, uint32_t nc, uint32_t nw, const g16_csr* a, const g16_csr* b, const g16_csr* c) override {
    if (!a || !b || !c || ni == 0) return fail(G16_ERR_BAD_ARGUMENT, "bad circuit description");
    G16_NOT_BUSY();
    uint64_t need = (uint64_t)nc + ni;
    int Ln = 0;
    while ((1ull << Ln) < need) Ln++;
    int rc = check_log((uint32_t)Ln);
    if (rc) return rc;
    G16_CUDA(cudaSetDevice(device));
    const g16_csr* ms[3] = {a, b, c};
    const uint32_t nvars = ni + nw;
    for (int m = 0; m < 3; m++) {
      if (!ms[m]->row_ptr) return fail(G16_ERR_BAD_ARGUMENT, "null row_ptr");
      if (ms[m]->row_ptr[0] != 0) return fail(G16_ERR_BAD_ARGUMENT, "row_ptr[0] must be 0");
      for (uint32_t i = 0; i < nc; i++)
        if (ms[m]->row_ptr[i + 1] < ms[m]->row_ptr[i]) return fail(G16_ERR_BAD_ARGUMENT, "row_ptr must be non-decreasing");
      const uint32_t nnz = ms[m]->row_ptr[nc];
      if (nnz && (!ms[m]->col || !ms[m]->val)) return fail(G16_ERR_BAD_ARGUMENT, "null col/val");
      for (uint32_t e = 0; e < nnz; e++) if (ms[m]->col[e] >= nvars) return fail(G16_ERR_BAD_ARGUMENT, "column index out of range");
      h_rp[m].assign(ms[m]->row_ptr, ms[m]->row_ptr + nc + 1);
      h_col[m].assign(ms[m]->col, ms[m]->col + nnz);
      h_val[m].resize(nnz);
      if (nnz) memcpy(h_val[m].data(), ms[m]->val, (size_t)nnz * 32);
      G16_CUDA(csr_rp[m].reserve((size_t)(nc + 1) * 4));
      G16_CUDA(csr_col[m].reserve((size_t)nnz * 4 + 4));
      G16_CUDA(csr_val[m].reserve((size_t)nnz * 32 + 32));
      G16_CUDA(cudaMemcpy(csr_rp[m].p, ms[m]->row_ptr, (size_t)(nc + 1) * 4, cudaMemcpyHostToDevice));
      if (nnz) {
        G16_CUDA(cudaMemcpy(csr_col[m].p, ms[m]->col, (size_t)nnz * 4, cudaMemcpyHostToDevice));
        G16_CUDA(cudaMemcpy(csr_val[m].p, ms[m]->val, (size_t)nnz * 32, cudaMemcpyHostToDevice));
      }
    }
    num_inputs = ni; num_constraints = nc; num_witness = nw; L = Ln;
    G16_CUDA(S0.d_z.reserve((size_t)nvars * 32));
    if ((rc = ensure_circuit_domain())) return rc;
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    have_circuit = true;
    have_pk = false;
    return G16_OK;
  }

  // ---- proving key ----
  void shard(Query& x, uint64_t pairs) {
    x.pairs = pairs;
    // Interleaved (strided) split: rank k owns pairs k, k + world, ...  Contiguous ranges would be badly unbalanced
    // whenever the density of a query varies with the variable index (early variables of a circuit are used more often).
    const uint64_t cnt = pairs > rank ? (pairs - rank + world - 1) / world : 0;
    x.lo = rank;
    x.hi = rank + cnt;
    x.geom = with_k0(pick_geom(x.hi - x.lo), &x == &q[M_B2]);
  }
  // sorted entries carry (copy * n + index) in 31 bits and offsets are 32-bit
  bool geom_fits(const Query& x) const {
    return (uint64_t)x.geom.copies * (x.hi - x.lo) < (1ull << 31) && x.geom.max_entries < (1ull << 32);
  }
  template <class F>
  int upload_query(Query& x, const uint64_t* host_full, uint64_t skip_first) {
    using AT = Affine<F>;
    const uint64_t cnt = x.hi - x.lo;
    G16_CUDA(x.bases.reserve((size_t)x.geom.copies * cnt * sizeof(AT) + 16));
    if (cnt) {
      const size_t limbs = sizeof(AT) / 8;
      // gather every world-th point of the full host array
      G16_CUDA(cudaMemcpy2DAsync(x.bases.p, sizeof(AT), host_full + (skip_first + x.lo) * limbs, (size_t)world * sizeof(AT), sizeof(AT), cnt,
                                 cudaMemcpyHostToDevice, S0.st_main));
    }
    return finish_query<F>(x);
  }
  uint64_t nvars() const { return (uint64_t)num_inputs + num_witness; }
  int pk_load(const g16_pk_desc* pk, uint32_t rk, uint32_t wd) override {
    if (!have_circuit) return fail(G16_ERR_BAD_ARGUMENT, "g16_circuit_load must precede g16_pk_load");
    if (!pk || wd == 0 || rk >= wd) return fail(G16_ERR_BAD_ARGUMENT, "bad pk / rank / world");
    G16_NOT_BUSY();
    if (!pk->a_query || !pk->b_g1_query || !pk->b_g2_query || !pk->alpha_g1 || !pk->beta_g1 || !pk->delta_g1 || !pk->beta_g2 || !pk->delta_g2)
      return fail(G16_ERR_BAD_ARGUMENT, "null pk member");
    if (pk->a_len < 1 || pk->b_g1_len < 1 || pk->b_g2_len < 1) return fail(G16_ERR_MALFORMED_KEY, "a/b queries must hold at least the constant-one base");
    if ((pk->h_len && !pk->h_query) || (pk->l_len && !pk->l_query)) return fail(G16_ERR_BAD_ARGUMENT, "null h/l query");
    G16_CUDA(cudaSetDevice(device));
    rank = rk; world = wd;
    const uint64_t n = 1ull << L;
    const uint64_t nz1 = nvars() - 1;  // |input_assignment ++ aux_assignment|, prover.rs:85
    // msm_bigint truncates to the shorter operand (SURVEY.md section 2a; relied upon at prover.rs:66)
    shard(q[M_H], std::min<uint64_t>(pk->h_len, n));
    shard(q[M_L], std::min<uint64_t>(pk->l_len, num_witness));
    shard(q[M_A], std::min<uint64_t>(pk->a_len - 1, nz1));
    shard(q[M_B1], std::min<uint64_t>(pk->b_g1_len - 1, nz1));
    shard(q[M_B2], std::min<uint64_t>(pk->b_g2_len - 1, nz1));
    for (int m = 0; m < 5; m++)
      if (!geom_fits(q[m])) return fail(G16_ERR_BAD_ARGUMENT, "query too large for one GPU: shard it (world > 1) or raise G16_MSM_NE");
    int rc;
    if ((rc = upload_query<Fq>(q[M_H], pk->h_query, 0))) return rc;
    if ((rc = upload_query<Fq>(q[M_L], pk->l_query, 0))) return rc;
    if ((rc = upload_query<Fq>(q[M_A], pk->a_query, 1))) return rc;
    if ((rc = upload_query<Fq>(q[M_B1], pk->b_g1_query, 1))) return rc;
    if ((rc = upload_query<Fq2>(q[M_B2], pk->b_g2_query, 1))) return rc;
    a0 = load_a1(pk->a_query); b1_0 = load_a1(pk->b_g1_query); b2_0 = load_a2(pk->b_g2_query);
    alpha_g1 = load_a1(pk->alpha_g1); beta_g1 = load_a1(pk->beta_g1); delta_g1 = load_a1(pk->delta_g1);
    beta_g2 = load_a2(pk->beta_g2); delta_g2 = load_a2(pk->delta_g2);
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    have_pk = true;
    from_setup = false;
    if ((rc = decide_b_sort_sharing())) return rc;
    decide_ba_memory();
    return G16_OK;
  }

  // ---- setup (generator.rs:47-208) ----
  template <class F>
  int batch_mul(const Affine<F>& gen, const Fr* d_scalars, uint64_t cnt, Affine<F>* d_out, DevBuf& table) {
    G16_CUDA(table.reserve((size_t)FB_WINDOWS * 255 * sizeof(XYZZ<F>)));
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
    std::vector<Fr> gabc(ni), lq(num_witness), hs(n - 1);
    for (uint64_t i = 0; i < nv; i++) {
      const Fr t = Fr::add(Fr::add(Fr::mul(beta, qa[i]), Fr::mul(alpha, qb[i])), qc[i]);
      if (i < ni) gabc[i] = Fr::mul(t, gi);                                        // generator.rs:113-117
      else lq[i - ni] = Fr::mul(t, di);                                            // generator.rs:119-123
    }
    {
      Fr p = Fr::mul(zt, di);                                                      // h_query_scalars, r1cs_to_qap.rs:237-247
      for (uint64_t i = 0; i + 1 < n; i++) { hs[i] = p; p = Fr::mul(p, tau); }
    }
    // --- fixed-base batch multiplications on the GPU (generator.rs:129-183) ---
    rank = 0; world = 1;
    DevBuf d_s, tab1, tab2;
    const uint64_t maxs = std::max<uint64_t>(nv, n);
    G16_CUDA(d_s.reserve(maxs * 32));
    int rc;
    auto up = [&](const std::vector<Fr>& v) -> cudaError_t {
      return v.empty() ? cudaSuccess : cudaMemcpyAsync(d_s.p, v.data(), v.size() * 32, cudaMemcpyHostToDevice, S0.st_main);
    };
    G16_CUDA(full_a.reserve(nv * sizeof(A1))); G16_CUDA(full_b1.reserve(nv * sizeof(A1))); G16_CUDA(full_b2.reserve(nv * sizeof(A2)));
    G16_CUDA(d_gamma_abc.reserve((size_t)ni * sizeof(A1)));
    shard(q[M_H], n - 1); shard(q[M_L], num_witness); shard(q[M_A], nv - 1); shard(q[M_B1], nv - 1); shard(q[M_B2], nv - 1);
    G16_CUDA(q[M_H].bases.reserve((size_t)q[M_H].geom.copies * (n - 1) * sizeof(A1) + 16));
    G16_CUDA(q[M_L].bases.reserve((size_t)q[M_L].geom.copies * num_witness * sizeof(A1) + 16));
    // a_query / b_g1_query / b_g2_query
    G16_CUDA(up(qa)); if ((rc = batch_mul<Fq>(g1, d_s.template as<Fr>(), nv, full_a.template as<A1>(), tab1))) return rc;
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    G16_CUDA(up(qb)); if ((rc = batch_mul<Fq>(g1, d_s.template as<Fr>(), nv, full_b1.template as<A1>(), tab1))) return rc;
    if ((rc = batch_mul<Fq2>(g2, d_s.template as<Fr>(), nv, full_b2.template as<A2>(), tab2))) return rc;
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    G16_CUDA(up(hs)); if ((rc = batch_mul<Fq>(g1, d_s.template as<Fr>(), n - 1, q[M_H].bases.template as<A1>(), tab1))) return rc;
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    G16_CUDA(up(lq)); if ((rc = batch_mul<Fq>(g1, d_s.template as<Fr>(), num_witness, q[M_L].bases.template as<A1>(), tab1))) return rc;
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    G16_CUDA(up(gabc)); if ((rc = batch_mul<Fq>(g1, d_s.template as<Fr>(), ni, d_gamma_abc.template as<A1>(), tab1))) return rc;
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    // MSM views: query[1..]
    auto view = [&](Query& x, DevBuf& full, size_t esz) -> int {
      G16_CUDA(x.bases.reserve((size_t)x.geom.copies * (nv - 1) * esz + 16));
      if (nv > 1) G16_CUDA(cudaMemcpyAsync(x.bases.p, (char*)full.p + esz, (nv - 1) * esz, cudaMemcpyDeviceToDevice, S0.st_main));
      return G16_OK;
    };
    if ((rc = view(q[M_A], full_a, sizeof(A1)))) return rc;
    if ((rc = view(q[M_B1], full_b1, sizeof(A1)))) return rc;
    if ((rc = view(q[M_B2], full_b2, sizeof(A2)))) return rc;
    for (int m = 0; m < 5; m++) {
      if ((rc = (m == M_B2) ? finish_query<Fq2>(q[m]) : finish_query<Fq>(q[m]))) return rc;
    }
    G16_CUDA(cudaMemcpyAsync(&a0, full_a.p, sizeof(A1), cudaMemcpyDeviceToHost, S0.st_main));
    G16_CUDA(cudaMemcpyAsync(&b1_0, full_b1.p, sizeof(A1), cudaMemcpyDeviceToHost, S0.st_main));
    G16_CUDA(cudaMemcpyAsync(&b2_0, full_b2.p, sizeof(A2), cudaMemcpyDeviceToHost, S0.st_main));
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    // single points on the host (generator.rs:147-151,182)
    uint32_t k[8];
    auto mul1 = [&](const Fr& s) { fr_to_canon(s, k); return P1::from_affine(g1).mul_u32(k, 8).to_affine(); };
    auto mul2 = [&](const Fr& s) { fr_to_canon(s, k); return P2::from_affine(g2).mul_u32(k, 8).to_affine(); };
    alpha_g1 = mul1(alpha); beta_g1 = mul1(beta); delta_g1 = mul1(delta);
    beta_g2 = mul2(beta); gamma_g2 = mul2(gamma); delta_g2 = mul2(delta);
    d_s.release(); tab1.release(); tab2.release();
    have_pk = true;
    from_setup = true;
    if ((rc = decide_b_sort_sharing())) return rc;
    decide_ba_memory();
    return G16_OK;
  }
  int pk_export(const g16_pk_export_desc* o) override {
    if (!have_pk || !from_setup) return fail(G16_ERR_BAD_ARGUMENT, "g16_pk_export needs a key produced by g16_setup");
    if (!o) return fail(G16_ERR_BAD_ARGUMENT, "null");
    G16_CUDA(cudaSetDevice(device));
    const uint64_t nv = nvars(), n = 1ull << L;
    if (o->a_query) G16_CUDA(cudaMemcpy(o->a_query, full_a.p, nv * sizeof(A1), cudaMemcpyDeviceToHost));
    if (o->b_g1_query) G16_CUDA(cudaMemcpy(o->b_g1_query, full_b1.p, nv * sizeof(A1), cudaMemcpyDeviceToHost));
    if (o->b_g2_query) G16_CUDA(cudaMemcpy(o->b_g2_query, full_b2.p, nv * sizeof(A2), cudaMemcpyDeviceToHost));
    if (o->h_query && n > 1) G16_CUDA(cudaMemcpy(o->h_query, q[M_H].bases.p, (n - 1) * sizeof(A1), cudaMemcpyDeviceToHost));
    if (o->l_query && num_witness) G16_CUDA(cudaMemcpy(o->l_query, q[M_L].bases.p, (size_t)num_witness * sizeof(A1), cudaMemcpyDeviceToHost));
    if (o->gamma_abc_g1) G16_CUDA(cudaMemcpy(o->gamma_abc_g1, d_gamma_abc.p, (size_t)num_inputs * sizeof(A1), cudaMemcpyDeviceToHost));
    if (o->alpha_g1) store_a1(o->alpha_g1, alpha_g1);
    if (o->beta_g1) store_a1(o->beta_g1, beta_g1);
    if (o->delta_g1) store_a1(o->delta_g1, delta_g1);
    if (o->beta_g2) store_a2(o->beta_g2, beta_g2);
    if (o->gamma_g2) store_a2(o->gamma_g2, gamma_g2);
    if (o->delta_g2) store_a2(o->delta_g2, delta_g2);
    return G16_OK;
  }

  // ---- proving ----
  // enqueue on sl.st_main: upload z, row evaluation, witness map
  int enqueue_witness_map(Slot& sl, const uint64_t* z, uint32_t flags) {
    const uint64_t nv = nvars();
    int rc = ensure_circuit_domain();   // no-op unless something rebuilt `dom` for another size
    if (rc) return rc;
    if ((rc = ensure_slot_buffers(sl, L))) return rc;
    G16_CUDA(sl.d_z.reserve((size_t)nv * 32));
    sl.tm.h2d_bytes = 0;
    G16_CUDA(cudaEventRecord(sl.ev_start, sl.st_main));
    if (flags & G16_ASSIGNMENT_ON_DEVICE) {
      G16_CUDA(cudaMemcpyAsync(sl.d_z.p, z, nv * 32, cudaMemcpyDeviceToDevice, sl.st_main));
    } else {
      G16_CUDA(cudaMemcpyAsync(sl.d_z.p, z, nv * 32, cudaMemcpyHostToDevice, sl.st_main));
      sl.tm.h2d_bytes = nv * 32;
    }
    G16_CUDA(cudaEventRecord(sl.ev_z, sl.st_main));
    const uint32_t n = 1u << L;
    CsrDev cs[3];
    for (int m = 0; m < 3; m++) cs[m] = CsrDev{csr_rp[m].template as<uint32_t>(), csr_col[m].template as<uint32_t>(), csr_val[m].p};
    r1cs_matvec<Fr>(sl.st_main, cs, sl.d_z.template as<Fr>(), num_constraints, num_inputs, n, sl.d_a.template as<Fr>(),
                    sl.d_b.template as<Fr>(), sl.d_c.template as<Fr>());
    ntt_launches++;
    if (sl.split_wm && nccl_comm_wm) {
      if ((rc = witness_map_split(sl))) return rc;
    } else {
      witness_map_device(sl, dom);
    }
    G16_CUDA(cudaGetLastError());
    G16_CUDA(cudaEventRecord(sl.ev_h, sl.st_main));
    return G16_OK;
  }
  int witness_map(const uint64_t* z, uint32_t flags, uint64_t* h) override {
    if (!have_circuit) return fail(G16_ERR_BAD_ARGUMENT, "no circuit resident");
    if (!z || !h) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    if (S0.busy) return fail(G16_ERR_BAD_ARGUMENT, "slot 0 has a proof in flight");
    G16_CUDA(cudaSetDevice(device));
    int rc = enqueue_witness_map(S0, z, flags);
    if (rc) return rc;
    G16_CUDA(cudaMemcpyAsync(h, S0.d_h.p, (size_t)32 << L, cudaMemcpyDeviceToHost, S0.st_main));
    G16_CUDA(cudaStreamSynchronize(S0.st_main));
    return G16_OK;
  }

  // Asynchronous half of a proof: everything is enqueued on the slot's streams, nothing is waited for.
  // s may be null (partial proof: the (r, s)-only scalar multiplications are skipped).
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
    const bool r_zero = sl.r.is_zero();
    if (sl.have_s) {
      if (sl.helper) sl.helper->wait();
      if (sl.helper2) sl.helper2->wait();
      sl.helper = pool->submit([this, &sl]() { fixed_muls_a(sl.r, sl.s, sl.fx); });
      sl.helper2 = pool->submit([this, &sl]() { fixed_muls_b(sl.r, sl.s, sl.fx); });
    }
    int rc;
    {
      NvtxSpan span_wm(SPAN_WITNESS_MAP);
      rc = enqueue_witness_map(sl, z, flags);
    }
    if (rc) return rc;
    const uint32_t* zs = sl.d_z.template as<uint32_t>();
    const uint32_t* hs = sl.d_h.template as<uint32_t>();
    // scalar sources (prover.rs:63-85): H <- h ; L <- aux ; A, B1, B2 <- input[1..] ++ aux
    const uint32_t* src[5] = {hs, zs + (size_t)num_inputs * 8, zs + 8, zs + 8, zs + 8};
    for (int m = 0; m < 5; m++) {
      const uint64_t cnt = q[m].hi - q[m].lo;
      sl.geom[m] = q[m].geom;
      sl.run[m] = cnt > 0 && !(m == M_B1 && r_zero);                     // prover.rs:98: B in G1 skipped when r == 0
      sl.tm.msm_pairs[m] = sl.run[m] ? cnt : 0;
    }
    const int order[5] = {M_L, M_A, M_B2, M_B1, M_H};                    // H last: it waits for the witness map; B2 (higher
                                                                         // stream priority) sorts, B1 borrows its sorted list
    for (int oi = 0; oi < 5; oi++) {
      const int m = order[oi];
      NvtxSpan span_msm(span_of(m));
      cudaStream_t st = sl.serial ? sl.st_main : sl.st_msm[m];
      if (!sl.serial) G16_CUDA(cudaStreamWaitEvent(st, m == M_H ? sl.ev_h : sl.ev_z, 0));
      G16_CUDA(cudaEventRecord(sl.ev_m0[m], st));
      if (sl.run[m]) {
        const uint32_t* sc = src[m] + q[m].lo * 8;   // first owned scalar; the digit kernel strides by `world`
        cudaError_t e;
        // B in G1 and B in G2 run over the same scalars and identity pattern: one counting sort serves both.  B2 sorts
        // (its stream has the higher priority and its tail is the longest), B1 borrows the list.
        const bool share = share_b_sort && sl.run[M_B1] && sl.run[M_B2];
        // "witness map first" (option, off by default): the MSMs that do not need h sort their entries at once but start
        // accumulating only when the witness map is done, so that their register-heavy blocks do not slow the NTT kernels.
        const bool wm_first = !sl.serial && (wm_first_opt > 0 || (wm_first_opt < 0 && world > 1));
        cudaEvent_t gate = (wm_first && m != M_H) ? sl.ev_h : nullptr;
        if (m == M_B2 && share) { sl.b_sorted = MsmSorted{}; sl.b_sorted.ready = sl.ev_bsort; }
        if (m == M_B2) e = msm_enqueue<Fq2, Fr>(st, sl.ws2, sl.geom[m], q[m].bases.template as<A2>(), q[m].mask.template as<uint8_t>(), sc, world, true, &ctr, sl.ev_a0[m], sl.ev_a1[m], share ? &sl.b_sorted : nullptr, nullptr, gate);
        else e = msm_enqueue<Fq, Fr>(st, sl.ws1[m], sl.geom[m], q[m].bases.template as<A1>(), q[m].mask.template as<uint8_t>(), sc, world, true, &ctr, sl.ev_a0[m], sl.ev_a1[m], nullptr, (m == M_B1 && share) ? &sl.b_sorted : nullptr, gate);
        if (e != cudaSuccess) return fail(G16_ERR_CUDA, std::string("msm_enqueue: ") + cudaGetErrorString(e));
      }
      G16_CUDA(cudaEventRecord(sl.ev_m1[m], st));
    }
    sl.launches0 = ctr.launches + ntt_launches - sl.launches0;   // kernels launched for this proof
    sl.busy = true;
    return G16_OK;
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
            uint32_t k[8];
            fr_to_canon(m == M_A ? sl.s : sl.r, k);
            if (m == M_A) out.sa = out.a.mul_u32(k, 8);
            else out.rb1 = out.b1.mul_u32(k, 8);
          }
        });
      }
      for (auto& t : tk) t->wait();
      out.scaled = sl.have_s;
      for (int m = 0; m < 5; m++)
        if (errs[m] != cudaSuccess) return fail(G16_ERR_CUDA, std::string("msm stream sync: ") + cudaGetErrorString(errs[m]));
      G16_CUDA(cudaStreamSynchronize(sl.st_main));
    }
    sl.tm.host_finish_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    // timings
    float ms = 0, tot = 0;
    cudaEventElapsedTime(&sl.tm.h2d_ms, sl.ev_start, sl.ev_z);
    cudaEventElapsedTime(&sl.tm.witness_map_ms, sl.ev_z, sl.ev_h);
    cudaEventElapsedTime(&tot, sl.ev_start, sl.ev_h);
    for (int m = 0; m < 5; m++) {
      cudaEventElapsedTime(&sl.tm.msm_ms[m], sl.ev_m0[m], sl.ev_m1[m]);
      sl.tm.msm_accum_ms[m] = 0;
      sl.tm.msm_entries[m] = 0;
      if (sl.run[m]) {
        cudaEventElapsedTime(&sl.tm.msm_accum_ms[m], sl.ev_a0[m], sl.ev_a1[m]);
        sl.tm.msm_entries[m] = m == M_B2 ? *sl.ws2.h_total : *sl.ws1[m].h_total;
      }
      cudaEventElapsedTime(&sl.tm.msm_begin_ms[m], sl.ev_start, sl.ev_m0[m]);
      cudaEventElapsedTime(&ms, sl.ev_start, sl.ev_m1[m]);
      sl.tm.msm_end_ms[m] = ms;
      if (ms > tot) tot = ms;
    }
    sl.tm.total_ms = tot;
    sl.tm.launches = sl.launches0;
    sl.tm.d2h_bytes = 0;
    for (int m = 0; m < 5; m++)
      if (sl.run[m]) sl.tm.d2h_bytes += (m == M_B2 ? sl.ws2.plan.leaf_pts * sizeof(P2) : sl.ws1[m].plan.leaf_pts * sizeof(P1)) * sl.geom[m].ne;
    tm = sl.tm;
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
    if ((rc = wait_partials(S0, x))) return rc;
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
    if (rc) return rc;
    store_partials(partial, x);
    return G16_OK;
  }
  // prover.rs:76-131 on the host, regrouped so that nothing heavy is left once the last MSM is done: with
  //   A, B1, B2, L, H the five MSM results,
  //   g_a  = (r d1 + a0 + alpha1) + A                                   = ga0 + A
  //   g2_b = (s d2 + b2_0 + beta2) + B2                                 = gb2_0 + B2
  //   g_c  = s g_a + r g1_b - rs d1 + L + H                             = s_ga0 + s A + r_gb0 + r B1 + neg_rs_d1 + L + H
  // (scalar multiplication distributes over the group law, so the affine proof is the reference's bit for bit).
  // fixed_muls_a / _b: six scalar multiplications that need only (r, s, key), on two pool threads during the GPU work.
  void fixed_muls_a(const Fr& r, const Fr& s, FixedMuls& f) const {
    uint32_t rk[8], sk[8], rsk[8];
    fr_to_canon(r, rk);
    fr_to_canon(s, sk);
    fr_to_canon(Fr::mul(r, s), rsk);
    const P1 d1 = P1::from_affine(delta_g1);
    f.neg_rs_d1 = d1.mul_u32(rsk, 8);                      // prover.rs:76
    f.neg_rs_d1.negate();
    f.ga0 = d1.mul_u32(rk, 8);                             // prover.rs:90
    f.ga0.madd(a0);
    f.ga0.madd(alpha_g1);
    f.s_ga0 = f.ga0.mul_u32(sk, 8);                        // prover.rs:94 (its key-only part)
  }
  void fixed_muls_b(const Fr& r, const Fr& s, FixedMuls& f) const {
    uint32_t rk[8], sk[8];
    fr_to_canon(r, rk);
    fr_to_canon(s, sk);
    f.r_gb0 = P1::inf();
    if (!r.is_zero()) {                                    // prover.rs:98-108
      P1 gb0 = P1::from_affine(delta_g1).mul_u32(sk, 8);   // prover.rs:100
      gb0.madd(b1_0);
      gb0.madd(beta_g1);
      f.r_gb0 = gb0.mul_u32(rk, 8);                        // prover.rs:114 (its key-only part)
    }
    f.gb2_0 = P2::from_affine(delta_g2).mul_u32(sk, 8);    // prover.rs:112
    f.gb2_0.madd(b2_0);
    f.gb2_0.madd(beta_g2);
  }
  FixedMuls fixed_muls(const Fr& r, const Fr& s) const {
    FixedMuls f;
    fixed_muls_a(r, s, f);
    fixed_muls_b(r, s, f);
    return f;
  }
  // a_sum, b2_sum: A and B2 MSM results (summed over the ranks); c_sum = s A + r B1 + L + H (summed over the ranks)
  int assemble_sums(const P1& a_sum, const P2& b2_sum, const P1& c_sum, const FixedMuls& f, uint64_t* proof) {
    NvtxSpan span_finish(SPAN_FINISH_C);
    P1 g_a = f.ga0;                                       // prover.rs:90-92,252-270
    g_a.add(a_sum);
    P2 g2_b = f.gb2_0;                                    // prover.rs:112-113
    g2_b.add(b2_sum);
    P1 g_c = f.s_ga0;                                     // prover.rs:119-124
    g_c.add(f.r_gb0);
    g_c.add(f.neg_rs_d1);
    g_c.add(c_sum);
    store_a1(proof, g_a.to_affine());                     // prover.rs:127-131
    store_a2(proof + 2 * NQ64, g2_b.to_affine());
    store_a1(proof + 6 * NQ64, g_c.to_affine());
    return G16_OK;
  }
  // this rank's contribution to g_c that depends on its MSM results: s A + r B1 + L + H
  P1 c_part(const Fr& r, const Fr& s, const Partials& x) const {
    uint32_t k[8];
    P1 c = x.scaled ? x.sa : (fr_to_canon(s, k), x.a.mul_u32(k, 8));
    if (!r.is_zero()) c.add(x.scaled ? x.rb1 : (fr_to_canon(r, k), x.b1.mul_u32(k, 8)));
    c.add(x.l);
    c.add(x.h);
    return c;
  }
  int assemble(const Fr& r, const Fr& s, const Partials& x, const FixedMuls& f, uint64_t* proof) {
    return assemble_sums(x.a, x.b2, c_part(r, s, x), f, proof);
  }
  int prove_submit(int slot, const uint64_t* r, const uint64_t* s, const uint64_t* z, uint32_t flags) override {
    if (slot < 0 || slot >= NSLOTS) return fail(G16_ERR_BAD_ARGUMENT, "bad slot");
    if (!s) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    if (world != 1) return fail(G16_ERR_BAD_ARGUMENT, "key is sharded: use g16_prove_partial + g16_prove_assemble");
    return submit(slots[slot], r, s, z, flags);
  }
  int prove_wait(int slot, uint64_t* proof) override {
    if (slot < 0 || slot >= NSLOTS || !proof) return fail(G16_ERR_BAD_ARGUMENT, "bad slot / null buffer");
    Slot& sl = slots[slot];
    Partials x;
    int rc = wait_partials(sl, x);
    if (sl.helper) { sl.helper->wait(); sl.helper.reset(); }
    if (sl.helper2) { sl.helper2->wait(); sl.helper2.reset(); }
    if (rc) return rc;
    if (!sl.have_s) return fail(G16_ERR_BAD_ARGUMENT, "slot holds a partial proof (use g16_prove_partial_wait)");
    auto t0 = std::chrono::steady_clock::now();
    rc = assemble(sl.r, sl.s, x, sl.fx, proof);
    sl.tm.host_finish_ms += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    sl.tm.d2h_bytes += 8 * NQ64 * 8;
    tm = sl.tm;
    return rc;
  }
  int prove(const uint64_t* r, const uint64_t* s, const uint64_t* z, uint32_t flags, uint64_t* proof) override {
    if (!proof) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    int rc = prove_submit(0, r, s, z, flags);
    if (rc) return rc;
    return prove_wait(0, proof);
  }
  // ---- sharded proof with the exchange inside the library (g16_comm_init + g16_prove_sharded*) ----
  // Every rank holds pair i of every MSM with i mod world == rank.  Per proof a rank contributes THREE points:
  //   A_k (its share of the A MSM), B2_k (its share of B in G2) and C_k = s A_k + r B1_k + L_k + H_k,
  // in XYZZ coordinates (no inversion on the exchange path): 2 * 4 * Fq + 4 * Fq2 limbs = 768 B on BLS12-381.  One
  // ncclAllGather of that record on a dedicated high-priority stream, then every rank adds the records in rank order and
  // finishes the same proof (EC addition is exactly associative and commutative: bit-identical for any world size).
  void* nccl_comm = nullptr;      // all-gather of the partial proof points (stream st_comm)
  void* nccl_comm_wm = nullptr;   // witness-map exchange (send / recv / broadcast on the proof slot's main stream)
  bool split_wm_wanted = true;    // g16_set_option "wm_split"
  uint32_t comm_rank = 0, comm_world = 0;
  cudaStream_t st_comm = nullptr;
  DevBuf d_comm_send, d_comm_recv;
  uint64_t* h_comm_send = nullptr;   // pinned
  uint64_t* h_comm_recv = nullptr;   // pinned, world records
  static constexpr size_t REC_LIMBS = 2 * 4 * (size_t)NQ64 + 4 * 2 * (size_t)NQ64;   // A_k, C_k (XYZZ G1), B2_k (XYZZ G2)
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
    slots[slot].split_wm = split_wm_wanted && comm_world > 1;
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
    int rc = wait_partials(sl, x);
    if (sl.helper) { sl.helper->wait(); sl.helper.reset(); }
    if (sl.helper2) { sl.helper2->wait(); sl.helper2.reset(); }
    if (rc) return rc;
    if (!sl.have_s) return fail(G16_ERR_BAD_ARGUMENT, "slot holds a partial proof");
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
    rc = assemble_sums(a_sum, b2_sum, c_sum, sl.fx, proof);
    sl.tm.host_finish_ms += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    sl.tm.d2h_bytes += REC_LIMBS * 8 * comm_world;
    tm = sl.tm;
    return rc;
  }

  // Sharded path: the (r, s)-only scalar multiplications can be started before the partial sums exist
  // (g16_prove_assemble_prepare), so that they overlap the GPU work and the gather; prove_assemble picks them up.
  Fr asm_r, asm_s;
  FixedMuls asm_fx;
  bool asm_valid = false;
  std::shared_ptr<HostPool::Ticket> asm_helper;
  int assemble_prepare(const uint64_t* r, const uint64_t* s) override {
    if (!have_pk) return fail(G16_ERR_BAD_ARGUMENT, "no proving key resident");
    if (!r || !s) return fail(G16_ERR_BAD_ARGUMENT, "null buffer");
    if (asm_helper) asm_helper->wait();
    asm_r = load_fr(r);
    asm_s = load_fr(s);
    asm_valid = true;
    asm_helper = pool->submit([this]() { asm_fx = fixed_muls(asm_r, asm_s); });
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
    if (asm_valid && rr == asm_r && ss == asm_s) {
      asm_valid = false;
      return assemble(rr, ss, x, asm_fx, proof);
    }
    return assemble(rr, ss, x, fixed_muls(rr, ss), proof);
  }
};

// extern-template declarations for one curve: put before make_engine<CP> is instantiated (engine_<curve>.cu)
#define G16_CURVE_KERNELS(X, CP)                                                                  \
  G16_NTT_TEMPLATES(X, Fp<CP::FrP>)                                                               \
  G16_NTT2_TEMPLATES(X, Fp<CP::FrP>)                                                              \
  G16_MSM_TEMPLATES(X, Fp<CP::FqP>, Fp<CP::FrP>)                                                  \
  G16_MSM_TEMPLATES(X, G16_FQ2(CP), Fp<CP::FrP>)
#define G16_FQ2(CP) Fp2<CP::FqP, CP::FQ2_NONRESIDUE_NEG>

template <class CP>
IEngine* make_engine(int device, int* rc) {
  auto* e = new Engine<CP>();
  *rc = e->init(device);
  if (*rc) { delete e; return nullptr; }
  return e;
}

}  // namespace g16
