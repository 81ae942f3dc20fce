/* g16b200.h -- C ABI of libg16b200.so: the H100-native Groth16 proving hot path (NTT witness map + five MSMs).
 *
 * Drop-in boundary for ark-groth16 0.5.0 (/root/reference).  Every entry point names the reference interface it
 * replaces; INTEGRATION.md shows the Rust `extern "C"` binding a maintainer would add.
 *
 * Data layout (SURVEY.md section 8b), identical to ark-ff / ark-ec in-memory values copied field-wise:
 *   Fr / Fq element : N64 little-endian uint64_t limbs in MONTGOMERY form (R = 2^(64*N64)); N64 = 4 for every Fr,
 *                     4 for BN254 Fq, 6 for BLS12-381 / BLS12-377 Fq.
 *   BigInt scalar   : 4 little-endian uint64_t limbs, canonical integer < r  (`PrimeField::into_bigint`).
 *   G1 affine       : x || y                      (2*N64 limbs);  point at infinity = all-zero limbs.
 *   G2 affine       : x.c0 || x.c1 || y.c0 || y.c1 (4*N64 limbs); point at infinity = all-zero limbs.
 *   G1/G2 projective output : X || Y || Z Jacobian, normalised to Z = 1 (identity: X = Y = 1, Z = 0, as ark).
 * All functions return G16_OK (0) or an error code; they never unwind or abort across the ABI
 * (the reference builds with panic = 'abort' for FFI safety, Cargo.toml:61).  A context is used by one host
 * thread at a time; use one context per GPU / per concurrent proof.
 */
#ifndef G16B200_H
#define G16B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
  G16_CURVE_BLS12_381 = 0,
  G16_CURVE_BN254 = 1,
  G16_CURVE_BLS12_377 = 2
};

enum {
  G16_OK = 0,
  G16_ERR_POLYNOMIAL_DEGREE_TOO_LARGE = 1, /* SynthesisError::PolynomialDegreeTooLarge, r1cs_to_qap.rs:134,179 */
  G16_ERR_BAD_ARGUMENT = 2,                /* null pointer / inconsistent length / unknown curve               */
  G16_ERR_CUDA = 3,                        /* CUDA failure or no usable sm_90 device; see g16_last_error()     */
  G16_ERR_MALFORMED_KEY = 4                /* SynthesisError::MalformedVerifyingKey-class length mismatch      */
};

typedef struct g16_ctx g16_ctx;

/* Flags for g16_prove* (bitwise or) */
enum {
  G16_ASSIGNMENT_ON_DEVICE = 1, /* `full_assignment` is a device pointer (bench.py's resident-input measurement) */
  G16_SERIAL_MSMS = 2           /* run the five MSMs one after another on one stream (kernel-level profiling)    */
};

/* ---- context ----------------------------------------------------------------------------------------------- */
/* One context = one curve on one CUDA device.  Fails with G16_ERR_CUDA when no GPU is present: there is no CPU
 * fallback anywhere in this library. */
int g16_ctx_create(int curve, int device, g16_ctx** out);
void g16_ctx_destroy(g16_ctx* ctx);
const char* g16_last_error(void);
/* sizes, in uint64_t limbs, for buffers of this context's curve */
int g16_fq_limbs(const g16_ctx* ctx);

/* ---- NTT: ark-poly Radix2EvaluationDomain (un-vendored dependency), call sites r1cs_to_qap.rs:201-207,220-221,232
 * In-place transform of 2^log_n Montgomery Fr elements in host memory, natural order in and out.
 *   inverse = 0, coset = 0 : domain.fft_in_place            inverse = 1, coset = 0 : domain.ifft_in_place
 *   inverse = 0, coset = 1 : domain.get_coset(F::GENERATOR).fft_in_place       inverse = 1, coset = 1 : ...ifft_in_place
 * log_n above the field's two-adicity -> G16_ERR_POLYNOMIAL_DEGREE_TOO_LARGE (D::new returning None). */
int g16_ntt(g16_ctx* ctx, uint32_t log_n, int inverse, int coset, uint64_t* inout);

/* ---- witness map from evaluation vectors: r1cs_to_qap.rs:201-234 (everything after the row evaluations).
 * a, b, c: 2^log_n Montgomery Fr each (host).  h_out: 2^log_n coefficients of h(X) (host). */
int g16_witness_map_evals(g16_ctx* ctx, uint32_t log_n, const uint64_t* a, const uint64_t* b, const uint64_t* c,
                          uint64_t* h_out);

/* ---- variable-base MSM: ark-ec VariableBaseMSM::msm_bigint, call sites prover.rs:66,74,262.
 * bases: n affine points (host); scalars: n BigInt<4> (host); result: projective (see layout).  As in ark,
 * the caller passes min(bases.len(), scalars.len()) as n. */
int g16_msm_g1(g16_ctx* ctx, const uint64_t* bases, const uint64_t* scalars, uint64_t n, uint64_t* out_xyz);
int g16_msm_g2(g16_ctx* ctx, const uint64_t* bases, const uint64_t* scalars, uint64_t n, uint64_t* out_xyz);

/* ---- constraint matrices: ark-relations ConstraintMatrices as consumed by
 * R1CSToQAP::witness_map_from_matrices (r1cs_to_qap.rs:172-199,213-218).  CSR per matrix: row_ptr has
 * num_constraints+1 entries, col[e] indexes the full assignment (instance first), val[e] is Montgomery Fr.
 * Uploaded once per circuit and kept resident. */
typedef struct {
  const uint32_t* row_ptr;
  const uint32_t* col;
  const uint64_t* val;
} g16_csr;
int g16_circuit_load(g16_ctx* ctx, uint32_t num_inputs /* instance variables incl. the constant One */,
                     uint32_t num_constraints, uint32_t num_witness, const g16_csr* a, const g16_csr* b,
                     const g16_csr* c);

/* ---- proving key: data_structures.rs:126-143.  Query arrays are the FULL ark vectors (a_query[0] included).
 * With world > 1 the context keeps only the index range of every query owned by `rank` (SURVEY.md section 8e):
 * round-robin split of each MSM's (base, scalar) pairs: pair i belongs to rank i mod world. */
typedef struct {
  const uint64_t* a_query;    uint64_t a_len;     /* G1, num_inputs + num_witness      (generator.rs:155) */
  const uint64_t* b_g1_query; uint64_t b_g1_len;  /* G1, same length                   (generator.rs:161) */
  const uint64_t* b_g2_query; uint64_t b_g2_len;  /* G2, same length                   (generator.rs:134) */
  const uint64_t* h_query;    uint64_t h_len;     /* G1, domain_size - 1               (generator.rs:168) */
  const uint64_t* l_query;    uint64_t l_len;     /* G1, num_witness                   (generator.rs:174) */
  const uint64_t* alpha_g1;   /* vk.alpha_g1 */
  const uint64_t* beta_g1;
  const uint64_t* delta_g1;
  const uint64_t* beta_g2;    /* vk.beta_g2  */
  const uint64_t* delta_g2;   /* vk.delta_g2 */
} g16_pk_desc;
int g16_pk_load(g16_ctx* ctx, const g16_pk_desc* pk, uint32_t rank, uint32_t world);

/* ---- trusted setup with explicit toxic waste: Groth16::generate_parameters_with_qap, generator.rs:47-208
 * (the fixed-base batch multiplications of generator.rs:129-183 run on the GPU).  Needs g16_circuit_load first.
 * alpha..tau are Montgomery Fr; g1/g2 are the affine group generators.  The resulting proving key becomes the
 * context's resident key (as after g16_pk_load with rank 0 / world 1); g16_pk_export copies it to the host. */
int g16_setup(g16_ctx* ctx, const uint64_t* alpha, const uint64_t* beta, const uint64_t* gamma,
              const uint64_t* delta, const uint64_t* tau, const uint64_t* g1, const uint64_t* g2);
typedef struct {
  uint64_t* a_query;    /* capacity (num_inputs + num_witness) G1 */
  uint64_t* b_g1_query;
  uint64_t* b_g2_query;
  uint64_t* h_query;    /* capacity domain_size - 1 */
  uint64_t* l_query;    /* capacity num_witness */
  uint64_t* alpha_g1; uint64_t* beta_g1; uint64_t* delta_g1;
  uint64_t* beta_g2; uint64_t* gamma_g2; uint64_t* delta_g2;
  uint64_t* gamma_abc_g1; /* capacity num_inputs G1 */
} g16_pk_export_desc;
int g16_pk_export(g16_ctx* ctx, const g16_pk_export_desc* out);

/* ---- proving: Groth16::create_proof_with_reduction_and_matrices, prover.rs:26-51
 *      = witness_map_from_matrices (r1cs_to_qap.rs:172-235) + create_proof_with_assignment (prover.rs:54-132).
 * r, s: Montgomery Fr.  full_assignment: (num_inputs + num_witness) Montgomery Fr, instance first.
 * proof_out: a (G1 affine) || b (G2 affine) || c (G1 affine) = 8*N64 limbs.  Needs circuit + key resident. */
int g16_prove(g16_ctx* ctx, const uint64_t* r, const uint64_t* s, const uint64_t* full_assignment, uint32_t flags,
              uint64_t* proof_out);

/* Sharded proving (world > 1): every rank computes its partial MSM sums, the host plumbing (torch.distributed /
 * NCCL all_gather of 5 points per rank) exchanges them, every rank assembles the same proof.
 * partial_out / partials: [h, l, a, b_g1] as G1 affine (4 * 2*N64 limbs) followed by b_g2 as G2 affine (4*N64). */
int g16_prove_partial(g16_ctx* ctx, const uint64_t* r, const uint64_t* full_assignment, uint32_t flags,
                      uint64_t* partial_out);
int g16_prove_assemble(g16_ctx* ctx, const uint64_t* r, const uint64_t* s, const uint64_t* partials,
                       uint32_t nparts, uint64_t* proof_out);
/* Optional: start the (r, s)-only scalar multiplications of prover.rs:76,90,100,112 on a helper thread before the partial
 * sums exist; the next g16_prove_assemble with the same (r, s) picks the result up instead of computing it inline. */
int g16_prove_assemble_prepare(g16_ctx* ctx, const uint64_t* r, const uint64_t* s);
/* Pipelined proving: a context owns two proof slots (0 and 1), each with its own streams and work buffers.
 * g16_prove_submit enqueues a whole proof asynchronously and returns; g16_prove_wait blocks until that slot's GPU
 * work is done, finishes on the host and writes the proof.  Submitting proof i+1 before waiting for proof i lets
 * the latency-bound tail of one proof overlap the bulk of the next (g16_prove == submit + wait on slot 0).
 * The host buffers passed to submit (r, s, and the assignment unless G16_ASSIGNMENT_ON_DEVICE) must stay valid
 * until the matching wait.  The *_partial_* pair is the same for the sharded path. */
int g16_prove_submit(g16_ctx* ctx, int slot, const uint64_t* r, const uint64_t* s, const uint64_t* full_assignment,
                     uint32_t flags);
int g16_prove_wait(g16_ctx* ctx, int slot, uint64_t* proof_out);
int g16_prove_partial_submit(g16_ctx* ctx, int slot, const uint64_t* r, const uint64_t* full_assignment, uint32_t flags);
int g16_prove_partial_wait(g16_ctx* ctx, int slot, uint64_t* partial_out);
/* limbs per partial record: 4*2*N64 + 4*N64 */
int g16_partial_limbs(const g16_ctx* ctx);

/* Sharded proving with the exchange INSIDE the library: one NCCL all-gather (over NVLink / NVSwitch) of three partial points
 * per rank, issued by the library on its own stream (SURVEY.md section 8e; no reference counterpart -- ark-groth16 is a
 * single-process CPU prover).  One process per GPU:
 *   rank 0: g16_comm_unique_id(id)  ->  the launcher broadcasts the G16_COMM_ID_BYTES bytes (torch.distributed / MPI / a file)
 *   every rank: g16_comm_init(ctx, id, rank, world); g16_pk_load(ctx, pk, rank, world);
 *   per proof, every rank with the same (r, s, assignment): g16_prove_sharded(...) -> every rank gets the same proof.
 * libnccl is resolved at run time (the copy the host process already loaded, else $G16_NCCL_LIB, else libnccl.so.2).
 * The submit / wait pair is the pipelined form (two slots, as g16_prove_submit / g16_prove_wait).
 * With a communicator the witness map is spread over the ranks as well (option "wm_split", default 1): the chains a, b, c
 * (r1cs_to_qap.rs:201-207,220-221) run on ranks 0, 1, 2 (mod world), meet on rank 3 mod world over ncclSend / ncclRecv
 * (32 B * n each), which runs (a*b - c)/Z and the last coset iFFT, and h is broadcast (ncclBroadcast) for the H MSM. */
#define G16_COMM_ID_BYTES 256 /* two NCCL unique ids: one communicator for the point all-gather, one for the witness map */
int g16_comm_unique_id(uint8_t* out /* G16_COMM_ID_BYTES */);
int g16_comm_init(g16_ctx* ctx, const uint8_t* id /* G16_COMM_ID_BYTES */, uint32_t rank, uint32_t world);
int g16_prove_sharded(g16_ctx* ctx, const uint64_t* r, const uint64_t* s, const uint64_t* full_assignment, uint32_t flags,
                      uint64_t* proof_out);
int g16_prove_sharded_submit(g16_ctx* ctx, int slot, const uint64_t* r, const uint64_t* s, const uint64_t* full_assignment,
                             uint32_t flags);
int g16_prove_sharded_wait(g16_ctx* ctx, int slot, uint64_t* proof_out);

/* ---- witness map alone on the resident circuit (R1CSToQAP::witness_map_from_matrices, r1cs_to_qap.rs:172-235):
 * h_out receives domain_size Montgomery Fr coefficients. */
int g16_witness_map(g16_ctx* ctx, const uint64_t* full_assignment, uint32_t flags, uint64_t* h_out);

/* ---- measurement hooks (bench.py) ---------------------------------------------------------------------------- */
typedef struct {
  float total_ms;        /* CUDA-event time of the last g16_prove / g16_prove_partial, first enqueue to last kernel */
  float h2d_ms;          /* assignment upload                                                                    */
  float witness_map_ms;  /* row evaluation + 7 NTTs                                                              */
  float msm_ms[5];       /* h, l, a, b_g1, b_g2: whole MSM pipeline on its stream                                 */
  float msm_accum_ms[5]; /* the bucket-accumulation kernel (msm_accum_l0) of each MSM                             */
  float host_finish_ms;  /* host Horner + final assembly (prover.rs:76-131)                                       */
  uint64_t msm_pairs[5]; /* (scalar, base) pairs fed to each MSM on this rank                                     */
  uint64_t msm_entries[5]; /* sorted bucket slots of each MSM: non-zero signed digits of live pairs (+ bucket padding
                              of the batched-affine rounds, < 2 %) = point additions of the accumulation stage     */
  uint64_t launches;     /* kernels launched by the last call                                                     */
  uint64_t h2d_bytes, d2h_bytes;
  float msm_begin_ms[5]; /* start / end of each MSM's stream work, measured from the first enqueue of the proof: the       */
  float msm_end_ms[5];   /* concurrent timeline of the five streams (h, l, a, b_g1, b_g2)                                  */
} g16_timings;
int g16_get_timings(const g16_ctx* ctx, g16_timings* out);

/* ---- tuning (no counterpart in the reference: ark-ec picks its window size internally) ---------------------------
 * Launch geometry of the MSM pipeline for the resident key (H query for the G1 fields, B-in-G2 for the G2 ones). */
typedef struct {
  int32_t c, ne, copies;              /* window bits, bucket sets, precomputed multiples per base                 */
  int32_t k0_g1, k0_g2;               /* sorted entries per thread of the level-0 accumulation                    */
  int32_t ba_rounds_g1, ba_rounds_g2; /* batched-affine rounds before the XYZZ accumulation (0 = none)            */
  int32_t ba_m, ba_g, ba_inv_gcd;     /* additions per thread and round; products per inversion; 1 = safegcd      */
  int32_t acc_block, sm_count;
  int32_t rank, world;
  int32_t ba_lean_g1, ba_lean_g2;     /* != 0: register-lean round kernels (more resident warps per SM)           */
  int32_t reserved[2];
} g16_config;
int g16_get_config(const g16_ctx* ctx, g16_config* out);
/* key: "msm_ba", "msm_ba_g2", "ba_m", "ba_g", "ba_inv_gcd", "acc_k0_g1", "acc_k0_g2", "acc_block", "share_b_sort", "ba_occ_g1", "ba_occ_g2",
 * "ba_min_entries_g1", "ba_min_entries_g2" (smallest MSM, in bucket entries, that runs the rounds), "ba_adaptive" (0 = exactly
 * "msm_ba" rounds, 1 = at most that many, fewer for sparsely filled buckets), "ba_cap_fwd_g1", "ba_cap_bwd_g1", "ba_cap_fwd_g2", "ba_cap_bwd_g2", "ntt_tma", "wm_split", "proof_slots", and -- effective at the next
 * g16_pk_load / g16_setup -- "msm_ne", "msm_c", "msm_maxcopies" (the G16_* environment
 * variables of INTEGRATION.md section 6, read once at g16_ctx_create, in lower case without the prefix).  Takes effect
 * from the next proof; results never depend on these knobs. */
int g16_set_option(g16_ctx* ctx, const char* key, int64_t value);
uint32_t g16_domain_log(const g16_ctx* ctx); /* log2 of the resident circuit's domain size */

/* ---- benchmark / test helper (no reference counterpart: arkworks users bring their own circuits) -----------------
 * The non-degenerate synthetic R1CS of SURVEY.md section 8d, generated on the host: constraint i is
 * (z_p + k_i) * z_q = z_new; nc = 2^log_n - 2 constraints, 2 instance variables (One, one public input),
 * nc + 1 witness variables.  Caller-allocated outputs: a_col[2 nc], a_val[2 nc] Montgomery Fr (row i = (1, col_p), (k_i, One)),
 * b_col[nc], c_col[nc] (coefficients 1), full_assignment[nc + 3] Montgomery Fr.  Needs no GPU and no context. */
int g16_synthetic_r1cs(int curve, uint32_t log_n, uint64_t seed, uint32_t* a_col, uint64_t* a_val, uint32_t* b_col,
                       uint32_t* c_col, uint64_t* full_assignment);

#ifdef __cplusplus
}
#endif
#endif /* G16B200_H */
