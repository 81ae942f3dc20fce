/* g16b200.h -- C ABI of libg16b200.so: the H100-native Groth16 proving hot path (NTT witness map + five MSMs).
 *
 * Drop-in boundary for ark-groth16 0.5.0 (/root/reference).  Every entry point names the reference interface it
 * replaces; INTEGRATION.md shows the Rust `extern "C"` binding a maintainer would add.
 *
 * Data layout (SURVEY.md section 8b), identical to ark-ff / ark-ec in-memory values copied field-wise:
 *   Fr / Fq element : N64 little-endian uint64_t limbs in MONTGOMERY form (R = 2^(64*N64)).  Fr: g16_fr_limbs (4 for
 *                     BLS12-381 / BN254 / BLS12-377, 6 for BW6-761).  Fq: g16_fq_limbs (4 for BN254, 6 for BLS12-381 /
 *                     BLS12-377, 12 for BW6-761).  Every Fr array of this ABI (assignments, r, s, setup scalars, NTT
 *                     and witness-map vectors, h_out) is g16_fr_limbs limbs per element.
 *   BigInt scalar   : g16_fr_limbs little-endian uint64_t limbs, canonical integer < r  (`PrimeField::into_bigint`).
 *   G1 affine       : x || y                      (2*N64 limbs);  point at infinity = all-zero limbs.
 *   G2 affine       : x.c0 || x.c1 || y.c0 || y.c1 (4*N64 limbs); point at infinity = all-zero limbs.  BW6-761's G2
 *                     is over Fq: x || y (2*N64 limbs).  g16_g2_limbs gives the size for the context's curve.
 *   Proof           : a (G1) || b (G2) || c (G1): 8*N64 limbs, 6*N64 on BW6-761.
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
  G16_CURVE_BLS12_377 = 2,
  G16_CURVE_BW6_761 = 3   /* the outer curve of BLS12-377 recursion: its r is BLS12-377's q; G2 over Fq */
};

enum {
  G16_OK = 0,
  G16_ERR_POLYNOMIAL_DEGREE_TOO_LARGE = 1, /* SynthesisError::PolynomialDegreeTooLarge, r1cs_to_qap.rs:134,179 */
  G16_ERR_BAD_ARGUMENT = 2,                /* null pointer / inconsistent length / unknown curve               */
  G16_ERR_CUDA = 3,                        /* CUDA failure or no usable sm_90 device; see g16_last_error()     */
  G16_ERR_MALFORMED_KEY = 4,               /* SynthesisError::MalformedVerifyingKey-class length mismatch      */
  G16_ERR_INVALID_DATA = 5,                /* ark_serialize::SerializationError::{InvalidData, UnexpectedFlags,
                                              NotEnoughSpace}: a rejected serialized key                         */
  G16_ERR_UNSATISFIED = 6                  /* SynthesisError::Unsatisfiable: G16_CHECK_WITNESS rejected the assignment;
                                              g16_last_error() names the constraint or element                  */
};

typedef struct g16_ctx g16_ctx;

/* Flags for g16_prove* (bitwise or) */
enum {
  G16_ASSIGNMENT_ON_DEVICE = 1, /* `full_assignment` is a device pointer (bench.py's resident-input measurement) */
  G16_SERIAL_MSMS = 2,          /* run the five MSMs one after another on one stream (kernel-level profiling)    */
  G16_CHECK_WITNESS = 4         /* refuse an assignment that does not satisfy the circuit: see g16_check_witness  */
};

/* ---- context ----------------------------------------------------------------------------------------------- */
/* One context = one curve on one CUDA device.  Fails with G16_ERR_CUDA when no GPU is present: there is no CPU
 * fallback anywhere in this library. */
int g16_ctx_create(int curve, int device, g16_ctx** out);
void g16_ctx_destroy(g16_ctx* ctx);
const char* g16_last_error(void);
/* sizes, in uint64_t limbs, for buffers of this context's curve */
int g16_fq_limbs(const g16_ctx* ctx);
/* one Fr element or BigInt scalar (4, or 6 on BW6-761); one G2 affine point (4*N64, or 2*N64 on BW6-761) */
int g16_fr_limbs(const g16_ctx* ctx);
int g16_g2_limbs(const g16_ctx* ctx);

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
 * Uploaded once per circuit and kept resident.  g16_circuit_load checks all three matrices (row_ptr starts at 0 and never
 * decreases, col / val are not null where entries exist, every column is below num_inputs + num_witness) before it
 * touches anything resident: a rejected circuit leaves the previous circuit and its key resident.  A circuit that passes
 * drops the resident key; a failure while it is uploaded leaves neither a circuit nor a key resident. */
typedef struct {
  const uint32_t* row_ptr;
  const uint32_t* col;
  const uint64_t* val;
} g16_csr;
int g16_circuit_load(g16_ctx* ctx, uint32_t num_inputs /* instance variables incl. the constant One */,
                     uint32_t num_constraints, uint32_t num_witness, const g16_csr* a, const g16_csr* b,
                     const g16_csr* c);

/* ---- R1CS-to-QAP reduction of the resident circuit: the second type parameter of ark-groth16's
 * Groth16<E, QAP: R1CSToQAP = LibsnarkReduction> (lib.rs:55, r1cs_to_qap.rs:71-120).
 *   G16_QAP_LIBSNARK : LibsnarkReduction (r1cs_to_qap.rs:122-248); what g16_circuit_load loads.
 *   G16_QAP_CIRCOM   : ark-circom's CircomReduction (circom circuits with snarkjs-compatible keys).  Its witness map never
 *                      reads matrix C: c = a o b; a, b, c are interpolated on the domain of size n and evaluated at the odd
 *                      powers omega_2n^(2j+1); h[j] = A[j] B[j] - C[j] (n evaluations, no division by Z).  Its H query
 *                      holds n points: the odd entries of the size-2n ifft of delta^-1 tau^i (i < 2n - 1; entry 2n - 1 = 0).
 * Everything that uses the circuit follows its reduction: g16_witness_map (n evaluations), g16_setup / g16_pk_export (H
 * query of n points), g16_prove, submit / wait, g16_prove_batch, g16_prove_partial / g16_prove_assemble and
 * g16_prove_sharded (with "wm_split").  g16_witness_map_evals has no circuit and stays LibsnarkReduction.  C must still
 * be passed: g16_setup needs it.
 * g16_circuit_load_qap(ctx, qap, ...) is g16_circuit_load with the reduction named; an unknown qap is G16_ERR_BAD_ARGUMENT,
 * and for G16_QAP_CIRCOM a domain of size 2n above the field's two-adicity is G16_ERR_POLYNOMIAL_DEGREE_TOO_LARGE (BN254
 * at n = 2^28).  Both are decided from the sizes alone, before any array is read or any resident state is released. */
enum {
  G16_QAP_LIBSNARK = 0,
  G16_QAP_CIRCOM = 1
};
int g16_circuit_load_qap(g16_ctx* ctx, int qap, uint32_t num_inputs, uint32_t num_constraints, uint32_t num_witness,
                         const g16_csr* a, const g16_csr* b, const g16_csr* c);

/* ---- proving key: data_structures.rs:126-143.  Query arrays are the FULL ark vectors (a_query[0] included).
 * With world > 1 the context keeps only the index range of every query owned by `rank` (SURVEY.md section 8e):
 * round-robin split of each MSM's (base, scalar) pairs: pair i belongs to rank i mod world.
 * g16_pk_load and g16_setup check their arguments and the query lengths (an empty a/b query is G16_ERR_MALFORMED_KEY) before
 * they release the resident key: a key rejected there leaves the previous key resident.  A failure after that leaves no key
 * resident. */
typedef struct {
  const uint64_t* a_query;    uint64_t a_len;     /* G1, num_inputs + num_witness      (generator.rs:155) */
  const uint64_t* b_g1_query; uint64_t b_g1_len;  /* G1, same length                   (generator.rs:161) */
  const uint64_t* b_g2_query; uint64_t b_g2_len;  /* G2, same length                   (generator.rs:134) */
  const uint64_t* h_query;    uint64_t h_len;     /* G1, domain_size - 1               (generator.rs:168);
                                                     G16_QAP_CIRCOM: domain_size */
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
  uint64_t* h_query;    /* capacity domain_size - 1 (G16_QAP_CIRCOM: domain_size) */
  uint64_t* l_query;    /* capacity num_witness */
  uint64_t* alpha_g1; uint64_t* beta_g1; uint64_t* delta_g1;
  uint64_t* beta_g2; uint64_t* gamma_g2; uint64_t* delta_g2;
  uint64_t* gamma_abc_g1; /* capacity num_inputs G1 */
} g16_pk_export_desc;
int g16_pk_export(g16_ctx* ctx, const g16_pk_export_desc* out);

/* ---- proving keys from a powers-of-tau transcript, with nobody holding tau: phase 2 of Bowe-Gabizon-Miers ("Scalable
 * Multi-Party Computation for zk-SNARK Parameters in the Random Beacon Model"), as snarkjs keys are made.
 * The transcript of a circuit with domain size n = 2^g16_domain_log holds, as affine Montgomery limbs (all-zero limbs for
 * the identity): tau_g1 = [tau^i]G1 (at least 2n - 1 points), tau_g2 = [tau^i]G2 (at least n), alpha_tau_g1 = [alpha
 * tau^i]G1 and beta_tau_g1 = [beta tau^i]G1 (at least n each), beta_g2 = [beta]G2.  Longer members are allowed (ceremonies
 * are sized for the largest circuit); only the prefixes above are read, checked and used.
 * g16_setup_from_srs derives the key of the resident circuit under its reduction on the GPU (four group inverse FFTs, the
 * sparse sums of the queries, the H query) and makes it resident as g16_setup does (rank 0 / world 1; g16_pk_export,
 * g16_pk_export_serialized and every prover path take it).  gamma = 1, and with no contribution delta = 1: the key equals
 * g16_setup(alpha, beta, 1, 1, tau, tau_g1[0], tau_g2[0]) point for point.  flags: 0 or G16_SER_VALIDATE (adds the
 * subgroup check [r]P = O of every point read; always checked: coordinates below q and on the curve).
 * Argument errors leave the previous key resident: a null pointer, unknown flags, no circuit, a member shorter than it
 * must be (G16_ERR_BAD_ARGUMENT naming the member and the length it needs), a proof in flight.  A point the checks refuse is
 * G16_ERR_INVALID_DATA, g16_last_error() naming the first one by member and index ("alpha_tau_g1[17]: point is not on the
 * curve"), and no key is resident afterwards.
 * g16_setup_contribute applies one phase-2 contribution delta (Montgomery Fr, non-zero) to the resident key: delta_g1 and
 * delta_g2 times delta, every h_query and l_query point times delta^-1.  After contributions delta_1 .. delta_k the key equals
 * g16_setup(alpha, beta, 1, delta_1 ... delta_k, tau, g1, g2); on a g16_setup key made with delta it equals g16_setup with
 * delta delta'.  It needs a key made by g16_setup or g16_setup_from_srs (world 1); any other, no key, or delta = 0 is
 * G16_ERR_BAD_ARGUMENT with the key unchanged.  The key is re-committed, so everything derived from it is rebuilt.
 * After g16_setup_from_srs, g16_get_timings describes that call instead of the last proof (the fields keep their types, not
 * their prover meaning; every other field is 0): total_ms = the whole call, h2d_ms = upload and point checks, witness_map_ms
 * = the four group inverse transforms, msm_ms[0] = the H query, msm_ms[1] = the sparse sums of the other queries. */
typedef struct {
  const uint64_t* tau_g1;       uint64_t tau_g1_len;
  const uint64_t* tau_g2;       uint64_t tau_g2_len;       /* g16_g2_limbs per point */
  const uint64_t* alpha_tau_g1; uint64_t alpha_tau_g1_len;
  const uint64_t* beta_tau_g1;  uint64_t beta_tau_g1_len;
  const uint64_t* beta_g2;
} g16_srs_desc;
int g16_setup_from_srs(g16_ctx* ctx, const g16_srs_desc* srs, uint32_t flags);
int g16_setup_contribute(g16_ctx* ctx, const uint64_t* delta);
/* Test and benchmark helper, no reference counterpart: the transcript of explicit secrets tau, alpha, beta (Montgomery Fr)
 * over the affine generators g1, g2, each member as long as the caller's *_len (fixed-base multiplications on the GPU).
 * Needs no circuit and leaves the resident circuit and key alone. */
typedef struct { uint64_t* tau_g1; uint64_t tau_g1_len; uint64_t* tau_g2; uint64_t tau_g2_len;
                 uint64_t* alpha_tau_g1; uint64_t alpha_tau_g1_len; uint64_t* beta_tau_g1; uint64_t beta_tau_g1_len;
                 uint64_t* beta_g2; } g16_srs_out;
int g16_srs_from_secrets(g16_ctx* ctx, const uint64_t* tau, const uint64_t* alpha, const uint64_t* beta,
                         const uint64_t* g1, const uint64_t* g2, const g16_srs_out* out);
/* Phase 1 of the ceremony, the contributor's side (snarkjs `powersoftau contribute`): one contribution tau, alpha, beta
 * (Montgomery Fr, g16_fr_limbs limbs each, all non-zero) to the transcript `in`, written to `out`.  Point i of each member is
 * the input point i times its own scalar: tau_g1[i] and tau_g2[i] times tau^i, alpha_tau_g1[i] times alpha tau^i,
 * beta_tau_g1[i] times beta tau^i, beta_g2 times beta; the identity (all-zero limbs) stays the identity.  After
 * contributions (tau_k, alpha_k, beta_k) to g16_srs_from_secrets(1, 1, 1, g1, g2) the transcript equals
 * g16_srs_from_secrets(prod tau_k, prod alpha_k, prod beta_k, g1, g2) limb for limb.  Phase 1 knows no circuit: any length
 * from 0 to 2^32 - 1 per member, out->*_len equal to in->*_len; a member of length 0 may be null and is skipped; beta_g2
 * (one point) is always read and written.  out->m may be the very same pointer as in->m (in place); any other overlap of an
 * output range with an input or another output range is refused.  The result does not depend on chunk_points, on in place
 * or not, or on flags.
 * Two passes over the members in chunks of at most chunk_points points (0: as many as the free device memory holds; any
 * value is also capped by it), so a transcript larger than the device streams through: first every point is uploaded and
 * checked (coordinates below q, on the curve; G16_SER_VALIDATE adds [r]P = O), and only when all have passed is each chunk
 * uploaded again, multiplied on the GPU (one thread per point, its scalar formed on the device from tau^(2^k)) and written
 * to out.  A refused point returns G16_ERR_INVALID_DATA with g16_last_error() naming the first one by member and then index
 * ("beta_tau_g1[70001]: point is not on the curve") and nothing written to out, so an in-place transcript is intact.
 * G16_ERR_BAD_ARGUMENT, decided before any point is read: a null pointer where a point or scalar is needed, flags other
 * than 0 or G16_SER_VALIDATE, a secret equal to 0 ("UnexpectedIdentity"), in and out lengths that differ, a length of 2^32
 * or more, overlapping ranges, a proof in flight.  Needs no circuit or key and leaves the resident ones and everything
 * derived from them alone.  Afterwards g16_get_timings describes this call (every other field 0): total_ms = the whole
 * call, h2d_ms = the check pass, msm_ms[0..3] = the transform of tau_g1, tau_g2, alpha_tau_g1, beta_tau_g1 (host clock
 * around work that ends in a stream synchronise), h2d_bytes / d2h_bytes = bytes copied each way, launches = kernels. */
int g16_srs_contribute(g16_ctx* ctx, const g16_srs_desc* in, const uint64_t* tau, const uint64_t* alpha, const uint64_t* beta,
                       uint32_t flags, uint64_t chunk_points, const g16_srs_out* out);
/* Phase 1 of the ceremony, the checker's side (snarkjs `powersoftau verify`; the contributions' proofs of knowledge are
 * g16_contribution_chain_pairs):
 * the GPU part of checking that `srs` is a powers-of-tau transcript T(tau, alpha, beta) over the agreed affine generators g1,
 * g2.  rho (Montgomery Fr, non-zero) is a challenge the caller draws after the transcript is fixed, which whoever made the
 * transcript cannot predict (a CSPRNG, or a hash of the transcript).  For a member X of N points let
 *   S_X = sum_{i<N} rho^i X_i        (one MSM per member, on the GPU)
 *   lo_X = S_X - rho^(N-1) X_(N-1) = sum_{i<N-1} rho^i X_i,   hi_X = rho^-1 (S_X - X_0) = sum_{i<N-1} rho^i X_(i+1)
 * (a member of one point has lo = hi = the identity).  The call writes ten affine G1 points P_0, P'_0, .., P_4, P'_4 to
 * pairs_g1 and ten affine G2 points Q_0, Q'_0, .., Q_4, Q'_4 to pairs_g2; equation k holds iff e(P_k, Q_k) = e(P'_k, Q'_k):
 *   k = 0  tau_g1        (hi_T1, g2)               = (lo_T1, tau_g2[1])
 *   k = 1  tau_g2        (g1, hi_T2)               = (tau_g1[1], lo_T2)
 *   k = 2  alpha_tau_g1  (hi_A, g2)                = (lo_A, tau_g2[1])
 *   k = 3  beta_tau_g1   (hi_B, g2)                = (lo_B, tau_g2[1])
 *   k = 4  beta_g2       (beta_tau_g1[0], g2)      = (g1, beta_g2)
 * The pairings are the caller's: this library has none.  The call itself checks every point (coordinates below q, on the
 * curve; G16_SER_VALIDATE adds [r]P = O, without which the answer means nothing on a curve whose cofactor is not 1), that no
 * point is the identity (it would mean tau, alpha or beta = 0), and that tau_g1[0] = g1 and tau_g2[0] = g2.  If those pass
 * and all five equations hold, then with probability at least 1 - N/r over rho (N the longest member) the transcript is
 * T(tau, alpha, beta) for some non-zero tau, alpha, beta with the same tau in both groups: a member that is not geometric
 * with ratio tau makes sum_i rho^i (X_(i+1) - tau X_i) a non-zero polynomial in rho of degree at most N - 2 (Schwartz-Zippel).
 * alpha has no G2 counterpart in a transcript, so its chain is checked against tau only, which is all Groth16 needs.
 * Lengths: tau_g1 and tau_g2 at least 2 points, alpha_tau_g1 and beta_tau_g1 at least 1, each below 2^32; beta_g2 is one
 * point.  One pass over the members in chunks of at most chunk_points points (0: as many as the free device memory holds,
 * counting the points, their scalars and the MSM workspace; any value is also capped by it and by 2^27 - 1), so a
 * transcript larger than the device streams through: each chunk is uploaded and checked, and only then are its scalars
 * rho^i formed on the device (one thread per point, from rho^(2^k)) and its MSM run.  A refused point returns
 * G16_ERR_INVALID_DATA with g16_last_error() naming the first one by member and then index ("tau_g2[5]: point is the
 * identity", "tau_g1[0]: not the generator g1") and nothing written; later chunks are not read.  The identity is refused by
 * this call only: g16_setup_from_srs and g16_srs_contribute accept it.
 * G16_ERR_BAD_ARGUMENT, decided before any point is read, with nothing written: a null pointer, flags other than 0 or
 * G16_SER_VALIDATE, rho = 0, a member shorter than the lengths above or of 2^32 points or more, a proof in flight.  Needs no
 * circuit or key and leaves the resident ones and everything derived from them alone.  The result does not depend on
 * chunk_points or on flags.  Afterwards g16_get_timings describes this call (every other field 0): total_ms = the whole
 * call, msm_ms[0..3] = the chunk loop (upload, check, scalars, MSM) of tau_g1, tau_g2, alpha_tau_g1, beta_tau_g1 (host
 * clock around work that ends in a stream synchronise), msm_pairs[0..3] = the points of each member's MSM, h2d_bytes /
 * d2h_bytes = bytes copied each way, launches = kernels. */
int g16_srs_verify_pairs(g16_ctx* ctx, const g16_srs_desc* srs, const uint64_t* g1, const uint64_t* g2, const uint64_t* rho,
                         uint32_t flags, uint64_t chunk_points, uint64_t* pairs_g1, uint64_t* pairs_g2);
/* Phase 2 of the ceremony, the user's side (snarkjs `zkey verify`; the contributions' proofs of knowledge are
 * g16_contribution_chain_pairs): the GPU
 * part of checking that `pk`, a proving key received from elsewhere, is the key of the resident circuit (under its
 * reduction) made from the transcript `srs`, i.e. g16_setup(alpha, beta, gamma, delta, tau) for the transcript's tau, alpha,
 * beta and some gamma, delta.  pk holds the members of g16_pk_export_desc, read-only, with the lengths g16_pk_export writes:
 * a_query, b_g1_query, b_g2_query num_inputs + num_witness points, h_query n - 1 (G16_QAP_CIRCOM: n), l_query num_witness,
 * gamma_abc_g1 num_inputs, the six single points one each (a member of no points may be null).  Transcript members may be
 * longer than the circuit needs; only the prefixes g16_setup_from_srs reads are read (tau_g1 2n - 1 points, tau_g2,
 * alpha_tau_g1, beta_tau_g1 n each, beta_g2).  rho (Montgomery Fr, non-zero) is a challenge the caller draws after the key
 * and transcript are fixed.
 * With z_j = rho^j (j < nv = num_inputs + num_witness) and g1 = tau_g1[0], g2 = tau_g2[0], the call forms
 *   S_X(K) = sum_j rho^j X_j over a key member X (for l_query: sum_t rho^(num_inputs + t) l_query[t])
 * and the same combination of the transcript, S_X(T), from field transforms of z as DESIGN.md section 16 gives (one MSM per
 * transcript member; no group transform).  It decides itself, and refuses the key with G16_ERR_INVALID_DATA naming the
 * member if one fails, in this order: tau_g1[0] and tau_g2[0] are not the identity; alpha_g1 = alpha_tau_g1[0], beta_g1 =
 * beta_tau_g1[0], beta_g2 = the transcript's beta_g2 ("alpha_g1: not alpha_tau_g1[0] of the transcript"); delta_g1, delta_g2
 * and gamma_g2 are not the identity; gamma_g2 != delta_g2 ("gamma_g2 equals delta_g2: ...": gamma = delta lets anyone forge
 * proofs for any public input, and an uncontributed g16_setup_from_srs key has gamma = delta = 1 -- flag
 * G16_PK_UNCONTRIBUTED accepts it, for the coordinator of a ceremony); S_X(K) = S_X(T) for a_query, b_g1_query and
 * b_g2_query ("b_g2_query: not the key of the resident circuit under this transcript").  Then it writes eight affine G1 points
 * P_0, P'_0, .., P_3, P'_3 to pairs_g1 and eight affine G2 points Q_0, Q'_0, .., Q_3, Q'_3 to pairs_g2; equation k holds iff
 * e(P_k, Q_k) = e(P'_k, Q'_k):
 *   k = 0  delta         (delta_g1, g2)          = (g1, delta_g2)
 *   k = 1  h_query       (S_H(K), delta_g2)      = (S_H(T), g2)
 *   k = 2  l_query       (S_L(K), delta_g2)      = (S_L(T), g2)
 *   k = 3  gamma_abc_g1  (S_IC(K), gamma_g2)     = (S_IC(T), g2)
 * The pairings are the caller's: this library has none.  If every point passes (with G16_SER_VALIDATE; without it the
 * answer means nothing on a curve whose cofactor is not 1), the call accepts and all four equations hold, then with
 * probability at least 1 - 6 N / r over rho (N = max(nv, n)) the key equals g16_setup(alpha, beta, gamma, delta, tau, g1, g2)
 * point for point, for the transcript's tau, alpha, beta and some non-zero gamma != delta: a member that differs anywhere
 * makes sum_j rho^j (K_j - K'_j) a non-zero polynomial in rho of degree below N that one of six equations forces to zero
 * (Schwartz-Zippel).  It does not show that nobody knows delta: g16_contribution_chain_pairs from tau_g1[0] to delta_g1
 * does.  The
 * transcript itself should have passed g16_srs_verify_pairs.
 * Points: coordinates below q and on the curve, with G16_SER_VALIDATE also [r]P = O; the identity is valid in the key (an
 * unused variable has it).  A refused point is G16_ERR_INVALID_DATA, g16_last_error() naming the first one, key members
 * before transcript members, by member and index ("l_query[17]: point is not on the curve", "tau_g1[3]: ...").
 * G16_ERR_BAD_ARGUMENT, decided before any point is read: a null pointer (pk members of no points excepted), flags other
 * than G16_SER_VALIDATE | G16_PK_UNCONTRIBUTED, rho = 0, no resident circuit, a transcript member shorter than the
 * circuit needs (naming the length it needs), a proof in flight.  Nothing is written to pairs_g1 / pairs_g2 unless the
 * call returns G16_OK.  Needs a resident circuit and no key, and leaves the resident circuit, key and everything derived
 * from them alone.  Afterwards g16_get_timings describes this call (every other field 0): total_ms = the whole call, h2d_ms
 * = upload and point checks, witness_map_ms = the field work (powers of rho, the matrix products, the transforms),
 * msm_ms[0] / msm_ms[1] = the key-side / transcript-side MSMs (host clock around work that ends in a stream synchronise),
 * msm_pairs[0] / msm_pairs[1] = their points (3 nv + |h_query| + num_witness + num_inputs; 11 n - 1), h2d_bytes /
 * d2h_bytes = bytes copied each way, launches = kernels. */
enum { G16_PK_UNCONTRIBUTED = 4 };
typedef struct {
  const uint64_t* a_query;
  const uint64_t* b_g1_query;
  const uint64_t* b_g2_query;
  const uint64_t* h_query;
  const uint64_t* l_query;
  const uint64_t* alpha_g1; const uint64_t* beta_g1; const uint64_t* delta_g1;
  const uint64_t* beta_g2; const uint64_t* gamma_g2; const uint64_t* delta_g2;
  const uint64_t* gamma_abc_g1;
} g16_pk_check_desc;
int g16_pk_verify_pairs(g16_ctx* ctx, const g16_srs_desc* srs, const g16_pk_check_desc* pk, const uint64_t* rho,
                        uint32_t flags, uint64_t* pairs_g1, uint64_t* pairs_g2);
/* Phase 2 of the ceremony, a contributor's side for a key it was sent (snarkjs `zkey contribute`): one contribution delta
 * (Montgomery Fr, non-zero) to the delta-dependent members of a proving key held in host memory, written to `out`.
 * delta_g1 and delta_g2 are multiplied by delta, every h_query and l_query point by delta^-1; the identity (all-zero limbs)
 * stays the identity (an unused variable has it in l_query).  No other key member changes, so the call does not take them.
 * On a key g16_setup(alpha, beta, gamma, delta0, tau) the result is g16_setup(alpha, beta, gamma, delta0 delta, tau) limb
 * for limb, and on the key g16_setup_contribute(delta) would change it is what that call makes.  Lengths run from 0 to
 * 2^32 - 1, out->h_len and out->l_len equal to the input's; a member of length 0 may be null; delta_g1 and delta_g2 are
 * always read and written.  out->m may be the very same pointer as in->m (in place); any other overlap of an output range
 * with an input or another output range is refused.  The result does not depend on chunk_points, on in place or not, or on
 * flags.
 * Two passes in chunks of at most chunk_points points (0: as many as the free device memory holds; any value is also capped
 * by it), so a key larger than the device streams through: first every point is uploaded and checked (coordinates below q,
 * on the curve; G16_SER_VALIDATE adds [r]P = O; delta_g1 and delta_g2 must not be the identity), and only when all have
 * passed is each chunk of h_query and l_query uploaded again, multiplied on the GPU (one thread per point, all by delta^-1)
 * and written to out; delta_g1 and delta_g2 are multiplied on the host.  A refused point returns G16_ERR_INVALID_DATA with
 * g16_last_error() naming the first one ("l_query[70001]: point is not on the curve", "delta_g2: point is the identity")
 * and nothing written to out, so an in-place key is intact.
 * G16_ERR_BAD_ARGUMENT, decided before any point is read: a null pointer where a point or scalar is needed, flags other
 * than 0 or G16_SER_VALIDATE, delta = 0 ("UnexpectedIdentity"), in and out lengths that differ, a length of 2^32 or more,
 * overlapping ranges, a proof in flight.  Needs no circuit or key and leaves the resident ones and everything derived from
 * them alone.  Afterwards g16_get_timings describes this call (every other field 0): total_ms = the whole call, h2d_ms =
 * the check pass, msm_ms[0] / msm_ms[1] = the transform of h_query / l_query (host clock around work that ends in a
 * stream synchronise), h2d_bytes / d2h_bytes = bytes copied each way, launches = kernels. */
typedef struct {
  const uint64_t* h_query; uint64_t h_len;
  const uint64_t* l_query; uint64_t l_len;
  const uint64_t* delta_g1; const uint64_t* delta_g2;
} g16_pk_delta_desc;
typedef struct {
  uint64_t* h_query; uint64_t h_len;
  uint64_t* l_query; uint64_t l_len;
  uint64_t* delta_g1; uint64_t* delta_g2;
} g16_pk_delta_out;
int g16_pk_contribute(g16_ctx* ctx, const g16_pk_delta_desc* in, const uint64_t* delta, uint32_t flags, uint64_t chunk_points,
                      const g16_pk_delta_out* out);
/* Both phases, the checker's side: the proofs of knowledge of a chain of contributions (the public keys of Bowe, Gabizon
 * and Miers, as snarkjs and bellman's phase2 publish them).  One contribution multiplies a running G1 point D by the
 * contributor's secret x: in phase 2 D is delta_g1 and x is delta; in phase 1 there are three chains, tau_g1[1] with x =
 * tau, alpha_tau_g1[0] with alpha, beta_tau_g1[0] with beta.  Contributor i publishes records[i]: after_g1 = D_(i+1) =
 * x_i D_i, a G1 point s of its choice, s_x_g1 = x_i s, and r_x_g2 = x_i r_i, where r_i (r_g2) is a G2 point
 * hashed from the contribution's transcript.
 * r_i MUST be derived by the checker itself from the ceremony's transcript (the hash to G2 and the file format that binds
 * it, such as snarkjs .zkey contribution sections or bellman's params, are the caller's; this library fixes no hash).  It
 * must never be taken from the contributor: an r whose discrete log is known makes the proof of knowledge empty.
 * With D_0 = start_g1, the call writes 2 count equations as 4 count affine G1 points P_0, P'_0, P_1, P'_1, .. to pairs_g1
 * and as many affine G2 points Q_0, Q'_0, .. to pairs_g2; equation k holds iff e(P_k, Q_k) = e(P'_k, Q'_k):
 *   k = 2i      proof of knowledge   (s_i, r_x_i)   = (s_x_i, r_i)
 *   k = 2i + 1  step                 (D_i, r_x_i)   = (D_(i+1), r_i)
 * If all hold, D_count = (prod x_i) D_0 with x_i the discrete log of r_x_i to the base r_i, and when r_i is a random-oracle
 * output over the contribution's transcript, contributor i knew x_i; one honest contributor then makes the product unknown.
 * In phase 2, D_0 is the uncontributed key's delta_g1 = tau_g1[0]; with g16_pk_verify_pairs on the final key, delta is
 * that product.  The pairings are the caller's: this library has none.
 * The call itself checks, in one upload of every point through the GPU point check: coordinates below q, on the curve,
 * G16_SER_VALIDATE adding [r]P = O; no point is the identity; and records[count - 1].after_g1 = end_g1.  A refusal is
 * G16_ERR_INVALID_DATA naming the first bad point by record, then member ("records[3].r_x_g2: point is the identity",
 * "records[4].after_g1: not end_g1", "start_g1: point is not on the curve").  G16_ERR_BAD_ARGUMENT: a null pointer, count = 0
 * or 2^30 or more, flags other than 0 or G16_SER_VALIDATE, a proof in flight.  Nothing is written unless the call returns
 * G16_OK.  Runs no MSM; needs no circuit or key and leaves the resident ones alone.  Afterwards g16_get_timings describes
 * this call (every other field 0): total_ms = the whole call, h2d_ms = upload and point checks, h2d_bytes / d2h_bytes =
 * bytes copied each way, launches = kernels. */
typedef struct {
  const uint64_t* after_g1; /* D_(i+1) = x_i D_i */
  const uint64_t* s_g1;     /* a G1 point the contributor chose */
  const uint64_t* s_x_g1;   /* x_i s */
  const uint64_t* r_g2;     /* hash to G2 of the contribution's transcript, recomputed by the checker */
  const uint64_t* r_x_g2;   /* x_i r */
} g16_contribution_record;
int g16_contribution_chain_pairs(g16_ctx* ctx, const uint64_t* start_g1, const uint64_t* end_g1,
                                 const g16_contribution_record* records, uint32_t count, uint32_t flags, uint64_t* pairs_g1,
                                 uint64_t* pairs_g2);

/* ---- ark-serialized proving keys: `ProvingKey::serialize_{compressed,uncompressed}` / `deserialize_with_mode`
 * (data_structures.rs:125 derives them).  The bytes are a whole ProvingKey<E> as ark-serialize 0.5 writes it: vk {alpha_g1,
 * beta_g2, gamma_g2, delta_g2, gamma_abc_g1}, beta_g1, delta_g1, a_query, b_g1_query, b_g2_query, h_query, l_query; vectors
 * are u64-LE length-prefixed.  Points: BLS12-381 zcash / IETF (big-endian, three flag bits, Fq2 as c1 || c0); BN254 and
 * BLS12-377 generic short Weierstrass (little-endian, SWFlags in the top bits of the last byte).  The VerifyingKey bytes are
 * the prefix of the ProvingKey bytes.
 *   G16_SER_COMPRESSED selects the encoding (x and a sign bit); G16_SER_VALIDATE adds the prime-order-subgroup check
 *   [r]P = O of every point (not needed, and skipped, for BN254 G1, whose cofactor is 1).  Always checked: truncation,
 *   trailing bytes, length prefixes above 2^28, the flag bits, zero bytes under the infinity flag, canonical coordinates
 *   (< q), that a compressed x has a curve point and that an uncompressed point is on the curve.
 * g16_pk_load_serialized decodes, validates and places the key on the GPU and makes it resident with exactly the rules of
 * g16_pk_load: truncation to the circuit, rank / world shares; every rank decodes and validates all points.  A rejected key
 * returns G16_ERR_INVALID_DATA, g16_last_error() naming the first bad item in stream order (member, index, reason); a
 * gamma_abc_g1 that does not hold num_inputs points, or an empty a/b query, returns G16_ERR_MALFORMED_KEY.  After either no
 * key is resident.  A non-null vk_out receives alpha_g1, beta_g1, delta_g1, beta_g2, gamma_g2, delta_g2 and gamma_abc_g1
 * (capacity num_inputs); its five query members must be NULL.
 * g16_pk_export_serialized writes the resident key (made by g16_setup; any other is G16_ERR_BAD_ARGUMENT) in the same
 * format; flags is 0 or G16_SER_COMPRESSED.  out == NULL: *len_out receives the size only; cap below it is
 * G16_ERR_BAD_ARGUMENT with the size in *len_out. */
enum { G16_SER_COMPRESSED = 1, G16_SER_VALIDATE = 2 };
int g16_pk_load_serialized(g16_ctx* ctx, const uint8_t* bytes, uint64_t len, uint32_t flags, uint32_t rank, uint32_t world,
                           const g16_pk_export_desc* vk_out);
int g16_pk_export_serialized(g16_ctx* ctx, uint32_t flags, uint8_t* out, uint64_t cap, uint64_t* len_out);

/* ---- snarkjs .zkey files: the circuit and its proving key in one call, the GPU counterpart of ark-circom's read_zkey followed
 * by Groth16<E, CircomReduction>.  `bytes` is a whole Groth16 .zkey (circuit_final.zkey) of the context's curve: "zkey",
 * version 1, nSections, then {id u32, size u64, body} records; sections 1 .. 9 exactly once each, in any order, ids >= 10
 * (section 10: the MPC contributions) skipped.  1: protocol = 1 (Groth16).  2: n8q, q, n8r, r, nVars, nPublic, domainSize,
 * alpha1, beta1, beta2, gamma2, delta1, delta2.  3: IC (nPublic + 1 G1) = gamma_abc_g1.  4: nCoefs, then {matrix (0 = A,
 * 1 = B), constraint, signal, value} records, value the canonical c R^2 mod r.  5 / 6 / 7: A / B1 / B2 (nVars points) =
 * a_query / b_g1_query / b_g2_query.  8: C (nVars - nPublic - 1 G1) = l_query.  9: H (domainSize G1) = h_query.  Integers
 * are little-endian; a coordinate is n8q bytes in Montgomery form, which is this ABI's; G2 is x.c0 || x.c1 || y.c0 || y.c1;
 * the identity is all-zero bytes.  snarkjs appends row nConstraints + s = {(s, 1)} to A for s = 0 .. nPublic; the call
 * derives num_inputs = nPublic + 1, num_witness = nVars - nPublic - 1, num_constraints = (largest constraint index) -
 * nPublic, checks that those rows are exactly the appended ones (B: empty) and drops them (CircomReduction appends them
 * itself), and that domainSize is the smallest power of two >= num_constraints + num_inputs.
 * One call makes the circuit resident under G16_QAP_CIRCOM with A and B built on the GPU (one thread per coefficient
 * record decodes and counts, an exclusive scan gives row_ptr, a scatter fills col / val; the order of entries within a row
 * is free, and no result depends on it or on the chunking), and makes the key resident with the rules of g16_pk_load
 * (rank / world shards; every rank decodes and checks everything).  Every prover path and g16_witness_map then take them.
 * flags: 0 or G16_SER_VALIDATE (adds [r]P = O of every point).  Always checked: coordinates below q, points on the curve;
 * coefficients with matrix < 2, constraint < domainSize, signal < nVars, value < r.
 *   Host checks, decided before anything resident is released (a refusal leaves the previous circuit and key resident):
 *   G16_ERR_BAD_ARGUMENT for a null pointer, flags other than 0 or G16_SER_VALIDATE, a vk_out with query members, bad
 *   rank / world, a proof in flight, and a BLS12-377 or BW6-761 context (snarkjs has neither curve; no byte is read);
 *   G16_ERR_INVALID_DATA for the section table (magic, version, truncation, trailing bytes, a missing or duplicated
 *   section), a section size that does not match the header, protocol != 1, n8q / q / n8r / r other than the context's
 *   curve, nVars < nPublic + 1, a domainSize that is not a power of two; G16_ERR_POLYNOMIAL_DEGREE_TOO_LARGE for a domain
 *   the CircomReduction cannot run.
 *   Device checks: then the old circuit and key are dropped, as g16_pk_load_serialized drops the old key.  A coefficient or
 *   point the GPU refuses, appended rows that are not the public-input rows, or a domainSize that is not the derived
 *   circuit's return G16_ERR_INVALID_DATA and leave neither a circuit nor a key resident.
 *   g16_last_error() names the first bad item in file order: "coefficient 1234: signal 70000 >= nVars 65536", "B2[17] (byte
 *   n): point is not on the curve", "coefficients: public-input row 3 of A is not {(3, 1)}".
 * A .zkey holds no C matrix: C is resident as an empty matrix, and the calls that read it refuse the circuit with
 * G16_ERR_BAD_ARGUMENT ("the resident circuit came from a .zkey, which holds no C matrix"): g16_check_witness, the flag
 * G16_CHECK_WITNESS on every path, g16_setup, g16_setup_from_srs and g16_pk_verify_pairs.  The CircomReduction witness map
 * never reads C (also on the sharded path with "wm_split": chain c starts from a o b).  The next g16_circuit_load* clears
 * the state.
 * vk_out as in g16_pk_load_serialized (nullable; capacity num_inputs in gamma_abc_g1; query members NULL).  info_out
 * (nullable) receives the derived sizes, log2 of the domain and the entries of A and B.  Afterwards g16_get_timings
 * describes this call (every other field 0): total_ms = the whole call, witness_map_ms = coefficient upload, decode and CSR
 * build, h2d_ms = upload and point checks (host clock around work that ends in a stream synchronise), h2d_bytes / d2h_bytes
 * = bytes copied each way, launches = kernels. */
typedef struct {
  uint32_t num_inputs, num_constraints, num_witness, log_n;
  uint64_t a_nnz, b_nnz;
} g16_zkey_info;
int g16_zkey_load(g16_ctx* ctx, const uint8_t* bytes, uint64_t len, uint32_t flags, uint32_t rank, uint32_t world,
                  const g16_pk_export_desc* vk_out, g16_zkey_info* info_out);
/* G16_ZKEY_KEY_ONLY (flags of g16_zkey_load, with or without G16_SER_VALIDATE): only the key of the .zkey is made resident,
 * onto the resident circuit, which stays as it is with its C matrix (the circom flow: g16_r1cs_load of circuit.r1cs, then
 * the key of circuit_final.zkey).  The same section walk, header checks and point decode run; the key is placed with the
 * rules of g16_pk_load (rank / world, vk_out).  Section 4 is not decoded: proofs use the resident A and B, and whether the
 * key belongs to the resident circuit is g16_pk_verify_pairs's question, as after g16_pk_load.
 *   Decided on the host, leaving the previous key resident: no resident circuit, or one under G16_QAP_LIBSNARK, is
 *   G16_ERR_BAD_ARGUMENT (a snarkjs H query has domainSize points: a CircomReduction key); nVars other than num_inputs +
 *   num_witness, nPublic + 1 other than num_inputs, or domainSize other than 2^log_n is G16_ERR_MALFORMED_KEY naming the
 *   field.  A point the GPU refuses is G16_ERR_INVALID_DATA and leaves the circuit resident and no key.  info_out
 *   (nullable) receives the resident circuit's sizes (a_nnz / b_nnz 0 for a circuit loaded by a full g16_zkey_load). */
enum { G16_ZKEY_KEY_ONLY = 16 };

/* ---- circom .r1cs circuits: all three matrices made resident, the GPU counterpart of ark-circom's R1CSFile followed by
 * CircomCircuit.  `bytes` is a whole .r1cs (iden3 r1csfile): "r1cs", version u32 = 1, nSections u32, then {type u32, size
 * u64, body} records in any order; integers little-endian.  Sections 1 and 2 exactly once each; 4 and 5 (custom gates,
 * PLONK only) are refused; every other section (3: the wire-to-label map) is skipped.
 *   1 (header, exactly 32 + n8 bytes): n8 u32, prime (n8 bytes), nWires u32, nPubOut u32, nPubIn u32, nPrvIn u32,
 *     nLabels u64, mConstraints u32.
 *   2 (constraints): mConstraints records of three linear combinations, A then B then C; each is nTerms u32 followed by
 *     nTerms {wire u32, coefficient (n8 bytes, canonical: standard form, below r)}.  A constraint means A.w * B.w - C.w = 0.
 * The circuit: num_inputs = 1 + nPubOut + nPubIn, num_witness = nWires - num_inputs, num_constraints = mConstraints,
 * column = wire id (wire 0 is One, instance first), under the reduction `qap` with g16_circuit_load_qap's rules.  Terms are
 * kept as the file has them, in file order (zero coefficients and repeated wires stay separate entries, as ark-circom
 * pushes them); every result is a field sum, so all results equal those of the compacted matrices.
 *   Host checks, decided before anything resident is released (a refusal leaves the previous circuit and key resident):
 *   G16_ERR_BAD_ARGUMENT for null bytes, an unknown qap, a proof in flight; G16_ERR_INVALID_DATA for the section table
 *   (magic, version, truncation, trailing bytes, section 1 or 2 missing or repeated, section 4 or 5), the header (its
 *   size, n8 other than the context's scalar size, a prime other than its r, nWires < 1 + nPubOut + nPubIn + nPrvIn), a
 *   constraint section whose size is not 12 mConstraints + (4 + n8) (all terms), and a matrix of 2^32 or more entries;
 *   G16_ERR_POLYNOMIAL_DEGREE_TOO_LARGE for the domain.  g16_last_error() names what failed ("section 2 holds 1234 bytes,
 *   its constraints need 1270", "section 1: prime is not the scalar field modulus of this curve").
 *   Device checks: then the old circuit and key are dropped.  One GPU thread per term checks wire < nWires and coefficient
 *   < r and writes c R at row_ptr[row] + its position (no atomics: the CSR is the file's order).  A refused term is
 *   G16_ERR_INVALID_DATA naming the first in file order ("constraint 17, C term 2 (byte 123456): wire 70000 >= nWires
 *   65536", "...: coefficient is not below r") and leaves neither a circuit nor a key resident.
 * On success the circuit stands as after g16_circuit_load_qap: every call that reads C takes it.  info_out (nullable)
 * receives the sizes, log2 of the domain and the entries of each matrix.  Afterwards g16_get_timings describes this call:
 * total_ms = the whole call, h2d_ms = the host walk, witness_map_ms = upload, decode and the host copies, h2d_bytes /
 * d2h_bytes, launches. */
typedef struct {
  uint32_t num_inputs, num_constraints, num_witness, log_n;
  uint64_t a_nnz, b_nnz, c_nnz;
} g16_r1cs_info;
int g16_r1cs_load(g16_ctx* ctx, int qap, const uint8_t* bytes, uint64_t len, g16_r1cs_info* info_out);

/* ---- circom / snarkjs .wtns witnesses, as this ABI's full assignment (ark-circom's read_witness).  `bytes` is a whole .wtns
 * (iden3 wtnsfile): "wtns", version u32 = 2, nSections u32, then {type u32, size u64, body} records; sections 1 and 2
 * exactly once each, others skipped.  1: n8 u32, prime (n8 bytes, the context's r), nWitness u32.  2: nWitness canonical
 * n8-byte values.  out receives nWitness Montgomery Fr (g16_fr_limbs each), decoded on the GPU (one thread per element
 * checks < r).  out == NULL writes the count only; cap (elements) below the count is G16_ERR_BAD_ARGUMENT with the count
 * in *count_out.  A bad file is G16_ERR_INVALID_DATA naming the problem or the first bad element ("witness[17] (byte 80):
 * not below r").  Needs no circuit and touches no resident state; element 0 and the length are g16_check_witness's
 * question. */
int g16_wtns_read(g16_ctx* ctx, const uint8_t* bytes, uint64_t len, uint64_t* out, uint64_t cap, uint64_t* count_out);

/* ---- snarkjs .ptau powers-of-tau transcripts, and proving keys from their Lagrange points (snarkjs `zkey new` on a
 * prepared file).  `bytes` is a whole .ptau (iden3 binary container): "ptau", version u32 = 1, nSections u32, then {id u32,
 * size u64, body} records in any order; integers little-endian; n8 = 8 g16_fq_limbs.  Points are affine Montgomery
 * little-endian, this ABI's limbs (all-zero bytes for the identity):
 *   1 header, exactly 12 + n8 bytes: n8 u32, q (n8 bytes, the context's base-field modulus), power u32, ceremonyPower u32
 *   2 tauG1 2^(power+1) - 1 points   3 tauG2 2^power   4 alphaTauG1 2^power   5 betaTauG1 2^power   6 betaG2 one point
 *   12..15 (prepared files, `powersoftau prepare phase2`): the Lagrange points of sections 2..5.  Level k holds the 2^k
 *     points (1/2^k) sum_{j<2^k} omega_k^(-ij) X_j over the first 2^k points of the source section, levels concatenated
 *     from k = 0 (level k starts at point 2^k - 1).  13..15 hold levels 0 .. power; 12 also holds level power + 1, formed
 *     from all of section 2 with entry 2^(power+1) - 1 taken as the identity: its odd entries are the CircomReduction H
 *     query at delta = 1.  For log_n < power, level log_n + 1 of section 12 is an interior level, taken over all 2n powers
 *     [tau^j], j < 2n (n = 2^log_n): its odd entries are the H query plus (omega_2n^(2i+1) / 2n) [tau^(2n-1)].
 * Sections 1..6 exactly once; 12..15 all four or none, each at most once; other ids (7: contributions) skipped.  When power
 * + 1 exceeds the scalar field's two-adicity (BN254 at power 28) level power + 1 cannot exist, and what snarkjs writes
 * there is unconfirmed: sections 12..15 are then not interpreted and the file reads as unprepared (prepared = 0).
 * g16_ptau_read copies the file's points into the caller's buffers on the host; nothing is decoded or checked on the device
 * (every call that takes the points checks them), no circuit is needed and no resident state is touched.  info receives
 * n8, power, ceremonyPower and prepared.  srs_out (nullable) receives the first *_len points of sections 2..5 (each at most
 * the file's length; a member of length 0 may be null) and betaG2: the result goes unchanged into g16_setup_from_srs,
 * g16_srs_verify_pairs (with the curve's generators), g16_srs_contribute and g16_pk_verify_pairs, so a circuit of domain n
 * needs only 2n - 1, n, n and n points.  lag_out (nullable; a null member is skipped) receives level log_n of sections
 * 12..15 (2^log_n points each) and, in tau_g1_h, the odd entries of level log_n + 1 of section 12 (2^log_n points; not
 * needed under LibsnarkReduction); the call sets lag_out->h_over_2n to 1 when that level is interior (log_n < power) and
 * to 0 when it is the top level (log_n = power).
 *   G16_ERR_INVALID_DATA: the section table (magic, version, truncation, trailing bytes, a missing or repeated section,
 *   only some of 12..15), the header (its size, n8, q, a power above 48) and every section size, g16_last_error() naming
 *   it ("section 14 holds 1234 bytes, 2^(power+1) - 1 points need 5678").
 *   G16_ERR_BAD_ARGUMENT: null bytes or info, a prefix longer than the file's member or a null member with a length,
 *   lag_out on a file that is not prepared, log_n above power.  Nothing is copied then; info is filled once the walk passed.
 * g16_setup_from_lagrange derives the key of the resident circuit under its reduction from the transcript prefixes `srs`
 * (g16_setup_from_srs's rules) and the level-log_n Lagrange points `lag` without any group transform: the key equals
 * g16_setup_from_srs on the same srs limb for limb (and so g16_setup(alpha, beta, 1, 1, tau, tau_g1[0], tau_g2[0])).  Every
 * point read is checked as g16_setup_from_srs checks it (a refusal names "lagrange.alpha_tau_g1[17]: point is not on the
 * curve").  Then, with z_i = rho^i (i < n) and z^ = iFFT_n(z) (n^-1 included), the call checks on the GPU, in one MSM per
 * side:
 *   sum_{i<n} rho^i lag.X[i] = sum_{j<n} z^_j srs.X[j]   for X = tau_g1, alpha_tau_g1, beta_tau_g1, tau_g2
 *   sum_{i<n} rho^i tau_g1_h[i] = sum_{j<m} w_j tau_g1[j],  w_j = omega_2n^(-j) z^_(j mod n) / 2   (G16_QAP_CIRCOM)
 * with m = 2n - 1, or m = 2n when lag->h_over_2n says tau_g1_h is taken over 2n powers (an interior level of section 12;
 * tau_g1 must then hold at least 2n points).
 * A member that differs from the inverse transform anywhere fails with probability at least 1 - (n - 1)/r over rho
 * (Schwartz-Zippel), given G16_SER_VALIDATE; without it the answer means nothing on a curve whose cofactor is not 1.  A
 * failed equation is G16_ERR_INVALID_DATA naming the member and level ("lagrange tau_g2 (level 2^14): not the inverse
 * transform of tau_g2[0, 16384)"); after it, as after a refused point, the circuit stays and no key is resident.  Then
 * the Lagrange points feed the sparse sums, the H query is tau_g1_h itself (G16_QAP_CIRCOM; with h_over_2n, tau_g1_h[i]
 * minus (omega_2n^(2i+1) / 2n) tau_g1[2n - 1], formed on the GPU) or [tau^(n+i)] - [tau^i] (G16_QAP_LIBSNARK), and the
 * key is made resident as g16_setup_from_srs makes it.  rho (Montgomery Fr, non-zero) is a
 * challenge the caller draws after the file is fixed.
 *   G16_ERR_BAD_ARGUMENT, with the previous key resident: g16_setup_from_srs's argument errors, a null lag, lag->log_n
 *   other than the circuit's log n, rho null or 0, a null lag member (tau_g1_h only under G16_QAP_CIRCOM).
 * Afterwards g16_get_timings describes this call: total_ms = the whole call, h2d_ms = upload and point checks,
 * witness_map_ms = the combination check (powers, transform, MSMs), msm_ms[0] = the H query, msm_ms[1] = the sparse sums. */
typedef struct { uint32_t n8, power, ceremony_power, prepared; } g16_ptau_info;
typedef struct {
  uint32_t log_n;          /* the level to copy: 2^log_n points per member */
  uint32_t h_over_2n;      /* written by the call: 1 when tau_g1_h comes from an interior level (log_n < power) */
  uint64_t* tau_g1; uint64_t* tau_g2; uint64_t* alpha_tau_g1; uint64_t* beta_tau_g1;   /* level log_n of sections 12..15 */
  uint64_t* tau_g1_h;      /* odd entries of level log_n + 1 of section 12 (2^log_n points) */
} g16_lagrange_out;
int g16_ptau_read(g16_ctx* ctx, const uint8_t* bytes, uint64_t len, const g16_srs_out* srs_out, g16_lagrange_out* lag_out,
                  g16_ptau_info* info);
typedef struct {
  uint32_t log_n;
  uint32_t h_over_2n;        /* tau_g1_h over 2n powers (g16_lagrange_out's h_over_2n); 0: over 2n - 1, the H query itself */
  const uint64_t* tau_g1; const uint64_t* tau_g2; const uint64_t* alpha_tau_g1; const uint64_t* beta_tau_g1;
  const uint64_t* tau_g1_h;  /* G16_QAP_CIRCOM only; may be null under G16_QAP_LIBSNARK */
} g16_lagrange_desc;
int g16_setup_from_lagrange(g16_ctx* ctx, const g16_srs_desc* srs, const g16_lagrange_desc* lag, const uint64_t* rho,
                            uint32_t flags);

/* g16_ptau_prepare is snarkjs `powersoftau prepare phase2` on the GPU: `in` is a whole .ptau of the context's curve, and
 * the output is the same file with sections 12..15 computed.  Level k of a member X holds the 2^k points (1/2^k)
 * sum_{j<2^k} omega_k^(-ij) X_j, X_j the identity for j >= len(X); 13..15 hold levels 0 .. power, 12 levels 0 .. power + 1
 * (the top one with the missing last power taken as the identity); level 0 is X_0.  The output is "ptau", version 1,
 * nSections; every section of `in` except 12..15 byte for byte in input order (7 and unknown ids included); then sections
 * 12, 13, 14 and 15.  Sections 12..15 of a prepared input are dropped and recomputed: the output never depends on them.
 * Affine limbs are canonical, so the output is a function of the input alone.
 * Size protocol as g16_pk_export_serialized: out = NULL writes the size to *len_out; cap below it is G16_ERR_BAD_ARGUMENT
 * with the size in *len_out; out must not overlap in.
 * Every point of sections 2..5 is checked on the GPU (canonical, on the curve, with G16_SER_VALIDATE also in the prime-order
 * subgroup; the identity is accepted) before anything is transformed or written.  A refused point is G16_ERR_INVALID_DATA,
 * g16_last_error() naming the first by member and index ("tau_g2[5]: point is not on the curve"), with nothing written to
 * out.  The call does not check that the file is a powers-of-tau transcript: g16_srs_verify_pairs does that.
 * Decided before any point is read, with nothing written:
 *   G16_ERR_INVALID_DATA: anything g16_ptau_read's walk refuses.
 *   G16_ERR_BAD_ARGUMENT: null in or len_out, flags other than 0 or G16_SER_VALIDATE, overlapping buffers, a proof in flight.
 *   G16_ERR_POLYNOMIAL_DEGREE_TOO_LARGE: power + 1 above the scalar field's two-adicity (BN254 at power 28), decided from
 *   section 1 before any other section's size is compared.
 *   G16_ERR_CUDA: a member's top level does not fit in the free device memory (its points, 2^top XYZZ points and 2^top
 *   affine points at once), g16_last_error() naming the member, the level, the bytes needed and the bytes free.
 * Each level is transformed whole on the device, one member at a time: the peak is about 2^(power+1) XYZZ tauG1 points
 * plus staging (BN254 at power 27: 32 GiB for that buffer).  No circuit or key is needed; the resident ones, and everything
 * derived from them, are left alone.  Afterwards g16_get_timings describes this call: total_ms, h2d_ms = the check pass,
 * msm_ms[0..3] = the transforms of tau_g1, tau_g2, alpha_tau_g1 and beta_tau_g1, h2d_bytes, d2h_bytes, launches; every
 * other field 0. */
int g16_ptau_prepare(g16_ctx* ctx, const uint8_t* in, uint64_t in_len, uint32_t flags, uint8_t* out, uint64_t cap,
                     uint64_t* len_out);

/* ---- proving: Groth16::create_proof_with_reduction_and_matrices, prover.rs:26-51
 *      = witness_map_from_matrices (r1cs_to_qap.rs:172-235) + create_proof_with_assignment (prover.rs:54-132).
 * r, s: Montgomery Fr.  full_assignment: (num_inputs + num_witness) Montgomery Fr, instance first.
 * proof_out: a (G1 affine) || b (G2 affine) || c (G1 affine) = 8*N64 limbs.  Needs circuit + key resident. */
int g16_prove(g16_ctx* ctx, const uint64_t* r, const uint64_t* s, const uint64_t* full_assignment, uint32_t flags,
              uint64_t* proof_out);

/* Sharded proving (world > 1): every rank computes its partial MSM sums, the host plumbing (torch.distributed /
 * NCCL all_gather of 5 points per rank) exchanges them, every rank assembles the same proof.
 * partial_out / partials: [h, l, a, b_g1] as G1 affine (4 * 2*N64 limbs) followed by b_g2 as G2 affine (g16_g2_limbs). */
int g16_prove_partial(g16_ctx* ctx, const uint64_t* r, const uint64_t* full_assignment, uint32_t flags,
                      uint64_t* partial_out);
int g16_prove_assemble(g16_ctx* ctx, const uint64_t* r, const uint64_t* s, const uint64_t* partials,
                       uint32_t nparts, uint64_t* proof_out);
/* Optional: start the (r, s)-only scalar multiplications of prover.rs:76,90,100,112 on a helper thread before the partial
 * sums exist; the next g16_prove_assemble with the same (r, s) picks the result up instead of computing it inline.
 * Loading a circuit or a key (g16_circuit_load, g16_pk_load, g16_setup, g16_pk_load_serialized, g16_setup_from_srs,
 * g16_setup_from_lagrange, g16_setup_contribute) discards the result. */
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
/* limbs per partial record: 4*2*N64 + g16_g2_limbs */
int g16_partial_limbs(const g16_ctx* ctx);

/* Batch proving (no reference counterpart: ark-groth16 proves one proof per call): `count` proofs of the resident circuit
 * under the resident key, one call.  Proof i is bit-identical to
 * g16_prove(ctx, r + F i, s + F i, full_assignments + F i nv, flags, proofs_out + P i), nv = num_inputs + num_witness,
 * F = g16_fr_limbs, P = the proof's limbs (8 N64, or 6 N64 on BW6-761).
 * r, s: count Montgomery Fr each.  full_assignments: count * nv Montgomery Fr (host, or device with
 * G16_ASSIGNMENT_ON_DEVICE).  proofs_out: count * P limbs.  group: at most this many proofs share one pass of the
 * kernels (0 = automatic: as many as fit); results never depend on it.  Sharded keys (world > 1) are refused, and so is a
 * call while a proof is in flight in either slot.  count == 0 returns G16_OK and touches nothing.  Afterwards
 * g16_get_timings describes the whole call: total_ms is its device span, msm_pairs / msm_entries are summed over the batch,
 * launches counts its kernels, host_finish_ms is the host time after the last group's GPU work. */
int g16_prove_batch(g16_ctx* ctx, uint32_t count, const uint64_t* r, const uint64_t* s, const uint64_t* full_assignments,
                    uint32_t group, uint32_t flags, uint64_t* proofs_out);

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
 * h_out receives domain_size Montgomery Fr coefficients (G16_QAP_CIRCOM: domain_size evaluations, see above). */
int g16_witness_map(g16_ctx* ctx, const uint64_t* full_assignment, uint32_t flags, uint64_t* h_out);

/* ---- R1CS satisfiability of assignments of the resident circuit: ark-relations ConstraintSystem::is_satisfied /
 * which_is_unsatisfied (ark-groth16 checks it only as debug_assert!, prover.rs:193).  A GPU pass over the resident
 * matrices, independent of the reduction (matrix C is read under G16_QAP_CIRCOM too, whose witness map never reads it).
 * Per assignment z:
 *   first_malformed   lowest j whose limbs, read as an integer, are >= r, or 0 when z[0] is not One (Montgomery R mod r);
 *                     G16_NONE if none.  When set, the rows are not evaluated: first_unsatisfied = G16_NONE and
 *                     num_unsatisfied = 0 (the field arithmetic assumes canonical inputs).
 *   first_unsatisfied lowest constraint i < num_constraints with <A_i,z> <B_i,z> != <C_i,z>, or G16_NONE.  Only the
 *                     constraints: the instance rows LibsnarkReduction appends are not checked.
 *   num_unsatisfied   how many constraints are unsatisfied.
 * g16_check_witness: `count` assignments of nv = num_inputs + num_witness Montgomery Fr each (host, or device with
 * G16_ASSIGNMENT_ON_DEVICE, the only flag it takes) -> reports_out[count].  Needs a resident circuit, no key.  Returns
 * G16_OK whatever the verdicts; an unknown flag, a null pointer, no circuit or a proof in flight in slot 0 is
 * G16_ERR_BAD_ARGUMENT; count == 0 returns G16_OK and touches nothing.  Runs on slot 0; host assignments are uploaded in
 * chunks bounded by the free device memory.  Results never depend on the chunking, the reduction or the options.
 *
 * G16_CHECK_WITNESS, a flag of g16_prove, g16_prove_submit, g16_prove_batch, g16_prove_partial (+ submit), g16_prove_sharded
 * (+ submit) and g16_witness_map, runs the same check on the device copy of the assignment, as one more kernel launch per
 * proof or batch group (g16_get_timings' launches grows by exactly 1; by one more per 65535 proofs of a group).  The check
 * never changes what else is enqueued: a rejected proof's GPU work, and a sharded proof's NCCL exchanges, run to completion,
 * and the slot is free after its wait.  The verdict is read where the results are collected (g16_prove_wait,
 * g16_prove_partial_wait, g16_prove_sharded_wait, the end of g16_prove_batch):
 *   single proof, partial, witness map: G16_ERR_UNSATISFIED and nothing written to proof_out / partial_out / h_out;
 *     g16_last_error() names the reason, e.g. "constraint 1234 unsatisfied (17 in all)" or "assignment element 5 is not a
 *     canonical Fr".
 *   batch: every proof is computed; a rejected proof's entry of proofs_out is all-zero limbs (three identity points, which
 *     never verify), every other entry is what the call without the flag writes.  The call returns G16_ERR_UNSATISFIED
 *     naming the lowest rejected proof and its reason ("proof 3: constraint 0 unsatisfied (1 in all)"); g16_check_witness
 *     gives every proof's report.
 * Without the flag nothing is launched or copied: outputs and launch counts are those of the call without it. */
#define G16_NONE UINT64_MAX
typedef struct {
  uint64_t first_unsatisfied;
  uint64_t num_unsatisfied;
  uint64_t first_malformed;
} g16_witness_report;
int g16_check_witness(g16_ctx* ctx, uint32_t count, const uint64_t* full_assignments, uint32_t flags,
                      g16_witness_report* reports_out);

/* ---- measurement hooks (bench.py) ---------------------------------------------------------------------------- */
typedef struct {
  float total_ms;        /* CUDA-event time of the last g16_prove / g16_prove_partial, first enqueue to last kernel */
  float h2d_ms;          /* assignment upload                                                                    */
  float witness_map_ms;  /* row evaluation + 7 NTTs (G16_QAP_CIRCOM: 6)                                             */
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
  int32_t reserved[4];
} g16_config;
int g16_get_config(const g16_ctx* ctx, g16_config* out);
/* Tuning options (INTEGRATION.md section 6) and the values each accepts:
 *   "msm_ne" 0 .. 32            "msm_c" 0 (automatic) .. 24          "msm_maxcopies" 1 .. 20
 *   "msm_ba", "msm_ba_g2" 0 .. 6                                      "ba_m" 1 .. 256          "ba_g" 1 .. 4096
 *   "ba_min_entries_g1", "ba_min_entries_g2" >= 0 (smallest MSM, in bucket entries, that runs the rounds)
 *   "acc_k0_g1", "acc_k0_g2" 0 (automatic) or 4 .. 1024               "acc_block" 32, 64 or 128
 *   "ba_inv_gcd", "ba_adaptive" (0 = exactly "msm_ba" rounds, 1 = fewer for sparsely filled buckets), "share_b_sort",
 *   "wm_split" 0 or 1           "wm_first" -1 (automatic), 0 or 1    "proof_slots" 1 or 2
 * "msm_ne", "msm_c" and "msm_maxcopies" take effect at the next g16_pk_load / g16_setup, the others from the next proof;
 * results never depend on them.  A value outside its set is refused with G16_ERR_BAD_ARGUMENT and changes nothing.
 * g16_ctx_create reads the environment variable G16_<KEY IN UPPER CASE> of every option; a value there that is not a
 * whole number in the option's set makes it fail with G16_ERR_BAD_ARGUMENT. */
int g16_set_option(g16_ctx* ctx, const char* key, int64_t value);
/* The value an option holds now (same keys; feeding it back to g16_set_option restores the option exactly). */
int g16_get_option(const g16_ctx* ctx, const char* key, int64_t* value);
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
