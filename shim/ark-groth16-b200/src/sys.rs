//! Raw bindings of include/g16b200.h (hand-written; tests/test_shim_abi.py checks every name and arity against the header
//! and against groth16_b200/_lib.py::SIGNATURES).  Types follow the header: plain pointers and sizes, no Rust types.
#![allow(non_camel_case_types, dead_code)]
use core::ffi::{c_char, c_int};

#[repr(C)]
pub struct g16_ctx {
    _private: [u8; 0],
}

pub const G16_CURVE_BLS12_381: c_int = 0;
pub const G16_CURVE_BN254: c_int = 1;
pub const G16_CURVE_BLS12_377: c_int = 2;
pub const G16_CURVE_BW6_761: c_int = 3;

pub const G16_OK: c_int = 0;
pub const G16_ERR_POLYNOMIAL_DEGREE_TOO_LARGE: c_int = 1;
pub const G16_ERR_BAD_ARGUMENT: c_int = 2;
pub const G16_ERR_CUDA: c_int = 3;
pub const G16_ERR_MALFORMED_KEY: c_int = 4;
pub const G16_ERR_INVALID_DATA: c_int = 5;
pub const G16_ERR_UNSATISFIED: c_int = 6;

pub const G16_SER_COMPRESSED: u32 = 1;
pub const G16_SER_VALIDATE: u32 = 2;

pub const G16_QAP_LIBSNARK: c_int = 0;
pub const G16_QAP_CIRCOM: c_int = 1;

pub const G16_ASSIGNMENT_ON_DEVICE: u32 = 1;
pub const G16_SERIAL_MSMS: u32 = 2;
pub const G16_CHECK_WITNESS: u32 = 4;

pub const G16_PK_UNCONTRIBUTED: u32 = 4;

pub const G16_NONE: u64 = u64::MAX;

pub const G16_ZKEY_KEY_ONLY: u32 = 16;

#[repr(C)]
#[derive(Default, Clone, Copy, Debug, PartialEq, Eq)]
pub struct g16_r1cs_info {
    pub num_inputs: u32,
    pub num_constraints: u32,
    pub num_witness: u32,
    pub log_n: u32,
    pub a_nnz: u64,
    pub b_nnz: u64,
    pub c_nnz: u64,
}

#[repr(C)]
#[derive(Default, Clone, Copy, Debug, PartialEq, Eq)]
pub struct g16_zkey_info {
    pub num_inputs: u32,
    pub num_constraints: u32,
    pub num_witness: u32,
    pub log_n: u32,
    pub a_nnz: u64,
    pub b_nnz: u64,
}

#[repr(C)]
#[derive(Default, Clone, Copy, Debug, PartialEq, Eq)]
pub struct g16_witness_report {
    pub first_unsatisfied: u64,
    pub num_unsatisfied: u64,
    pub first_malformed: u64,
}

#[repr(C)]
pub struct g16_csr {
    pub row_ptr: *const u32,
    pub col: *const u32,
    pub val: *const u64,
}

#[repr(C)]
pub struct g16_pk_desc {
    pub a_query: *const u64,
    pub a_len: u64,
    pub b_g1_query: *const u64,
    pub b_g1_len: u64,
    pub b_g2_query: *const u64,
    pub b_g2_len: u64,
    pub h_query: *const u64,
    pub h_len: u64,
    pub l_query: *const u64,
    pub l_len: u64,
    pub alpha_g1: *const u64,
    pub beta_g1: *const u64,
    pub delta_g1: *const u64,
    pub beta_g2: *const u64,
    pub delta_g2: *const u64,
}

/// g16_srs_desc: a powers-of-tau transcript, affine Montgomery limbs (g16_setup_from_srs)
#[repr(C)]
pub struct g16_srs_desc {
    pub tau_g1: *const u64,
    pub tau_g1_len: u64,
    pub tau_g2: *const u64,
    pub tau_g2_len: u64,
    pub alpha_tau_g1: *const u64,
    pub alpha_tau_g1_len: u64,
    pub beta_tau_g1: *const u64,
    pub beta_tau_g1_len: u64,
    pub beta_g2: *const u64,
}

/// g16_srs_out: where g16_srs_from_secrets writes a transcript
#[repr(C)]
pub struct g16_srs_out {
    pub tau_g1: *mut u64,
    pub tau_g1_len: u64,
    pub tau_g2: *mut u64,
    pub tau_g2_len: u64,
    pub alpha_tau_g1: *mut u64,
    pub alpha_tau_g1_len: u64,
    pub beta_tau_g1: *mut u64,
    pub beta_tau_g1_len: u64,
    pub beta_g2: *mut u64,
}

/// g16_ptau_info: the header of a snarkjs .ptau file (g16_ptau_read)
#[repr(C)]
#[derive(Default, Clone, Copy, Debug, PartialEq, Eq)]
pub struct g16_ptau_info {
    pub n8: u32,
    pub power: u32,
    pub ceremony_power: u32,
    pub prepared: u32,
}

/// g16_lagrange_out: where g16_ptau_read writes one level of a prepared file's Lagrange points
#[repr(C)]
pub struct g16_lagrange_out {
    pub log_n: u32,
    pub h_over_2n: u32,
    pub tau_g1: *mut u64,
    pub tau_g2: *mut u64,
    pub alpha_tau_g1: *mut u64,
    pub beta_tau_g1: *mut u64,
    pub tau_g1_h: *mut u64,
}

/// g16_lagrange_desc: one level of Lagrange points (g16_setup_from_lagrange)
#[repr(C)]
pub struct g16_lagrange_desc {
    pub log_n: u32,
    pub h_over_2n: u32,
    pub tau_g1: *const u64,
    pub tau_g2: *const u64,
    pub alpha_tau_g1: *const u64,
    pub beta_tau_g1: *const u64,
    pub tau_g1_h: *const u64,
}

#[repr(C)]
pub struct g16_pk_export_desc {
    pub a_query: *mut u64,
    pub b_g1_query: *mut u64,
    pub b_g2_query: *mut u64,
    pub h_query: *mut u64,
    pub l_query: *mut u64,
    pub alpha_g1: *mut u64,
    pub beta_g1: *mut u64,
    pub delta_g1: *mut u64,
    pub beta_g2: *mut u64,
    pub gamma_g2: *mut u64,
    pub delta_g2: *mut u64,
    pub gamma_abc_g1: *mut u64,
}

#[repr(C)]
pub struct g16_pk_check_desc {
    pub a_query: *const u64,
    pub b_g1_query: *const u64,
    pub b_g2_query: *const u64,
    pub h_query: *const u64,
    pub l_query: *const u64,
    pub alpha_g1: *const u64,
    pub beta_g1: *const u64,
    pub delta_g1: *const u64,
    pub beta_g2: *const u64,
    pub gamma_g2: *const u64,
    pub delta_g2: *const u64,
    pub gamma_abc_g1: *const u64,
}

#[repr(C)]
pub struct g16_pk_delta_desc {
    pub h_query: *const u64,
    pub h_len: u64,
    pub l_query: *const u64,
    pub l_len: u64,
    pub delta_g1: *const u64,
    pub delta_g2: *const u64,
}

#[repr(C)]
pub struct g16_pk_delta_out {
    pub h_query: *mut u64,
    pub h_len: u64,
    pub l_query: *mut u64,
    pub l_len: u64,
    pub delta_g1: *mut u64,
    pub delta_g2: *mut u64,
}

/// One contribution's public record; r_g2 is recomputed by the checker from the ceremony's transcript, never taken from
/// the contributor.
#[repr(C)]
pub struct g16_contribution_record {
    pub after_g1: *const u64,
    pub s_g1: *const u64,
    pub s_x_g1: *const u64,
    pub r_g2: *const u64,
    pub r_x_g2: *const u64,
}

#[repr(C)]
#[derive(Default, Clone, Copy)]
pub struct g16_timings {
    pub total_ms: f32,
    pub h2d_ms: f32,
    pub witness_map_ms: f32,
    pub msm_ms: [f32; 5],
    pub msm_accum_ms: [f32; 5],
    pub host_finish_ms: f32,
    pub msm_pairs: [u64; 5],
    pub msm_entries: [u64; 5],
    pub launches: u64,
    pub h2d_bytes: u64,
    pub d2h_bytes: u64,
    pub msm_begin_ms: [f32; 5],
    pub msm_end_ms: [f32; 5],
}

#[repr(C)]
#[derive(Default, Clone, Copy)]
pub struct g16_config {
    pub c: i32,
    pub ne: i32,
    pub copies: i32,
    pub k0_g1: i32,
    pub k0_g2: i32,
    pub ba_rounds_g1: i32,
    pub ba_rounds_g2: i32,
    pub ba_m: i32,
    pub ba_g: i32,
    pub ba_inv_gcd: i32,
    pub acc_block: i32,
    pub sm_count: i32,
    pub rank: i32,
    pub world: i32,
    pub reserved: [i32; 4],
}

extern "C" {
    pub fn g16_ctx_create(curve: c_int, device: c_int, out: *mut *mut g16_ctx) -> c_int;
    pub fn g16_ctx_destroy(ctx: *mut g16_ctx);
    pub fn g16_last_error() -> *const c_char;
    pub fn g16_fq_limbs(ctx: *const g16_ctx) -> c_int;
    pub fn g16_fr_limbs(ctx: *const g16_ctx) -> c_int;
    pub fn g16_g2_limbs(ctx: *const g16_ctx) -> c_int;
    pub fn g16_partial_limbs(ctx: *const g16_ctx) -> c_int;
    pub fn g16_domain_log(ctx: *const g16_ctx) -> u32;
    pub fn g16_ntt(ctx: *mut g16_ctx, log_n: u32, inverse: c_int, coset: c_int, inout: *mut u64) -> c_int;
    pub fn g16_witness_map_evals(ctx: *mut g16_ctx, log_n: u32, a: *const u64, b: *const u64, c: *const u64, h_out: *mut u64) -> c_int;
    pub fn g16_msm_g1(ctx: *mut g16_ctx, bases: *const u64, scalars: *const u64, n: u64, out_xyz: *mut u64) -> c_int;
    pub fn g16_msm_g2(ctx: *mut g16_ctx, bases: *const u64, scalars: *const u64, n: u64, out_xyz: *mut u64) -> c_int;
    pub fn g16_circuit_load(ctx: *mut g16_ctx, num_inputs: u32, num_constraints: u32, num_witness: u32, a: *const g16_csr, b: *const g16_csr, c: *const g16_csr) -> c_int;
    pub fn g16_circuit_load_qap(ctx: *mut g16_ctx, qap: c_int, num_inputs: u32, num_constraints: u32, num_witness: u32, a: *const g16_csr, b: *const g16_csr, c: *const g16_csr) -> c_int;
    pub fn g16_pk_load(ctx: *mut g16_ctx, pk: *const g16_pk_desc, rank: u32, world: u32) -> c_int;
    pub fn g16_setup(ctx: *mut g16_ctx, alpha: *const u64, beta: *const u64, gamma: *const u64, delta: *const u64, tau: *const u64, g1: *const u64, g2: *const u64) -> c_int;
    pub fn g16_pk_export(ctx: *mut g16_ctx, out: *const g16_pk_export_desc) -> c_int;
    pub fn g16_setup_from_srs(ctx: *mut g16_ctx, srs: *const g16_srs_desc, flags: u32) -> c_int;
    pub fn g16_setup_contribute(ctx: *mut g16_ctx, delta: *const u64) -> c_int;
    pub fn g16_srs_from_secrets(ctx: *mut g16_ctx, tau: *const u64, alpha: *const u64, beta: *const u64, g1: *const u64, g2: *const u64, out: *const g16_srs_out) -> c_int;
    pub fn g16_srs_contribute(ctx: *mut g16_ctx, srs_in: *const g16_srs_desc, tau: *const u64, alpha: *const u64, beta: *const u64, flags: u32, chunk_points: u64, out: *const g16_srs_out) -> c_int;
    pub fn g16_srs_verify_pairs(ctx: *mut g16_ctx, srs: *const g16_srs_desc, g1: *const u64, g2: *const u64, rho: *const u64, flags: u32, chunk_points: u64, pairs_g1: *mut u64, pairs_g2: *mut u64) -> c_int;
    pub fn g16_pk_verify_pairs(ctx: *mut g16_ctx, srs: *const g16_srs_desc, pk: *const g16_pk_check_desc, rho: *const u64, flags: u32, pairs_g1: *mut u64, pairs_g2: *mut u64) -> c_int;
    pub fn g16_pk_contribute(ctx: *mut g16_ctx, input: *const g16_pk_delta_desc, delta: *const u64, flags: u32, chunk_points: u64, out: *const g16_pk_delta_out) -> c_int;
    pub fn g16_contribution_chain_pairs(ctx: *mut g16_ctx, start_g1: *const u64, end_g1: *const u64, records: *const g16_contribution_record, count: u32, flags: u32, pairs_g1: *mut u64, pairs_g2: *mut u64) -> c_int;
    pub fn g16_pk_load_serialized(ctx: *mut g16_ctx, bytes: *const u8, len: u64, flags: u32, rank: u32, world: u32, vk_out: *const g16_pk_export_desc) -> c_int;
    pub fn g16_zkey_load(ctx: *mut g16_ctx, bytes: *const u8, len: u64, flags: u32, rank: u32, world: u32, vk_out: *const g16_pk_export_desc, info_out: *mut g16_zkey_info) -> c_int;
    pub fn g16_r1cs_load(ctx: *mut g16_ctx, qap: c_int, bytes: *const u8, len: u64, info_out: *mut g16_r1cs_info) -> c_int;
    pub fn g16_wtns_read(ctx: *mut g16_ctx, bytes: *const u8, len: u64, out: *mut u64, cap: u64, count_out: *mut u64) -> c_int;
    pub fn g16_ptau_read(ctx: *mut g16_ctx, bytes: *const u8, len: u64, srs_out: *const g16_srs_out, lag_out: *mut g16_lagrange_out, info: *mut g16_ptau_info) -> c_int;
    pub fn g16_setup_from_lagrange(ctx: *mut g16_ctx, srs: *const g16_srs_desc, lag: *const g16_lagrange_desc, rho: *const u64, flags: u32) -> c_int;
    pub fn g16_ptau_prepare(ctx: *mut g16_ctx, input: *const u8, in_len: u64, flags: u32, out: *mut u8, cap: u64, len_out: *mut u64) -> c_int;
    pub fn g16_pk_export_serialized(ctx: *mut g16_ctx, flags: u32, out: *mut u8, cap: u64, len_out: *mut u64) -> c_int;
    pub fn g16_prove(ctx: *mut g16_ctx, r: *const u64, s: *const u64, full_assignment: *const u64, flags: u32, proof_out: *mut u64) -> c_int;
    pub fn g16_prove_partial(ctx: *mut g16_ctx, r: *const u64, full_assignment: *const u64, flags: u32, partial_out: *mut u64) -> c_int;
    pub fn g16_prove_assemble(ctx: *mut g16_ctx, r: *const u64, s: *const u64, partials: *const u64, nparts: u32, proof_out: *mut u64) -> c_int;
    pub fn g16_prove_assemble_prepare(ctx: *mut g16_ctx, r: *const u64, s: *const u64) -> c_int;
    pub fn g16_prove_submit(ctx: *mut g16_ctx, slot: c_int, r: *const u64, s: *const u64, full_assignment: *const u64, flags: u32) -> c_int;
    pub fn g16_prove_wait(ctx: *mut g16_ctx, slot: c_int, proof_out: *mut u64) -> c_int;
    pub fn g16_prove_batch(ctx: *mut g16_ctx, count: u32, r: *const u64, s: *const u64, full_assignments: *const u64, group: u32, flags: u32, proofs_out: *mut u64) -> c_int;
    pub fn g16_prove_partial_submit(ctx: *mut g16_ctx, slot: c_int, r: *const u64, full_assignment: *const u64, flags: u32) -> c_int;
    pub fn g16_prove_partial_wait(ctx: *mut g16_ctx, slot: c_int, partial_out: *mut u64) -> c_int;
    pub fn g16_comm_unique_id(out128: *mut u8) -> c_int;
    pub fn g16_comm_init(ctx: *mut g16_ctx, id128: *const u8, rank: u32, world: u32) -> c_int;
    pub fn g16_prove_sharded(ctx: *mut g16_ctx, r: *const u64, s: *const u64, full_assignment: *const u64, flags: u32, proof_out: *mut u64) -> c_int;
    pub fn g16_prove_sharded_submit(ctx: *mut g16_ctx, slot: c_int, r: *const u64, s: *const u64, full_assignment: *const u64, flags: u32) -> c_int;
    pub fn g16_prove_sharded_wait(ctx: *mut g16_ctx, slot: c_int, proof_out: *mut u64) -> c_int;
    pub fn g16_witness_map(ctx: *mut g16_ctx, full_assignment: *const u64, flags: u32, h_out: *mut u64) -> c_int;
    pub fn g16_check_witness(ctx: *mut g16_ctx, count: u32, full_assignments: *const u64, flags: u32, reports_out: *mut g16_witness_report) -> c_int;
    pub fn g16_get_timings(ctx: *const g16_ctx, out: *mut g16_timings) -> c_int;
    pub fn g16_synthetic_r1cs(curve: c_int, log_n: u32, seed: u64, a_col: *mut u32, a_val: *mut u64, b_col: *mut u32, c_col: *mut u32, full_assignment: *mut u64) -> c_int;
    pub fn g16_get_config(ctx: *const g16_ctx, out: *mut g16_config) -> c_int;
    pub fn g16_set_option(ctx: *mut g16_ctx, key: *const c_char, value: i64) -> c_int;
    pub fn g16_get_option(ctx: *const g16_ctx, key: *const c_char, value: *mut i64) -> c_int;
}
