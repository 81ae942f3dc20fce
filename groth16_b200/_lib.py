"""ctypes binding of libg16b200.so (include/g16b200.h).  No fallback: a missing library or GPU raises."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libg16b200.so")

u64p = C.POINTER(C.c_uint64)
u32p = C.POINTER(C.c_uint32)


class Csr(C.Structure):
    _fields_ = [("row_ptr", u32p), ("col", u32p), ("val", u64p)]


class PkDesc(C.Structure):
    _fields_ = [("a_query", u64p), ("a_len", C.c_uint64), ("b_g1_query", u64p), ("b_g1_len", C.c_uint64),
                ("b_g2_query", u64p), ("b_g2_len", C.c_uint64), ("h_query", u64p), ("h_len", C.c_uint64),
                ("l_query", u64p), ("l_len", C.c_uint64), ("alpha_g1", u64p), ("beta_g1", u64p),
                ("delta_g1", u64p), ("beta_g2", u64p), ("delta_g2", u64p)]


class PkExportDesc(C.Structure):
    _fields_ = [(n, u64p) for n in ("a_query", "b_g1_query", "b_g2_query", "h_query", "l_query", "alpha_g1",
                                    "beta_g1", "delta_g1", "beta_g2", "gamma_g2", "delta_g2", "gamma_abc_g1")]


class PkCheckDesc(C.Structure):
    _fields_ = PkExportDesc._fields_


class SrsDesc(C.Structure):
    _fields_ = [("tau_g1", u64p), ("tau_g1_len", C.c_uint64), ("tau_g2", u64p), ("tau_g2_len", C.c_uint64),
                ("alpha_tau_g1", u64p), ("alpha_tau_g1_len", C.c_uint64), ("beta_tau_g1", u64p),
                ("beta_tau_g1_len", C.c_uint64), ("beta_g2", u64p)]


class SrsOut(C.Structure):
    _fields_ = SrsDesc._fields_


class PkDeltaDesc(C.Structure):
    _fields_ = [("h_query", u64p), ("h_len", C.c_uint64), ("l_query", u64p), ("l_len", C.c_uint64), ("delta_g1", u64p),
                ("delta_g2", u64p)]


class PkDeltaOut(C.Structure):
    _fields_ = PkDeltaDesc._fields_


class ContributionRecord(C.Structure):
    _fields_ = [(n, u64p) for n in ("after_g1", "s_g1", "s_x_g1", "r_g2", "r_x_g2")]


class Timings(C.Structure):
    _fields_ = [("total_ms", C.c_float), ("h2d_ms", C.c_float), ("witness_map_ms", C.c_float),
                ("msm_ms", C.c_float * 5), ("msm_accum_ms", C.c_float * 5), ("host_finish_ms", C.c_float),
                ("msm_pairs", C.c_uint64 * 5), ("msm_entries", C.c_uint64 * 5), ("launches", C.c_uint64),
                ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64), ("msm_begin_ms", C.c_float * 5), ("msm_end_ms", C.c_float * 5)]


class Config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("c", "ne", "copies", "k0_g1", "k0_g2", "ba_rounds_g1", "ba_rounds_g2", "ba_m", "ba_g",
                                         "ba_inv_gcd", "acc_block", "sm_count", "rank", "world")] + [("reserved", C.c_int32 * 4)]


class ZkeyInfo(C.Structure):
    _fields_ = [("num_inputs", C.c_uint32), ("num_constraints", C.c_uint32), ("num_witness", C.c_uint32), ("log_n", C.c_uint32),
                ("a_nnz", C.c_uint64), ("b_nnz", C.c_uint64)]


class R1csInfo(C.Structure):
    _fields_ = [("num_inputs", C.c_uint32), ("num_constraints", C.c_uint32), ("num_witness", C.c_uint32), ("log_n", C.c_uint32),
                ("a_nnz", C.c_uint64), ("b_nnz", C.c_uint64), ("c_nnz", C.c_uint64)]


class PtauInfo(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("n8", "power", "ceremony_power", "prepared")]


class LagrangeOut(C.Structure):
    _fields_ = [("log_n", C.c_uint32), ("h_over_2n", C.c_uint32)] + [(n, u64p) for n in ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1", "tau_g1_h")]


class LagrangeDesc(C.Structure):
    _fields_ = LagrangeOut._fields_


class WitnessReport(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("first_unsatisfied", "num_unsatisfied", "first_malformed")]


# every symbol include/g16b200.h declares: (name, restype, argtypes)
SIGNATURES = [
    ("g16_ctx_create", C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    ("g16_ctx_destroy", None, [C.c_void_p]),
    ("g16_last_error", C.c_char_p, []),
    ("g16_fq_limbs", C.c_int, [C.c_void_p]),
    ("g16_fr_limbs", C.c_int, [C.c_void_p]),
    ("g16_g2_limbs", C.c_int, [C.c_void_p]),
    ("g16_partial_limbs", C.c_int, [C.c_void_p]),
    ("g16_domain_log", C.c_uint32, [C.c_void_p]),
    ("g16_ntt", C.c_int, [C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_void_p]),
    ("g16_witness_map_evals", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("g16_msm_g1", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    ("g16_msm_g2", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    ("g16_circuit_load", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(Csr), C.POINTER(Csr), C.POINTER(Csr)]),
    ("g16_circuit_load_qap", C.c_int, [C.c_void_p, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(Csr), C.POINTER(Csr),
                                       C.POINTER(Csr)]),
    ("g16_pk_load", C.c_int, [C.c_void_p, C.POINTER(PkDesc), C.c_uint32, C.c_uint32]),
    ("g16_setup", C.c_int, [C.c_void_p] + [C.c_void_p] * 7),
    ("g16_pk_export", C.c_int, [C.c_void_p, C.POINTER(PkExportDesc)]),
    ("g16_setup_from_srs", C.c_int, [C.c_void_p, C.POINTER(SrsDesc), C.c_uint32]),
    ("g16_setup_contribute", C.c_int, [C.c_void_p, C.c_void_p]),
    ("g16_srs_from_secrets", C.c_int, [C.c_void_p] + [C.c_void_p] * 5 + [C.POINTER(SrsOut)]),
    ("g16_srs_contribute", C.c_int, [C.c_void_p, C.POINTER(SrsDesc)] + [C.c_void_p] * 3 + [C.c_uint32, C.c_uint64,
                                                                                          C.POINTER(SrsOut)]),
    ("g16_srs_verify_pairs", C.c_int, [C.c_void_p, C.POINTER(SrsDesc)] + [C.c_void_p] * 3 + [C.c_uint32, C.c_uint64]
     + [C.c_void_p] * 2),
    ("g16_pk_verify_pairs", C.c_int, [C.c_void_p, C.POINTER(SrsDesc), C.POINTER(PkCheckDesc), C.c_void_p, C.c_uint32]
     + [C.c_void_p] * 2),
    ("g16_pk_contribute", C.c_int, [C.c_void_p, C.POINTER(PkDeltaDesc), C.c_void_p, C.c_uint32, C.c_uint64,
                                    C.POINTER(PkDeltaOut)]),
    ("g16_contribution_chain_pairs", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(ContributionRecord), C.c_uint32,
                                               C.c_uint32, C.c_void_p, C.c_void_p]),
    ("g16_pk_load_serialized", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32,
                                         C.POINTER(PkExportDesc)]),
    ("g16_zkey_load", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(PkExportDesc),
                                C.POINTER(ZkeyInfo)]),
    ("g16_r1cs_load", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_uint64, C.POINTER(R1csInfo)]),
    ("g16_wtns_read", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]),
    ("g16_ptau_read", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(SrsOut), C.POINTER(LagrangeOut), C.POINTER(PtauInfo)]),
    ("g16_setup_from_lagrange", C.c_int, [C.c_void_p, C.POINTER(SrsDesc), C.POINTER(LagrangeDesc), C.c_void_p, C.c_uint32]),
    ("g16_ptau_prepare", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]),
    ("g16_pk_export_serialized", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]),
    ("g16_prove", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]),
    ("g16_prove_partial", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]),
    ("g16_prove_assemble", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]),
    ("g16_prove_assemble_prepare", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    ("g16_prove_submit", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]),
    ("g16_prove_wait", C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    ("g16_prove_batch", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]),
    ("g16_prove_partial_submit", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_uint32]),
    ("g16_prove_partial_wait", C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    ("g16_witness_map", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]),
    ("g16_check_witness", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(WitnessReport)]),
    ("g16_get_timings", C.c_int, [C.c_void_p, C.POINTER(Timings)]),
    ("g16_comm_unique_id", C.c_int, [C.c_void_p]),
    ("g16_comm_init", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32]),
    ("g16_prove_sharded", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]),
    ("g16_prove_sharded_submit", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]),
    ("g16_prove_sharded_wait", C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    ("g16_synthetic_r1cs", C.c_int, [C.c_int, C.c_uint32, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("g16_get_config", C.c_int, [C.c_void_p, C.POINTER(Config)]),
    ("g16_set_option", C.c_int, [C.c_void_p, C.c_char_p, C.c_int64]),
    ("g16_get_option", C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_int64)]),
]

G16_OK = 0
ERR_POLYNOMIAL_DEGREE_TOO_LARGE = 1
ERR_BAD_ARGUMENT = 2
ERR_CUDA = 3
ERR_MALFORMED_KEY = 4
ERR_INVALID_DATA = 5
ERR_UNSATISFIED = 6
SER_COMPRESSED = 1
SER_VALIDATE = 2
ASSIGNMENT_ON_DEVICE = 1
SERIAL_MSMS = 2
CHECK_WITNESS = 4
PK_UNCONTRIBUTED = 4   # a flag of g16_pk_verify_pairs
ZKEY_KEY_ONLY = 16     # a flag of g16_zkey_load
NONE = (1 << 64) - 1   # G16_NONE
QAP_LIBSNARK = 0
QAP_CIRCOM = 1
QAPS = {"libsnark": QAP_LIBSNARK, "circom": QAP_CIRCOM}

_lib = None


def load():
    """Load libg16b200.so; raises (never falls back) when the CUDA extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(there is no CPU fallback)")
        lib = C.CDLL(LIB_PATH)
        for name, res, args in SIGNATURES:
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def last_error() -> str:
    return load().g16_last_error().decode(errors="replace")
