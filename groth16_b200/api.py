"""Host-side mirror of ark-groth16's proving interface over the C ABI of libg16b200.so.

Names, argument meaning and error behaviour follow /root/reference:
  Groth16.create_proof_with_reduction_and_matrices  <- prover.rs:26-51
  Groth16.generate_parameters_with_qap              <- generator.rs:47-208 (explicit toxic waste)
  ProvingKey / VerifyingKey / Proof                 <- data_structures.rs:9-16,32-47,126-143
  ConstraintMatrices                                <- ark-relations `ConstraintMatrices` as consumed at r1cs_to_qap.rs:172-218
  SynthesisError variants                           <- r1cs_to_qap.rs:134,179 ; verifier.rs:30
Field elements cross this layer as numpy uint64 limb arrays in Montgomery form (codec.py converts Python ints).
The Rust shim a maintainer would write against the same symbols is in INTEGRATION.md.
"""
from __future__ import annotations

import ctypes as C
import secrets
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from .codec import CurveCodec
from .params import GENERATORS, CurveParams, get_curve
from .serialize import DeserializeError


class SynthesisError(Exception):
    """ark_relations::r1cs::SynthesisError"""


class PolynomialDegreeTooLarge(SynthesisError):
    pass


class MalformedKey(SynthesisError):
    pass


class Unsatisfiable(SynthesisError):
    """SynthesisError::Unsatisfiable: CHECK_WITNESS refused an assignment; the message names the constraint or element"""


class CudaError(RuntimeError):
    pass


def _check(rc: int):
    if rc == _lib.G16_OK:
        return
    msg = _lib.last_error()
    if rc == _lib.ERR_POLYNOMIAL_DEGREE_TOO_LARGE:
        raise PolynomialDegreeTooLarge(msg)
    if rc == _lib.ERR_MALFORMED_KEY:
        raise MalformedKey(msg)
    if rc == _lib.ERR_CUDA:
        raise CudaError(msg)
    if rc == _lib.ERR_INVALID_DATA:
        raise DeserializeError(msg)
    if rc == _lib.ERR_UNSATISFIED:
        raise Unsatisfiable(msg)
    raise ValueError(msg)


def _zkey_num_inputs(data: bytes, nq: int) -> int:
    """nPublic + 1 from section 2 of a .zkey, found by walking the section table; 1 when the file is too broken to say
    (the C side then refuses it before writing anything)"""
    mv = memoryview(data)
    if len(mv) < 12:
        return 1
    pos, nsec = 12, int.from_bytes(mv[8:12], "little")
    for _ in range(nsec):
        if len(mv) - pos < 12:
            return 1
        sid, size = int.from_bytes(mv[pos:pos + 4], "little"), int.from_bytes(mv[pos + 4:pos + 12], "little")
        pos += 12
        if sid == 2 and size >= 4:
            n8q = int.from_bytes(mv[pos:pos + 4], "little")
            if n8q != 8 * nq or size < 8 + n8q:
                return 1
            n8r = int.from_bytes(mv[pos + 4 + n8q:pos + 8 + n8q], "little")
            f = pos + 8 + n8q + n8r
            if size < f + 8 - pos:
                return 1
            return int.from_bytes(mv[f + 4:f + 8], "little") + 1
        pos += size
    return 1


def _zkey_host_refusal() -> bool:
    """the last g16_zkey_load failure was decided on the host, before the resident circuit and key were released"""
    msg = _lib.last_error()
    return not (msg.startswith("coefficient") or "(byte " in msg or "is not the domain of the circuit" in msg)


def _ptr(a: Optional[np.ndarray]):
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"] and a.dtype == np.uint64
    return a.ctypes.data_as(C.c_void_p)


def _u64p(a: Optional[np.ndarray]):
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"] and a.dtype == np.uint64
    return a.ctypes.data_as(_lib.u64p)


def _u32p(a: np.ndarray):
    assert a.flags["C_CONTIGUOUS"] and a.dtype == np.uint32
    return a.ctypes.data_as(_lib.u32p)


@dataclass
class ConstraintMatrices:
    """CSR form of ark-relations' ConstraintMatrices (rows of (coeff, column); column < num_instance_variables is an
    instance variable, otherwise witness index + num_instance_variables)."""
    num_instance_variables: int
    num_witness_variables: int
    num_constraints: int
    a: Tuple[np.ndarray, np.ndarray, np.ndarray]  # row_ptr u32 [nc+1], col u32 [nnz], val u64 [nnz,4] Montgomery
    b: Tuple[np.ndarray, np.ndarray, np.ndarray]
    c: Tuple[np.ndarray, np.ndarray, np.ndarray]

    @staticmethod
    def from_rows(curve, num_instance: int, num_witness: int, a_rows, b_rows, c_rows) -> "ConstraintMatrices":
        cd = CurveCodec(get_curve(curve))

        def csr(rows):
            rp = np.zeros(len(rows) + 1, dtype=np.uint32)
            cols, vals = [], []
            for i, row in enumerate(rows):
                for cf, idx in row:
                    cols.append(idx)
                    vals.append(cf)
                rp[i + 1] = len(cols)
            col = np.asarray(cols, dtype=np.uint32)
            val = cd.fr.enc(vals) if vals else np.zeros((0, cd.fr.nl), dtype=np.uint64)
            return rp, col, np.ascontiguousarray(val)

        return ConstraintMatrices(num_instance, num_witness, len(a_rows), csr(a_rows), csr(b_rows), csr(c_rows))


@dataclass
class ZkeyCircuit:
    """The circuit g16_zkey_load derived from a .zkey and made resident (A and B on the GPU only; a .zkey has no C).  Its
    sizes stand in for ConstraintMatrices wherever the resident circuit's sizes are needed."""
    num_instance_variables: int
    num_constraints: int
    num_witness_variables: int
    log_n: int
    a_nnz: int
    b_nnz: int


@dataclass
class R1csCircuit:
    """The circuit g16_r1cs_load read from a circom .r1cs and made resident with all three matrices (on the GPU, and host
    copies for the setup calls).  Its sizes stand in for ConstraintMatrices wherever the resident circuit's sizes are
    needed."""
    num_instance_variables: int
    num_constraints: int
    num_witness_variables: int
    log_n: int
    a_nnz: int
    b_nnz: int
    c_nnz: int


@dataclass
class VerifyingKey:
    alpha_g1: np.ndarray
    beta_g2: np.ndarray
    gamma_g2: Optional[np.ndarray]
    delta_g2: np.ndarray
    gamma_abc_g1: Optional[np.ndarray]


@dataclass
class ProvingKey:
    vk: VerifyingKey
    beta_g1: np.ndarray
    delta_g1: np.ndarray
    a_query: np.ndarray
    b_g1_query: np.ndarray
    b_g2_query: np.ndarray
    h_query: np.ndarray
    l_query: np.ndarray


@dataclass
class Srs:
    """A powers-of-tau transcript (phase 1 of a Groth16 ceremony) as affine Montgomery limbs, identity = all-zero limbs:
    tau_g1[i] = [tau^i]G1, tau_g2[i] = [tau^i]G2, alpha_tau_g1[i] = [alpha tau^i]G1, beta_tau_g1[i] = [beta tau^i]G1,
    beta_g2 = [beta]G2.  A circuit with domain size n needs at least 2n - 1, n, n and n points."""
    tau_g1: np.ndarray
    tau_g2: np.ndarray
    alpha_tau_g1: np.ndarray
    beta_tau_g1: np.ndarray
    beta_g2: np.ndarray


SRS_VECTORS = ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1")


@dataclass
class Lagrange:
    """One level of a prepared .ptau file's Lagrange points as affine Montgomery limbs: for the domain of n = 2^log_n points,
    tau_g1[i] = [L_i(tau)]G1, tau_g2[i] = [L_i(tau)]G2, alpha_tau_g1[i] = [alpha L_i(tau)]G1, beta_tau_g1[i] = [beta
    L_i(tau)]G1 (i < n), and tau_g1_h the odd entries of level log_n + 1 (None when not read, as under LibsnarkReduction):
    the CircomReduction H query at delta = 1 when that level is the file's top one, and with h_over_2n (an interior level,
    taken over 2n powers) that query plus (omega_2n^(2i+1) / 2n) [tau^(2n-1)], which the key setup takes off."""
    log_n: int
    tau_g1: np.ndarray
    tau_g2: np.ndarray
    alpha_tau_g1: np.ndarray
    beta_tau_g1: np.ndarray
    tau_g1_h: Optional[np.ndarray] = None
    h_over_2n: bool = False   # tau_g1_h from an interior level of the file (log_n < power): taken over 2n powers


LAGRANGE_MEMBERS = ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1", "tau_g1_h")


@dataclass
class Ptau:
    """What Groth16.read_ptau read from a snarkjs .ptau file: its header (n8, power, ceremony_power; prepared when its
    Lagrange sections 12-15 are present and read), the transcript `srs`, and one level of Lagrange points or None."""
    n8: int
    power: int
    ceremony_power: int
    prepared: bool
    srs: Srs
    lagrange: Optional[Lagrange] = None


def srs_arrays(srs: Srs, g1_width: int, g2_width: int, in_place: bool = False) -> dict:
    """The members of `srs` as C-contiguous uint64 arrays, as Groth16.contribute_srs hands them to the library: the vectors
    as (points, limbs) (None: no points), beta_g2 as one point of g2_width limbs.  ValueError names a member that is not
    made of whole points, a missing beta_g2, and with `in_place` a member that cannot be written where it is (not a
    C-contiguous, writable uint64 array)."""
    out = {}
    for k in SRS_VECTORS + ("beta_g2",):
        v = getattr(srs, k)
        w = g2_width if k in ("tau_g2", "beta_g2") else g1_width
        if v is None:
            if k == "beta_g2":
                raise ValueError("srs.beta_g2 is missing: it is always read and written")
            out[k] = np.zeros((0, w), dtype=np.uint64)
            continue
        a = np.ascontiguousarray(v, dtype=np.uint64)
        if in_place and (a is not v or not a.flags["WRITEABLE"]):
            raise ValueError(f"in_place needs srs.{k} to be a C-contiguous, writable uint64 array")
        if k == "beta_g2":
            if a.size != w:
                raise ValueError(f"srs.beta_g2 holds {a.size} limbs, one G2 point is {w}")
            out[k] = a.reshape(w)
        else:
            if a.ndim not in (1, 2) or a.size % w or (a.ndim == 2 and a.shape[1] != w):
                raise ValueError(f"srs.{k} of shape {a.shape} is not a list of points of {w} limbs")
            out[k] = a.reshape(-1, w)
    return out


SRS_EQUATIONS = ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1", "beta_g2")


@dataclass
class SrsPairs:
    """g16_srs_verify_pairs: the five pairing equations of a transcript check.  Equation k (the member members[k]) holds iff
    e(g1[2k], g2[2k]) = e(g1[2k + 1], g2[2k + 1]); g1 is (10, G1 limbs) and g2 is (10, G2 limbs), affine Montgomery limbs."""
    g1: np.ndarray
    g2: np.ndarray
    members: Tuple[str, ...] = SRS_EQUATIONS

    def equation(self, k: int) -> tuple:
        """(P_k, Q_k, P'_k, Q'_k) of equation k, as limb arrays"""
        return self.g1[2 * k], self.g2[2 * k], self.g1[2 * k + 1], self.g2[2 * k + 1]


SRS_VERIFY_MIN = dict(tau_g1=2, tau_g2=2, alpha_tau_g1=1, beta_tau_g1=1)


def srs_verify_args(srs: Srs, rho, r: int, g1_width: int, g2_width: int, chunk_points: int = 0) -> tuple:
    """The arguments of Groth16.srs_verification_pairs as the library takes them: (the members as srs_arrays gives them,
    rho mod r, chunk_points).  ValueError, before any device work: a member that is not made of whole points, a member
    shorter than the check needs (tau_g1 and tau_g2 two points, alpha_tau_g1 and beta_tau_g1 one) or of 2^32 points or
    more, rho = 0 mod r, chunk_points outside [0, 2^64)."""
    arrs = srs_arrays(srs, g1_width, g2_width)
    for k, need in SRS_VERIFY_MIN.items():
        have = arrs[k].shape[0]
        if have < need:
            raise ValueError(f"srs.{k} holds {have} points, the check needs at least {need}")
        if have >= 1 << 32:
            raise ValueError(f"srs.{k} holds {have} points, at most 2^32 - 1 are allowed")
    rho = int(rho) % r
    if rho == 0:
        raise ValueError("the challenge rho must be non-zero mod r")
    chunk_points = int(chunk_points)
    if not 0 <= chunk_points < 1 << 64:
        raise ValueError(f"chunk_points must be in [0, 2^64), not {chunk_points}")
    return arrs, rho, chunk_points


KEY_EQUATIONS = ("delta", "h_query", "l_query", "gamma_abc_g1")


@dataclass
class KeyPairs:
    """g16_pk_verify_pairs: the four pairing equations of a key check.  Equation k (members[k]) holds iff
    e(g1[2k], g2[2k]) = e(g1[2k + 1], g2[2k + 1]); g1 is (8, G1 limbs) and g2 is (8, G2 limbs), affine Montgomery limbs."""
    g1: np.ndarray
    g2: np.ndarray
    members: Tuple[str, ...] = KEY_EQUATIONS

    def equation(self, k: int) -> tuple:
        """(P_k, Q_k, P'_k, Q'_k) of equation k, as limb arrays"""
        return self.g1[2 * k], self.g2[2 * k], self.g1[2 * k + 1], self.g2[2 * k + 1]


KEY_VECTORS = ("a_query", "b_g1_query", "b_g2_query", "h_query", "l_query", "gamma_abc_g1")
KEY_POINTS = ("alpha_g1", "beta_g1", "delta_g1", "beta_g2", "gamma_g2", "delta_g2")


def key_members(pk: ProvingKey) -> dict:
    """the members of g16_pk_check_desc, by name, as `pk` holds them (None where it has none)"""
    vk = pk.vk
    return dict(a_query=pk.a_query, b_g1_query=pk.b_g1_query, b_g2_query=pk.b_g2_query, h_query=pk.h_query,
                l_query=pk.l_query, gamma_abc_g1=vk.gamma_abc_g1, alpha_g1=vk.alpha_g1, beta_g1=pk.beta_g1,
                delta_g1=pk.delta_g1, beta_g2=vk.beta_g2, gamma_g2=vk.gamma_g2, delta_g2=vk.delta_g2)


def pk_verify_args(pk: ProvingKey, srs: Srs, rho, r: int, g1_width: int, g2_width: int, num_inputs: int, num_witness: int,
                   log_n: int, qap: str = "libsnark") -> tuple:
    """The arguments of Groth16.key_verification_pairs as the library takes them: (the key's members as (points, limbs)
    arrays, the transcript's as srs_arrays gives them, rho mod r).  ValueError, before any device work: a key member missing
    or not of exactly the length g16_pk_export writes for the circuit (num_inputs + num_witness points in a_query,
    b_g1_query, b_g2_query; n - 1 in h_query, n under qap="circom"; num_witness in l_query; num_inputs in gamma_abc_g1;
    one point each for the others), a transcript member that is not made of whole points or is shorter than the circuit
    needs (tau_g1 2n - 1 points, the other vectors n), rho = 0 mod r."""
    n = 1 << log_n
    nv = num_inputs + num_witness
    want = dict(a_query=nv, b_g1_query=nv, b_g2_query=nv, h_query=n if qap == "circom" else n - 1, l_query=num_witness,
                gamma_abc_g1=num_inputs)
    keys = {}
    for k, v in key_members(pk).items():
        w = g2_width if k in ("b_g2_query", "beta_g2", "gamma_g2", "delta_g2") else g1_width
        if v is None:
            raise ValueError(f"the key has no {k}")
        a = np.ascontiguousarray(v, dtype=np.uint64)
        if a.size % w or (a.ndim == 2 and a.shape[1] != w) or a.ndim > 2:
            raise ValueError(f"{k} of shape {a.shape} is not made of points of {w} limbs")
        a = a.reshape(-1, w)
        need = want.get(k, 1)
        if a.shape[0] != need:
            raise ValueError(f"{k} holds {a.shape[0]} points, the circuit's key has {need}")
        keys[k] = a
    arrs = srs_arrays(srs, g1_width, g2_width)
    for k, need in zip(SRS_VECTORS, (2 * n - 1, n, n, n)):
        if arrs[k].shape[0] < need:
            raise ValueError(f"srs.{k} holds {arrs[k].shape[0]} points, the circuit (domain 2^{log_n}) needs at least {need}")
    rho = int(rho) % r
    if rho == 0:
        raise ValueError("the challenge rho must be non-zero mod r")
    return keys, arrs, rho


PK_DELTA_MEMBERS = ("h_query", "l_query", "delta_g1", "delta_g2")


def pk_contribute_args(pk: ProvingKey, delta, r: int, g1_width: int, g2_width: int, chunk_points: int = 0,
                       in_place: bool = False) -> tuple:
    """The arguments of Groth16.contribute_key as the library takes them: (h_query, l_query as (points, limbs) arrays and
    delta_g1, delta_g2 as one point each, by name; delta mod r; chunk_points).  ValueError, before any device work: a member
    missing or not made of whole points, h_query or l_query of 2^32 points or more, delta = 0 mod r (UnexpectedIdentity),
    chunk_points outside [0, 2^64), and with `in_place` a member that cannot be written where it is (not a C-contiguous,
    writable uint64 array)."""
    held = dict(h_query=pk.h_query, l_query=pk.l_query, delta_g1=pk.delta_g1, delta_g2=pk.vk.delta_g2)
    out = {}
    for k, v in held.items():
        w = g2_width if k == "delta_g2" else g1_width
        if v is None:
            raise ValueError(f"the key has no {k}")
        a = np.ascontiguousarray(v, dtype=np.uint64)
        if in_place and (a is not v or not a.flags["WRITEABLE"]):
            raise ValueError(f"in_place needs the key's {k} to be a C-contiguous, writable uint64 array")
        if a.ndim > 2 or a.size % w or (a.ndim == 2 and a.shape[1] != w):
            raise ValueError(f"{k} of shape {a.shape} is not made of points of {w} limbs")
        if k in ("delta_g1", "delta_g2"):
            if a.size != w:
                raise ValueError(f"{k} holds {a.size // w} points, it is one point")
            out[k] = a.reshape(w)
        else:
            out[k] = a.reshape(-1, w)
            if out[k].shape[0] >= 1 << 32:
                raise ValueError(f"{k} holds {out[k].shape[0]} points, at most 2^32 - 1 are allowed")
    delta = int(delta) % r
    if delta == 0:
        raise ValueError("delta must be non-zero mod r (UnexpectedIdentity)")
    chunk_points = int(chunk_points)
    if not 0 <= chunk_points < 1 << 64:
        raise ValueError(f"chunk_points must be in [0, 2^64), not {chunk_points}")
    return out, delta, chunk_points


@dataclass
class ContributionRecord:
    """One contribution's public record (the public key of Bowe, Gabizon and Miers), affine Montgomery limbs: after_g1 =
    x D for the running point D (phase 2: delta_g1; phase 1: tau_g1[1], alpha_tau_g1[0], beta_tau_g1[0]), s_g1 a point the
    contributor chose, s_x_g1 = x s, r_x_g2 = x r.  r_g2 must be derived by the checker from the ceremony's transcript (a
    hash to G2 of the contribution; the hash and the file format that binds it are the caller's) and never taken from the
    contributor: an r whose discrete log is known makes the proof of knowledge empty."""
    after_g1: np.ndarray
    s_g1: np.ndarray
    s_x_g1: np.ndarray
    r_g2: np.ndarray
    r_x_g2: np.ndarray


RECORD_MEMBERS = ("after_g1", "s_g1", "s_x_g1", "r_g2", "r_x_g2")
CHAIN_MAX = (1 << 30) - 1


@dataclass
class ChainPairs:
    """g16_contribution_chain_pairs: 2 count equations.  Equation k holds iff e(g1[2k], g2[2k]) = e(g1[2k + 1], g2[2k + 1]):
    k = 2i is record i's proof of knowledge (s_i, r_x_i) = (s_x_i, r_i), k = 2i + 1 its step (D_i, r_x_i) = (D_(i+1), r_i).
    g1 is (4 count, G1 limbs) and g2 is (4 count, G2 limbs), affine Montgomery limbs."""
    g1: np.ndarray
    g2: np.ndarray

    def __len__(self) -> int:
        return self.g1.shape[0] // 2

    def equation(self, k: int) -> tuple:
        """(P_k, Q_k, P'_k, Q'_k) of equation k, as limb arrays"""
        if not 0 <= k < len(self):
            raise IndexError(f"equation {k} of {len(self)}")
        return self.g1[2 * k], self.g2[2 * k], self.g1[2 * k + 1], self.g2[2 * k + 1]


def chain_args(start_g1, end_g1, records: Sequence[ContributionRecord], g1_width: int, g2_width: int) -> tuple:
    """The arguments of Groth16.contribution_chain_pairs as the library takes them: (start_g1, end_g1, and per record its
    five members by name, each one point as a C-contiguous uint64 array).  ValueError, before any device work: no records
    or more than 2^30 - 1, a point missing or not exactly one point of its group."""
    n = len(records)
    if not 1 <= n <= CHAIN_MAX:
        raise ValueError(f"a chain has 1 to 2^30 - 1 records, not {n}")

    def one(v, w, what):
        if v is None:
            raise ValueError(f"{what} is missing")
        a = np.ascontiguousarray(v, dtype=np.uint64)
        if a.size != w:
            raise ValueError(f"{what} holds {a.size} limbs, one point is {w}")
        return a.reshape(w)

    recs = [{m: one(getattr(c, m), g2_width if m.endswith("g2") else g1_width, f"records[{i}].{m}") for m in RECORD_MEMBERS}
            for i, c in enumerate(records)]
    return one(start_g1, g1_width, "start_g1"), one(end_g1, g1_width, "end_g1"), recs


@dataclass
class WitnessReport:
    """g16_witness_report of one assignment, None where the library reports G16_NONE"""
    first_unsatisfied: Optional[int]   # lowest constraint i with <A_i,z><B_i,z> != <C_i,z>
    num_unsatisfied: int
    first_malformed: Optional[int]     # lowest element with limbs >= r, or 0 when z[0] is not One; rows not evaluated then

    @property
    def ok(self) -> bool:
        return self.first_malformed is None and self.num_unsatisfied == 0


@dataclass
class Proof:
    a: np.ndarray  # G1 affine limbs
    b: np.ndarray  # G2 affine limbs
    c: np.ndarray  # G1 affine limbs


class Groth16:
    """One instance = one curve on one GPU (a g16_ctx).  The circuit (matrices) and the proving key are made
    resident once and reused by every proof, like a long-lived prover process would.

    `qap` is the R1CS-to-QAP reduction, the second type parameter of ark-groth16's Groth16<E, QAP>: "libsnark"
    (LibsnarkReduction, ark-groth16's default) or "circom" (ark-circom's CircomReduction, for circom circuits with
    snarkjs-compatible keys).  It decides the witness map (circom: n evaluations at the odd powers of omega_2n) and the
    H query of generate_parameters_with_qap / export_proving_key (circom: n points instead of n - 1)."""

    def __init__(self, curve, device: int = 0, qap: str = "libsnark"):
        if qap not in _lib.QAPS:
            raise ValueError(f"qap must be one of {sorted(_lib.QAPS)}, not {qap!r}")
        self.qap = qap
        self.curve: CurveParams = get_curve(curve)
        self.codec = CurveCodec(self.curve)
        self._lib = _lib.load()
        h = C.c_void_p()
        _check(self._lib.g16_ctx_create(self.curve.cid, device, C.byref(h)))
        self._ctx = h
        self.nq = self._lib.g16_fq_limbs(self._ctx)
        self._matrices: Optional[ConstraintMatrices] = None
        self._pk_resident = False
        self._pk_obj: Optional[ProvingKey] = None   # identity of the resident key (None: minted by g16_setup and not exported)
        self.world = 1

    @property
    def nr(self) -> int:
        """u64 limbs per Fr element / BigInt scalar (g16_fr_limbs)"""
        return self.curve.fr_limbs

    @property
    def ng2(self) -> int:
        """u64 limbs per G2 affine point (g16_g2_limbs)"""
        return self.curve.g2_limbs

    def close(self):
        if getattr(self, "_ctx", None):
            self._lib.g16_ctx_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- the two dependency-level operations (ark-poly / ark-ec) ----
    def ntt(self, values: np.ndarray, inverse: bool = False, coset: bool = False) -> np.ndarray:
        """Radix2EvaluationDomain::{fft,ifft}_in_place / coset variants on 2^k Montgomery Fr elements."""
        v = np.ascontiguousarray(values, dtype=np.uint64).reshape(-1, self.nr).copy()
        n = v.shape[0]
        log_n = max(n - 1, 0).bit_length()
        if (1 << log_n) != n:
            raise ValueError("length must be a power of two (ark resizes to domain.size(); do that in the caller)")
        _check(self._lib.g16_ntt(self._ctx, log_n, int(inverse), int(coset), _ptr(v)))
        return v

    def ntt_log(self, log_n: int, values: np.ndarray, inverse=False, coset=False) -> np.ndarray:
        """Same transform with the domain size given explicitly (error-path tests: log_n above the two-adicity).  The C side
        copies 8 * nr << log_n bytes in and out of `values`, so the length is checked here."""
        v = np.ascontiguousarray(values, dtype=np.uint64).reshape(-1, self.nr).copy()
        if log_n < 0 or (log_n <= self.curve.two_adicity and v.shape[0] != (1 << log_n)):
            raise ValueError(f"values must hold exactly 2^{log_n} field elements")
        # log_n above the two-adicity: the C side returns PolynomialDegreeTooLarge before it touches the buffer
        _check(self._lib.g16_ntt(self._ctx, log_n, int(inverse), int(coset), _ptr(v)))
        return v

    def witness_map_from_evals(self, a: np.ndarray, b: np.ndarray, c: np.ndarray) -> np.ndarray:
        a = np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, self.nr)
        b = np.ascontiguousarray(b, dtype=np.uint64).reshape(-1, self.nr)
        c = np.ascontiguousarray(c, dtype=np.uint64).reshape(-1, self.nr)
        n = a.shape[0]
        log_n = max(n - 1, 0).bit_length()
        if (1 << log_n) != n or b.shape != a.shape or c.shape != a.shape:
            raise ValueError("a, b, c must have the same power-of-two length")
        h = np.empty_like(a)
        _check(self._lib.g16_witness_map_evals(self._ctx, log_n, _ptr(a), _ptr(b), _ptr(c), _ptr(h)))
        return h

    def msm_g1(self, bases: np.ndarray, scalars: np.ndarray) -> np.ndarray:
        """VariableBaseMSM::msm_bigint on G1: truncates to the shorter operand like ark (prover.rs:66 relies on it)."""
        bases = np.ascontiguousarray(bases, dtype=np.uint64).reshape(-1, 2 * self.nq)
        scalars = np.ascontiguousarray(scalars, dtype=np.uint64).reshape(-1, self.nr)
        n = min(bases.shape[0], scalars.shape[0])
        out = np.zeros(3 * self.nq, dtype=np.uint64)
        _check(self._lib.g16_msm_g1(self._ctx, _ptr(bases), _ptr(scalars), n, _ptr(out)))
        return out

    def msm_g2(self, bases: np.ndarray, scalars: np.ndarray) -> np.ndarray:
        bases = np.ascontiguousarray(bases, dtype=np.uint64).reshape(-1, self.ng2)
        scalars = np.ascontiguousarray(scalars, dtype=np.uint64).reshape(-1, self.nr)
        n = min(bases.shape[0], scalars.shape[0])
        out = np.zeros(3 * self.ng2 // 2, dtype=np.uint64)
        _check(self._lib.g16_msm_g2(self._ctx, _ptr(bases), _ptr(scalars), n, _ptr(out)))
        return out

    def prepare_inputs(self, vk: VerifyingKey, public_inputs) -> np.ndarray:
        """Groth16::prepare_inputs (verifier.rs:25-39): gamma_abc_g1[0] + sum_i x_i * gamma_abc_g1[i + 1], computed as ONE G1
        MSM with scalars (1, x_0, x_1, ...).  `public_inputs`: Python ints, or an (l, 4) array of Montgomery Fr limbs (ark's
        memory image).  Returns the projective point in msm_g1's encoding.  A length mismatch is
        SynthesisError::MalformedVerifyingKey (verifier.rs:30)."""
        if vk.gamma_abc_g1 is None:
            raise MalformedKey("verifying key has no gamma_abc_g1")
        abc = np.ascontiguousarray(vk.gamma_abc_g1, dtype=np.uint64).reshape(-1, 2 * self.nq)
        if isinstance(public_inputs, np.ndarray):
            xs = self.codec.fr.dec(np.ascontiguousarray(public_inputs, dtype=np.uint64).reshape(-1, self.nr))
        else:
            xs = [int(x) % self.curve.r for x in public_inputs]
        if len(xs) + 1 != abc.shape[0]:
            raise MalformedKey("public input count does not match the verifying key")
        return self.msm_g1(abc, self.codec.fr.bigint([1] + xs))

    # ---- resident state ----
    def load_matrices(self, m: ConstraintMatrices):
        def csr(t):
            rp, col, val = t
            s = _lib.Csr()
            rpc = np.ascontiguousarray(rp, dtype=np.uint32)
            colc = np.ascontiguousarray(col, dtype=np.uint32)
            valc = np.ascontiguousarray(val, dtype=np.uint64)
            s.row_ptr = _u32p(rpc)
            s.col = _u32p(colc) if colc.size else None
            s.val = _u64p(valc) if valc.size else None
            return s, (rpc, colc, valc)

        keep = []
        structs = []
        for t in (m.a, m.b, m.c):
            s, k = csr(t)
            structs.append(s)
            keep.append(k)
        _check(self._lib.g16_circuit_load_qap(self._ctx, _lib.QAPS[self.qap], m.num_instance_variables, m.num_constraints,
                                              m.num_witness_variables, C.byref(structs[0]), C.byref(structs[1]),
                                              C.byref(structs[2])))
        self._matrices = m
        self._pk_resident = False
        self._pk_obj = None

    def load_proving_key(self, pk: ProvingKey, rank: int = 0, world: int = 1):
        d = _lib.PkDesc()
        arrs = {}
        for name in ("a_query", "b_g1_query", "b_g2_query", "h_query", "l_query"):
            arr = np.ascontiguousarray(getattr(pk, name), dtype=np.uint64)
            arrs[name] = arr
            width = self.ng2 if name == "b_g2_query" else 2 * self.nq
            arr2 = arr.reshape(-1, width)
            setattr(d, name, _u64p(arr) if arr.size else None)
            setattr(d, name.replace("_query", "_len"), arr2.shape[0])
        singles = dict(alpha_g1=pk.vk.alpha_g1, beta_g1=pk.beta_g1, delta_g1=pk.delta_g1, beta_g2=pk.vk.beta_g2,
                       delta_g2=pk.vk.delta_g2)
        for k, v in singles.items():
            arrs[k] = np.ascontiguousarray(v, dtype=np.uint64)
            setattr(d, k, _u64p(arrs[k]))
        _check(self._lib.g16_pk_load(self._ctx, C.byref(d), rank, world))
        self._pk_resident = True
        self._pk_obj = pk
        self.world = world

    # ---- generator.rs:47-208 with explicit toxic waste and generators ----
    def generate_parameters_with_qap(self, matrices: ConstraintMatrices, alpha, beta, gamma, delta, tau, g1_generator,
                                     g2_generator, export: bool = True) -> Optional[ProvingKey]:
        """alpha..tau: Python ints (canonical); g1/g2 generators: affine int tuples.  The key becomes resident."""
        self.load_matrices(matrices)
        cd = self.codec
        sc = [np.ascontiguousarray(cd.fr.enc1(x)) for x in (alpha, beta, gamma, delta, tau)]
        g1 = np.ascontiguousarray(cd.enc_g1([g1_generator])[0])
        g2 = np.ascontiguousarray(cd.enc_g2([g2_generator])[0])
        _check(self._lib.g16_setup(self._ctx, *[_ptr(x) for x in sc], _ptr(g1), _ptr(g2)))
        self._pk_resident = True
        self.world = 1
        self._pk_obj = self.export_proving_key() if export else None
        return self._pk_obj

    # ---- keys from a powers-of-tau transcript (g16_setup_from_srs) and phase-2 contributions ----
    def srs_from_secrets(self, g1_len: int, g2_len: int, tau, alpha, beta, g1_generator, g2_generator) -> Srs:
        """g16_srs_from_secrets, for tests and benchmarks: the transcript of known secrets (Python ints), with g1_len points in
        tau_g1 and g2_len in tau_g2, alpha_tau_g1 and beta_tau_g1."""
        cd = self.codec
        z = lambda rows, w: np.zeros((rows, w), dtype=np.uint64)
        srs = Srs(z(g1_len, 2 * self.nq), z(g2_len, self.ng2), z(g2_len, 2 * self.nq), z(g2_len, 2 * self.nq),
                  np.zeros(self.ng2, dtype=np.uint64))
        d = _lib.SrsOut()
        for k in ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1"):
            v = getattr(srs, k)
            setattr(d, k, _u64p(v) if v.size else None)
            setattr(d, k + "_len", v.shape[0])
        d.beta_g2 = _u64p(srs.beta_g2)
        sc = [np.ascontiguousarray(cd.fr.enc1(x)) for x in (tau, alpha, beta)]
        g1 = np.ascontiguousarray(cd.enc_g1([g1_generator])[0])
        g2 = np.ascontiguousarray(cd.enc_g2([g2_generator])[0])
        _check(self._lib.g16_srs_from_secrets(self._ctx, *[_ptr(x) for x in sc], _ptr(g1), _ptr(g2), C.byref(d)))
        return srs

    def generate_parameters_from_srs(self, matrices: Optional[ConstraintMatrices], srs: Srs, validate: bool = False,
                                     export: bool = True) -> Optional[ProvingKey]:
        """g16_setup_from_srs: the proving key of `matrices` (None: the resident circuit) derived on the GPU from a
        powers-of-tau transcript, with gamma = delta = 1 until contribute_delta.  The key becomes resident; a point the checks
        refuse raises serialize.DeserializeError naming it, and leaves no key resident."""
        if matrices is not None:
            self.load_matrices(matrices)
        d, keep = self._srs_desc(srs)
        rc = self._lib.g16_setup_from_srs(self._ctx, C.byref(d), _lib.SER_VALIDATE if validate else 0)
        return self._after_setup(rc, export)

    def _srs_desc(self, srs: Srs) -> tuple:
        """g16_srs_desc of `srs` (a missing member: null, length 0) and the arrays it points into"""
        d = _lib.SrsDesc()
        keep = []
        for k in SRS_VECTORS:
            v = getattr(srs, k)
            v = None if v is None else np.ascontiguousarray(v, dtype=np.uint64)
            keep.append(v)
            setattr(d, k, _u64p(v) if v is not None and v.size else None)
            width = self.ng2 if k == "tau_g2" else 2 * self.nq
            setattr(d, k + "_len", 0 if v is None else v.size // width)
        bg2 = None if srs.beta_g2 is None else np.ascontiguousarray(srs.beta_g2, dtype=np.uint64)
        keep.append(bg2)
        d.beta_g2 = _u64p(bg2)
        return d, keep

    def _after_setup(self, rc: int, export: bool) -> Optional[ProvingKey]:
        self._after_key_change(rc)
        self._pk_resident = True
        self.world = 1
        self._pk_obj = self.export_proving_key() if export else None
        return self._pk_obj

    # ---- snarkjs .ptau files (g16_ptau_read) and keys from their Lagrange points (g16_setup_from_lagrange) ----
    def read_ptau(self, data: bytes, log_n: Optional[int] = None) -> Ptau:
        """g16_ptau_read: a snarkjs .ptau transcript as this ABI's limbs, copied on the host (every call that takes the points
        checks them on the GPU).  With `log_n`, only what a circuit of domain 2^log_n needs: the prefixes of 2n - 1 (2n when
        log_n is below the file's power), n, n and n points and, for a prepared file, level log_n of the Lagrange points (with
        tau_g1_h under CircomReduction).
        Without it, the whole powers and no Lagrange points.  A malformed file raises serialize.DeserializeError naming the
        problem; a request the file cannot serve (log_n above its power) raises ValueError."""
        buf = np.frombuffer(data, dtype=np.uint8)
        ptr = buf.ctypes.data_as(C.c_void_p) if buf.size else None
        info = _lib.PtauInfo()
        _check(self._lib.g16_ptau_read(self._ctx, ptr, buf.size, None, None, C.byref(info)))
        np_ = 1 << info.power
        n = np_ if log_n is None else 1 << int(log_n)
        # below the file's power, the interior H level is checked against and corrected by tau_g1[2n - 1]
        lens = (2 * np_ - 1, np_, np_, np_) if log_n is None else (min(2 * n, 2 * np_ - 1), n, n, n)
        z = lambda rows, w: np.zeros((rows, w), dtype=np.uint64)
        widths = [self.ng2 if k == "tau_g2" else 2 * self.nq for k in SRS_VECTORS]
        srs = Srs(*[z(ln, w) for ln, w in zip(lens, widths)], np.zeros(self.ng2, dtype=np.uint64))
        so = _lib.SrsOut()
        for k, ln in zip(SRS_VECTORS, lens):
            setattr(so, k, _u64p(getattr(srs, k)))
            setattr(so, k + "_len", ln)
        so.beta_g2 = _u64p(srs.beta_g2)
        lag = None
        lo = None
        if log_n is not None and info.prepared:
            lag = Lagrange(int(log_n), z(n, 2 * self.nq), z(n, self.ng2), z(n, 2 * self.nq), z(n, 2 * self.nq),
                           z(n, 2 * self.nq) if self.qap == "circom" else None)
            lo = _lib.LagrangeOut()
            lo.log_n = int(log_n)
            for k in LAGRANGE_MEMBERS:
                setattr(lo, k, _u64p(getattr(lag, k)))
        _check(self._lib.g16_ptau_read(self._ctx, ptr, buf.size, C.byref(so), C.byref(lo) if lo is not None else None,
                                       C.byref(info)))
        if lag is not None:
            lag.h_over_2n = bool(lo.h_over_2n)
        return Ptau(info.n8, info.power, info.ceremony_power, bool(info.prepared), srs, lag)

    def generate_parameters_from_lagrange(self, matrices: Optional[ConstraintMatrices], srs: Srs, lagrange: Lagrange, rho=None,
                                          validate: bool = False, export: bool = True) -> Optional[ProvingKey]:
        """g16_setup_from_lagrange: the key generate_parameters_from_srs derives from `srs`, limb for limb, made from the
        Lagrange points `lagrange` (level log n of a prepared .ptau) instead of group transforms of the powers.  The points
        are first checked against `srs` on the GPU under the challenge rho (a Python int, non-zero mod r; None: drawn with
        `secrets`).  A point the checks refuse or a member that is not the transform of the transcript raises
        serialize.DeserializeError naming it and leaves the circuit and no key resident; argument errors raise ValueError
        and keep the previous key.  `validate` adds the subgroup check of every point, without which the answer means
        nothing on a curve whose cofactor is not 1."""
        if matrices is not None:
            self.load_matrices(matrices)
        d, keep = self._srs_desc(srs)
        ld = _lib.LagrangeDesc()
        ld.log_n = int(lagrange.log_n)
        ld.h_over_2n = int(bool(lagrange.h_over_2n))
        for k in LAGRANGE_MEMBERS:
            v = getattr(lagrange, k)
            v = None if v is None else np.ascontiguousarray(v, dtype=np.uint64)
            keep.append(v)
            setattr(ld, k, _u64p(v) if v is not None and v.size else None)
        r = self.curve.r
        rho = secrets.randbelow(r - 1) + 1 if rho is None else int(rho) % r
        r_ = np.ascontiguousarray(self.codec.fr.enc1(rho))
        rc = self._lib.g16_setup_from_lagrange(self._ctx, C.byref(d), C.byref(ld), _ptr(r_), _lib.SER_VALIDATE if validate else 0)
        return self._after_setup(rc, export)

    def generate_parameters_from_ptau(self, matrices: Optional[ConstraintMatrices], data: bytes, rho=None, validate: bool = False,
                                      export: bool = True) -> Optional[ProvingKey]:
        """The key of `matrices` (None: the resident circuit) from a snarkjs .ptau file: read for the circuit's domain, then
        generate_parameters_from_lagrange when the file is prepared and generate_parameters_from_srs when it is not.  Both
        give the same key."""
        if matrices is not None:
            self.load_matrices(matrices)
        if self._matrices is None:
            raise ValueError("load_matrices must come first")
        p = self.read_ptau(data, self._lib.g16_domain_log(self._ctx))
        if p.lagrange is not None:
            return self.generate_parameters_from_lagrange(None, p.srs, p.lagrange, rho, validate, export)
        return self.generate_parameters_from_srs(None, p.srs, validate, export)

    def prepare_ptau(self, data, validate: bool = False, out=None):
        """g16_ptau_prepare: snarkjs `powersoftau prepare phase2` on the GPU.  Returns the .ptau `data` with its Lagrange
        sections 12..15 computed from the powers (those of a prepared input are recomputed), as bytes.  With `out`, a
        writable uint8 buffer (an np.memmap of the target file, say) of at least the prepared size, writes into it instead
        and returns the length, so a large file needs no second copy in RAM.  Every point of sections 2..5 is checked on the
        GPU first (`validate`: also in the prime-order subgroup); a refused point or a malformed file raises
        serialize.DeserializeError naming it, power + 1 above the scalar field's two-adicity PolynomialDegreeTooLarge, and a
        level larger than the free device memory CudaError.  The file is not checked to be a powers-of-tau transcript
        (srs_verification_pairs does that)."""
        buf = np.frombuffer(data, dtype=np.uint8)
        ptr = buf.ctypes.data_as(C.c_void_p) if buf.size else None
        flags = _lib.SER_VALIDATE if validate else 0
        n = C.c_uint64()
        _check(self._lib.g16_ptau_prepare(self._ctx, ptr, buf.size, flags, None, 0, C.byref(n)))
        if out is None:
            res = np.empty(n.value, dtype=np.uint8)
        else:
            res = out if isinstance(out, np.ndarray) else np.frombuffer(out, dtype=np.uint8)
            if res.dtype != np.uint8 or res.ndim != 1 or not res.flags.c_contiguous or not res.flags.writeable:
                raise ValueError("out must be a writable, contiguous 1-D uint8 buffer")
        _check(self._lib.g16_ptau_prepare(self._ctx, ptr, buf.size, flags, res.ctypes.data_as(C.c_void_p), res.size,
                                          C.byref(n)))
        return res.tobytes() if out is None else n.value

    def contribute_delta(self, delta, export: bool = True) -> Optional[ProvingKey]:
        """g16_setup_contribute: one phase-2 contribution delta (Python int) to the resident key made by
        generate_parameters_with_qap or generate_parameters_from_srs.  Returns the new key when `export`."""
        dl = np.ascontiguousarray(self.codec.fr.enc1(delta))
        self._after_key_change(self._lib.g16_setup_contribute(self._ctx, _ptr(dl)))
        self._pk_obj = self.export_proving_key() if export else None
        return self._pk_obj

    def contribute_srs(self, srs: Srs, tau, alpha, beta, validate: bool = False, chunk_points: int = 0,
                       in_place: bool = False) -> Srs:
        """g16_srs_contribute: one phase-1 contribution of the secrets tau, alpha, beta (Python ints) to the transcript `srs`,
        on the GPU: point i of tau_g1 and tau_g2 times tau^i, of alpha_tau_g1 times alpha tau^i, of beta_tau_g1 times
        beta tau^i, and beta_g2 times beta.  Returns the new transcript; with `in_place` it is written into srs's own arrays
        (each then a C-contiguous, writable uint64 array) and srs is returned.  `validate` adds the subgroup check of every
        point; `chunk_points` caps the points per chunk (0: as many as the free device memory holds).  A refused point raises
        serialize.DeserializeError naming it, with nothing written.  Needs no circuit or key and leaves the resident ones
        alone."""
        ins = srs_arrays(srs, 2 * self.nq, self.ng2, in_place)
        chunk_points = int(chunk_points)
        if not 0 <= chunk_points < 1 << 64:
            raise ValueError(f"chunk_points must be in [0, 2^64), not {chunk_points}")
        outs = ins if in_place else {k: np.empty_like(v) for k, v in ins.items()}
        d_in, d_out = _lib.SrsDesc(), _lib.SrsOut()
        for d, arrs in ((d_in, ins), (d_out, outs)):
            for k in SRS_VECTORS:
                v = arrs[k]
                setattr(d, k, _u64p(v) if v.size else None)
                setattr(d, k + "_len", v.shape[0])
            d.beta_g2 = _u64p(arrs["beta_g2"])
        sc = [np.ascontiguousarray(self.codec.fr.enc1(x)) for x in (tau, alpha, beta)]
        _check(self._lib.g16_srs_contribute(self._ctx, C.byref(d_in), *[_ptr(x) for x in sc],
                                            _lib.SER_VALIDATE if validate else 0, chunk_points, C.byref(d_out)))
        return srs if in_place else Srs(**outs)

    def srs_verification_pairs(self, srs: Srs, rho, g1=None, g2=None, validate: bool = True,
                               chunk_points: int = 0) -> SrsPairs:
        """g16_srs_verify_pairs: the GPU part of checking that `srs` is a powers-of-tau transcript T(tau, alpha, beta) over
        the generators g1, g2 (affine int tuples; default params.GENERATORS[curve]).  rho (a Python int, non-zero mod r) is
        the challenge: draw it after the transcript is fixed, so that whoever made the transcript cannot predict it (e.g.
        secrets.randbelow(r - 1) + 1, or a hash of the transcript).

        The library checks every point (canonical, on the curve, and with `validate` in the prime-order subgroup), refuses
        the identity anywhere and checks tau_g1[0] = g1 and tau_g2[0] = g2; a refused point raises
        serialize.DeserializeError naming it.  It returns five equations, one per member (SrsPairs): with
        (P, Q, P', Q') = pairs.equation(k), the caller evaluates e(P, Q) = e(P', Q') with its own pairing, e.g.
        multi_pairing([P, -P'], [Q, Q']) == 1.  The transcript is accepted iff all five hold; then, with probability at
        least 1 - N/r over rho, it is T(tau, alpha, beta) for non-zero tau, alpha, beta with one tau in both groups.
        `validate` defaults to True: without the subgroup check the answer means nothing on a curve whose cofactor is not
        1.  `chunk_points` caps the points per chunk (0: as many as the free device memory holds).  Needs no circuit or key
        and leaves the resident ones alone."""
        arrs, rho, chunk_points = srs_verify_args(srs, rho, self.curve.r, 2 * self.nq, self.ng2, chunk_points)
        G = GENERATORS[self.curve.name]
        cd = self.codec
        g1 = np.ascontiguousarray(cd.enc_g1([G["g1"] if g1 is None else g1])[0])
        g2 = np.ascontiguousarray(cd.enc_g2([G["g2"] if g2 is None else g2])[0])
        d = _lib.SrsDesc()
        for k in SRS_VECTORS:
            setattr(d, k, _u64p(arrs[k]))
            setattr(d, k + "_len", arrs[k].shape[0])
        d.beta_g2 = _u64p(arrs["beta_g2"])
        out1 = np.zeros((10, 2 * self.nq), dtype=np.uint64)
        out2 = np.zeros((10, self.ng2), dtype=np.uint64)
        r_ = np.ascontiguousarray(cd.fr.enc1(rho))
        _check(self._lib.g16_srs_verify_pairs(self._ctx, C.byref(d), _ptr(g1), _ptr(g2), _ptr(r_),
                                              _lib.SER_VALIDATE if validate else 0, chunk_points, _ptr(out1), _ptr(out2)))
        return SrsPairs(out1, out2)

    def key_verification_pairs(self, pk: ProvingKey, srs: Srs, rho, validate: bool = True,
                               uncontributed: bool = False) -> KeyPairs:
        """g16_pk_verify_pairs: the GPU part of checking that `pk` is the key of the resident circuit (under this instance's
        reduction) made from the transcript `srs`: g16_setup(alpha, beta, gamma, delta, tau) for the transcript's tau,
        alpha, beta.  rho (a Python int, non-zero mod r) is the challenge: draw it after the key and transcript are fixed.

        The library checks every point (canonical, on the curve, and with `validate` in the prime-order subgroup), that
        alpha_g1, beta_g1 and beta_g2 are the transcript's, that delta and gamma are not the identity, that gamma_g2 !=
        delta_g2 (`uncontributed` accepts gamma = delta, the key generate_parameters_from_srs makes before any
        contribution), and that the a_query, b_g1_query and b_g2_query combinations match the transcript's; a refusal raises
        serialize.DeserializeError naming the member.  It returns four equations (KeyPairs): with (P, Q, P', Q') =
        pairs.equation(k), the caller evaluates e(P, Q) = e(P', Q') with its own pairing.  The key is accepted iff all four
        hold; then, with probability at least 1 - 6 max(nv, n) / r over rho, it is that setup point for point.  Needs a
        resident circuit, no key, and leaves the resident key alone."""
        m = self._matrices
        if m is None:
            raise ValueError("load_matrices must come first")
        keys, arrs, rho = pk_verify_args(pk, srs, rho, self.curve.r, 2 * self.nq, self.ng2, m.num_instance_variables,
                                         m.num_witness_variables, self._lib.g16_domain_log(self._ctx), self.qap)
        d = _lib.PkCheckDesc()
        for k, v in keys.items():
            setattr(d, k, _u64p(v) if v.size else None)
        s = _lib.SrsDesc()
        for k in SRS_VECTORS:
            setattr(s, k, _u64p(arrs[k]))
            setattr(s, k + "_len", arrs[k].shape[0])
        s.beta_g2 = _u64p(arrs["beta_g2"])
        out1 = np.zeros((8, 2 * self.nq), dtype=np.uint64)
        out2 = np.zeros((8, self.ng2), dtype=np.uint64)
        r_ = np.ascontiguousarray(self.codec.fr.enc1(rho))
        flags = (_lib.SER_VALIDATE if validate else 0) | (_lib.PK_UNCONTRIBUTED if uncontributed else 0)
        _check(self._lib.g16_pk_verify_pairs(self._ctx, C.byref(s), C.byref(d), _ptr(r_), flags, _ptr(out1), _ptr(out2)))
        return KeyPairs(out1, out2)

    def contribute_key(self, pk: ProvingKey, delta, validate: bool = False, chunk_points: int = 0,
                       in_place: bool = False) -> ProvingKey:
        """g16_pk_contribute: one phase-2 contribution delta (a Python int) to a key received from another party, on the GPU:
        delta_g1 and delta_g2 times delta, every h_query and l_query point times delta^-1.  Returns a new ProvingKey whose
        other members are pk's own arrays; with `in_place` the four members are written into pk's arrays (each then a
        C-contiguous, writable uint64 array) and pk is returned.  `validate` adds the subgroup check of every point;
        `chunk_points` caps the points per chunk (0: as many as the free device memory holds).  A refused point (delta_g1
        or delta_g2 the identity among them) raises serialize.DeserializeError naming it, with nothing written.  Needs no
        circuit or key and leaves the resident ones alone."""
        ins, delta, chunk_points = pk_contribute_args(pk, delta, self.curve.r, 2 * self.nq, self.ng2, chunk_points, in_place)
        outs = ins if in_place else {k: np.empty_like(v) for k, v in ins.items()}
        d_in, d_out = _lib.PkDeltaDesc(), _lib.PkDeltaOut()
        for d, arrs in ((d_in, ins), (d_out, outs)):
            for k in ("h_query", "l_query"):
                setattr(d, k, _u64p(arrs[k]) if arrs[k].size else None)
                setattr(d, k.replace("_query", "_len"), arrs[k].shape[0])
            d.delta_g1, d.delta_g2 = _u64p(arrs["delta_g1"]), _u64p(arrs["delta_g2"])
        dl = np.ascontiguousarray(self.codec.fr.enc1(delta))
        _check(self._lib.g16_pk_contribute(self._ctx, C.byref(d_in), _ptr(dl), _lib.SER_VALIDATE if validate else 0,
                                           chunk_points, C.byref(d_out)))
        if in_place:
            return pk
        vk = pk.vk
        return ProvingKey(VerifyingKey(vk.alpha_g1, vk.beta_g2, vk.gamma_g2, outs["delta_g2"], vk.gamma_abc_g1), pk.beta_g1,
                          outs["delta_g1"], pk.a_query, pk.b_g1_query, pk.b_g2_query, outs["h_query"], outs["l_query"])

    def contribution_chain_pairs(self, start_g1, end_g1, records: Sequence[ContributionRecord],
                                 validate: bool = True) -> ChainPairs:
        """g16_contribution_chain_pairs: the proofs of knowledge of a chain of contributions, either phase.  With D_0 =
        start_g1 (phase 2: the uncontributed key's delta_g1 = tau_g1[0]; phase 1: tau_g1[1], alpha_tau_g1[0] or
        beta_tau_g1[0] of the transcript before the first contribution) and D_(i+1) = records[i].after_g1, it returns 2
        len(records) equations (ChainPairs): with (P, Q, P', Q') = pairs.equation(k), the caller evaluates e(P, Q) = e(P',
        Q') with its own pairing.  If all hold, end_g1 = (prod x_i) start_g1, and contributor i knew x_i provided each
        records[i].r_g2 was derived by the checker from the ceremony's transcript (never taken from the contributor).
        The library checks every point (canonical, on the curve, with `validate` in the prime-order subgroup, never the
        identity) and that the last record's after_g1 is end_g1; a refusal raises serialize.DeserializeError naming the
        record and member.  `validate` defaults to True: without the subgroup check the answer means nothing on a curve
        whose cofactor is not 1.  Needs no circuit or key and leaves the resident ones alone."""
        start, end, recs = chain_args(start_g1, end_g1, records, 2 * self.nq, self.ng2)
        descs = (_lib.ContributionRecord * len(recs))()
        for d, rc in zip(descs, recs):
            for m in RECORD_MEMBERS:
                setattr(d, m, _u64p(rc[m]))
        out1 = np.zeros((4 * len(recs), 2 * self.nq), dtype=np.uint64)
        out2 = np.zeros((4 * len(recs), self.ng2), dtype=np.uint64)
        _check(self._lib.g16_contribution_chain_pairs(self._ctx, _ptr(start), _ptr(end), descs, len(recs),
                                                      _lib.SER_VALIDATE if validate else 0, _ptr(out1), _ptr(out2)))
        return ChainPairs(out1, out2)

    def _after_key_change(self, rc: int):
        """Status of g16_setup_from_srs / g16_setup_contribute: argument errors (G16_ERR_BAD_ARGUMENT,
        G16_ERR_MALFORMED_KEY) leave the previous key resident, any other failure happens after it was released."""
        if rc not in (_lib.G16_OK, _lib.ERR_BAD_ARGUMENT, _lib.ERR_MALFORMED_KEY):
            self._pk_resident = False
            self._pk_obj = None
        _check(rc)

    def export_proving_key(self) -> ProvingKey:
        m = self._matrices
        nq, ng2 = self.nq, self.ng2
        nv = m.num_instance_variables + m.num_witness_variables
        n = 1 << self._lib.g16_domain_log(self._ctx)
        hn = n if self.qap == "circom" else n - 1   # CircomReduction::h_query_scalars gives n scalars, libsnark n - 1
        z = lambda rows, w: np.zeros((rows, w), dtype=np.uint64)
        out = dict(a_query=z(nv, 2 * nq), b_g1_query=z(nv, 2 * nq), b_g2_query=z(nv, ng2), h_query=z(hn, 2 * nq),
                   l_query=z(m.num_witness_variables, 2 * nq), alpha_g1=z(1, 2 * nq), beta_g1=z(1, 2 * nq),
                   delta_g1=z(1, 2 * nq), beta_g2=z(1, ng2), gamma_g2=z(1, ng2), delta_g2=z(1, ng2),
                   gamma_abc_g1=z(m.num_instance_variables, 2 * nq))
        d = _lib.PkExportDesc()
        for k, v in out.items():
            setattr(d, k, _u64p(v) if v.size else None)
        _check(self._lib.g16_pk_export(self._ctx, C.byref(d)))
        vk = VerifyingKey(out["alpha_g1"][0], out["beta_g2"][0], out["gamma_g2"][0], out["delta_g2"][0], out["gamma_abc_g1"])
        return ProvingKey(vk, out["beta_g1"][0], out["delta_g1"][0], out["a_query"], out["b_g1_query"], out["b_g2_query"],
                          out["h_query"], out["l_query"])

    # ---- ark-serialized proving keys (ProvingKey::serialize_* / deserialize_with_mode), decoded and encoded on the GPU ----
    def load_proving_key_bytes(self, data: bytes, compress: bool = True, validate: bool = True, rank: int = 0,
                               world: int = 1) -> VerifyingKey:
        """g16_pk_load_serialized: make the key in `data` (a whole ark-serialized ProvingKey of this curve) resident, exactly as
        load_proving_key would the same key in limbs, and return its verifying key (with beta_g1 / delta_g1 on the side as
        attributes).  A rejected key raises serialize.DeserializeError naming the first bad item; a gamma_abc_g1 that does not
        match the circuit raises MalformedKey.  Afterwards no key is resident until a load succeeds."""
        m = self._matrices
        if m is None:
            raise ValueError("load_matrices must come first")
        buf = np.frombuffer(data, dtype=np.uint8)
        nq, ng2, ni = self.nq, self.ng2, m.num_instance_variables
        z = lambda rows, w: np.zeros((rows, w), dtype=np.uint64)
        out = dict(alpha_g1=z(1, 2 * nq), beta_g1=z(1, 2 * nq), delta_g1=z(1, 2 * nq), beta_g2=z(1, ng2),
                   gamma_g2=z(1, ng2), delta_g2=z(1, ng2), gamma_abc_g1=z(ni, 2 * nq))
        d = _lib.PkExportDesc()
        for k, v in out.items():
            setattr(d, k, _u64p(v) if v.size else None)
        flags = (_lib.SER_COMPRESSED if compress else 0) | (_lib.SER_VALIDATE if validate else 0)
        self._pk_resident = False
        self._pk_obj = None
        _check(self._lib.g16_pk_load_serialized(self._ctx, buf.ctypes.data_as(C.c_void_p) if buf.size else None, buf.size, flags,
                                                rank, world, C.byref(d)))
        self._pk_resident = True
        self.world = world
        vk = VerifyingKey(out["alpha_g1"][0], out["beta_g2"][0], out["gamma_g2"][0], out["delta_g2"][0], out["gamma_abc_g1"])
        vk.beta_g1, vk.delta_g1 = out["beta_g1"][0], out["delta_g1"][0]
        return vk

    def load_zkey(self, data: bytes, validate: bool = True, rank: int = 0, world: int = 1) -> Tuple[VerifyingKey, ZkeyCircuit]:
        """g16_zkey_load: make the circuit (A and B; under CircomReduction) and the proving key of a snarkjs .zkey resident in
        one call, the GPU counterpart of ark-circom's read_zkey followed by Groth16<E, CircomReduction>.  Sets this
        context's reduction to "circom".  Returns the verifying key (beta_g1 / delta_g1 on the side as attributes) and the
        derived circuit sizes.  A malformed file raises serialize.DeserializeError naming the first bad item (the previous
        circuit and key stay resident when the file's structure or header is refused, none when a coefficient or point is);
        another curve's context raises ValueError."""
        buf = np.frombuffer(data, dtype=np.uint8)
        nq, ng2 = self.nq, self.ng2
        z = lambda rows, w: np.zeros((rows, w), dtype=np.uint64)
        # gamma_abc_g1 holds nPublic + 1 points: read nPublic from the header when it is there, the C side checks the rest
        ni = _zkey_num_inputs(data, nq)
        out = dict(alpha_g1=z(1, 2 * nq), beta_g1=z(1, 2 * nq), delta_g1=z(1, 2 * nq), beta_g2=z(1, ng2),
                   gamma_g2=z(1, ng2), delta_g2=z(1, ng2), gamma_abc_g1=z(ni, 2 * nq))
        d = _lib.PkExportDesc()
        for k, v in out.items():
            setattr(d, k, _u64p(v) if v.size else None)
        info = _lib.ZkeyInfo()
        flags = _lib.SER_VALIDATE if validate else 0
        rc = self._lib.g16_zkey_load(self._ctx, buf.ctypes.data_as(C.c_void_p) if buf.size else None, buf.size, flags, rank,
                                     world, C.byref(d), C.byref(info))
        if rc not in (_lib.G16_OK, _lib.ERR_BAD_ARGUMENT, _lib.ERR_POLYNOMIAL_DEGREE_TOO_LARGE) and not _zkey_host_refusal():
            self._matrices = None
            self._pk_resident = False
            self._pk_obj = None
        _check(rc)
        self.qap = "circom"
        self._matrices = ZkeyCircuit(info.num_inputs, info.num_constraints, info.num_witness, info.log_n, info.a_nnz,
                                     info.b_nnz)
        self._pk_resident = True
        self._pk_obj = None
        self.world = world
        vk = VerifyingKey(out["alpha_g1"][0], out["beta_g2"][0], out["gamma_g2"][0], out["delta_g2"][0],
                          out["gamma_abc_g1"][:info.num_inputs])
        vk.beta_g1, vk.delta_g1 = out["beta_g1"][0], out["delta_g1"][0]
        return vk, self._matrices

    def load_zkey_key(self, data: bytes, validate: bool = True, rank: int = 0, world: int = 1) -> VerifyingKey:
        """g16_zkey_load with G16_ZKEY_KEY_ONLY: make only the proving key of a snarkjs .zkey resident, onto the resident
        circuit (typically from load_r1cs, which keeps C), with the rules of load_proving_key.  Its coefficient section is not
        read: whether the key belongs to the circuit is key_verification_pairs's question.  Needs a resident circuit under
        qap="circom" (ValueError otherwise); sizes other than the circuit's raise MalformedKey and a malformed file
        serialize.DeserializeError, both leaving the previous key resident; a refused point leaves no key."""
        m = self._matrices
        if m is None:
            raise ValueError("load_r1cs or load_matrices must come first")
        buf = np.frombuffer(data, dtype=np.uint8)
        nq, ng2 = self.nq, self.ng2
        z = lambda rows, w: np.zeros((rows, w), dtype=np.uint64)
        out = dict(alpha_g1=z(1, 2 * nq), beta_g1=z(1, 2 * nq), delta_g1=z(1, 2 * nq), beta_g2=z(1, ng2),
                   gamma_g2=z(1, ng2), delta_g2=z(1, ng2), gamma_abc_g1=z(m.num_instance_variables, 2 * nq))
        d = _lib.PkExportDesc()
        for k, v in out.items():
            setattr(d, k, _u64p(v) if v.size else None)
        flags = _lib.ZKEY_KEY_ONLY | (_lib.SER_VALIDATE if validate else 0)
        rc = self._lib.g16_zkey_load(self._ctx, buf.ctypes.data_as(C.c_void_p) if buf.size else None, buf.size, flags, rank,
                                     world, C.byref(d), None)
        if rc == _lib.ERR_INVALID_DATA and "(byte " in _lib.last_error():
            self._pk_resident = False
            self._pk_obj = None
        _check(rc)
        self._pk_resident = True
        self._pk_obj = None
        self.world = world
        vk = VerifyingKey(out["alpha_g1"][0], out["beta_g2"][0], out["gamma_g2"][0], out["delta_g2"][0], out["gamma_abc_g1"])
        vk.beta_g1, vk.delta_g1 = out["beta_g1"][0], out["delta_g1"][0]
        return vk

    # ---- circom .r1cs circuits and .wtns witnesses, decoded on the GPU ----
    def load_r1cs(self, data: bytes) -> R1csCircuit:
        """g16_r1cs_load: make the circuit of a circom .r1cs resident with all three matrices, under this context's qap, as
        load_matrices would the same terms (the GPU counterpart of ark-circom's R1CSFile + CircomCircuit).  Every call that
        reads C (check_witness, CHECK_WITNESS, generate_parameters_from_srs, key_verification_pairs) then works.  A
        malformed file raises serialize.DeserializeError naming the problem: the previous circuit and key stay resident
        when the structure or header is refused, none when a term is."""
        buf = np.frombuffer(data, dtype=np.uint8)
        info = _lib.R1csInfo()
        rc = self._lib.g16_r1cs_load(self._ctx, _lib.QAPS[self.qap], buf.ctypes.data_as(C.c_void_p) if buf.size else None,
                                     buf.size, C.byref(info))
        if rc == _lib.ERR_INVALID_DATA and "(byte " in _lib.last_error():
            self._matrices = None
            self._pk_resident = False
            self._pk_obj = None
        _check(rc)
        self._matrices = R1csCircuit(info.num_inputs, info.num_constraints, info.num_witness, info.log_n, info.a_nnz,
                                     info.b_nnz, info.c_nnz)
        self._pk_resident = False
        self._pk_obj = None
        return self._matrices

    def read_wtns(self, data: bytes) -> np.ndarray:
        """g16_wtns_read: the witness of a circom .wtns as (n, nr) Montgomery limbs, usable directly as full_assignment.  A
        malformed file or element raises serialize.DeserializeError naming it.  Needs no circuit; touches no resident state."""
        buf = np.frombuffer(data, dtype=np.uint8)
        ptr = buf.ctypes.data_as(C.c_void_p) if buf.size else None
        n = C.c_uint64()
        _check(self._lib.g16_wtns_read(self._ctx, ptr, buf.size, None, 0, C.byref(n)))
        out = np.zeros((n.value, self.nr), dtype=np.uint64)
        if n.value:
            _check(self._lib.g16_wtns_read(self._ctx, ptr, buf.size, _ptr(out), n.value, C.byref(n)))
        return out

    def export_proving_key_bytes(self, compress: bool = True) -> bytes:
        """g16_pk_export_serialized: the resident key (made by generate_parameters_with_qap) as ark-serialize writes it,
        byte for byte ArkCodec.proving_key of the exported limbs."""
        flags = _lib.SER_COMPRESSED if compress else 0
        n = C.c_uint64()
        _check(self._lib.g16_pk_export_serialized(self._ctx, flags, None, 0, C.byref(n)))
        out = np.zeros(n.value, dtype=np.uint8)
        _check(self._lib.g16_pk_export_serialized(self._ctx, flags, out.ctypes.data_as(C.c_void_p), out.size, C.byref(n)))
        return out.tobytes()

    # ---- prover.rs:26-51 ----
    def create_proof_with_reduction_and_matrices(self, pk: Optional[ProvingKey], r, s,
                                                 matrices: Optional[ConstraintMatrices], num_inputs: int,
                                                 num_constraints: int, full_assignment: np.ndarray,
                                                 flags: int = 0) -> Proof:
        """r, s, full_assignment: Montgomery Fr limbs (r, s may also be Python ints).  `pk` / `matrices` may be None
        to reuse what is already resident on the GPU."""
        if matrices is not None and matrices is not self._matrices:
            self.load_matrices(matrices)
        # the reference always proves under the `pk` argument (prover.rs:26): a key other than the resident one is loaded
        if pk is not None and (not self._pk_resident or pk is not self._pk_obj):
            self.load_proving_key(pk)
        m = self._matrices
        if m is None or not self._pk_resident:
            raise ValueError("matrices and proving key must be loaded")
        if num_inputs != m.num_instance_variables or num_constraints != m.num_constraints:
            raise ValueError("num_inputs / num_constraints do not match the matrices")
        rr = self._fr_arg(r)
        ss = self._fr_arg(s)
        z = np.ascontiguousarray(full_assignment, dtype=np.uint64).reshape(-1, self.nr)
        if z.shape[0] != m.num_instance_variables + m.num_witness_variables:
            raise ValueError("full_assignment has the wrong length")
        nq, ng2 = self.nq, self.ng2
        out = np.zeros(4 * nq + ng2, dtype=np.uint64)
        _check(self._lib.g16_prove(self._ctx, _ptr(rr), _ptr(ss), _ptr(z), flags, _ptr(out)))
        return Proof(out[:2 * nq].copy(), out[2 * nq:2 * nq + ng2].copy(), out[2 * nq + ng2:].copy())

    def prove_raw(self, r_limbs: np.ndarray, s_limbs: np.ndarray, z_ptr, flags: int, out: np.ndarray):
        """Thin call used by bench.py: everything already in ABI form; z_ptr is a host or device address."""
        _check(self._lib.g16_prove(self._ctx, _ptr(r_limbs), _ptr(s_limbs), C.c_void_p(z_ptr), flags, _ptr(out)))

    # ---- pipelined proving: two slots per context (g16_prove_submit / g16_prove_wait) ----
    def prove_submit_raw(self, slot: int, r_limbs: np.ndarray, s_limbs: np.ndarray, z_ptr, flags: int):
        """Enqueue a whole proof on `slot` and return; r/s/z buffers must stay alive until prove_wait_raw(slot)."""
        _check(self._lib.g16_prove_submit(self._ctx, slot, _ptr(r_limbs), _ptr(s_limbs), C.c_void_p(z_ptr), flags))

    def prove_wait_raw(self, slot: int, out: np.ndarray):
        _check(self._lib.g16_prove_wait(self._ctx, slot, _ptr(out)))

    # ---- batch proving: many proofs of the resident circuit in one call (g16_prove_batch) ----
    def create_proofs_batch(self, r, s, full_assignments: np.ndarray, group: int = 0, flags: int = 0) -> List[Proof]:
        """Proof i equals create_proof_with_reduction_and_matrices(None, r[i], s[i], None, ..., full_assignments[i]).
        r, s: sequences of ints or (K, 4) Montgomery limbs; full_assignments: (K, nv, 4) Montgomery limbs.  `group` caps the
        proofs that share one pass of the kernels (0 = as many as fit); results never depend on it."""
        m = self._matrices
        if m is None or not self._pk_resident:
            raise ValueError("matrices and proving key must be loaded")
        nv = m.num_instance_variables + m.num_witness_variables
        z = np.ascontiguousarray(full_assignments, dtype=np.uint64)
        if z.ndim != 3 or z.shape[1:] != (nv, self.nr):
            raise ValueError(f"full_assignments must have shape (K, {nv}, {self.nr})")
        k = z.shape[0]
        rr, ss = self._fr_args(r), self._fr_args(s)
        if rr.shape[0] != k or ss.shape[0] != k:
            raise ValueError("r, s and full_assignments must hold the same number of proofs")
        if not 0 <= group < 1 << 32:
            raise ValueError("group must be a non-negative 32-bit count")
        nq, ng2 = self.nq, self.ng2
        out = np.zeros((k, 4 * nq + ng2), dtype=np.uint64)
        if k:
            self.prove_batch_raw(k, rr, ss, z.ctypes.data, group, flags, out)
        return [Proof(p[:2 * nq].copy(), p[2 * nq:2 * nq + ng2].copy(), p[2 * nq + ng2:].copy()) for p in out]

    def prove_batch_raw(self, count: int, r_limbs: np.ndarray, s_limbs: np.ndarray, z_ptr, group: int, flags: int,
                        out: np.ndarray):
        """g16_prove_batch with everything in ABI form; z_ptr is a host or (G16_ASSIGNMENT_ON_DEVICE) device address of
        count * nv Montgomery Fr; out holds count * 8 * N64 limbs."""
        _check(self._lib.g16_prove_batch(self._ctx, count, _ptr(r_limbs), _ptr(s_limbs), C.c_void_p(z_ptr), group, flags,
                                         _ptr(out)))

    def prove_partial_submit_raw(self, slot: int, r_limbs: np.ndarray, z_ptr, flags: int):
        _check(self._lib.g16_prove_partial_submit(self._ctx, slot, _ptr(r_limbs), C.c_void_p(z_ptr), flags))

    def prove_partial_wait_raw(self, slot: int, out: np.ndarray):
        _check(self._lib.g16_prove_partial_wait(self._ctx, slot, _ptr(out)))

    def prove_partial_raw(self, r_limbs: np.ndarray, z_ptr, flags: int, out: np.ndarray):
        _check(self._lib.g16_prove_partial(self._ctx, _ptr(r_limbs), C.c_void_p(z_ptr), flags, _ptr(out)))

    # ---- sharded proving with the NCCL exchange inside the library ----
    def comm_unique_id(self) -> np.ndarray:
        out = np.zeros(256, dtype=np.uint8)
        _check(self._lib.g16_comm_unique_id(out.ctypes.data_as(C.c_void_p)))
        return out

    def comm_init(self, unique_id: np.ndarray, rank: int, world: int):
        uid = np.ascontiguousarray(unique_id, dtype=np.uint8)
        assert uid.size == 256
        _check(self._lib.g16_comm_init(self._ctx, uid.ctypes.data_as(C.c_void_p), rank, world))

    def prove_sharded_raw(self, r_limbs, s_limbs, z_ptr, flags: int, out: np.ndarray):
        _check(self._lib.g16_prove_sharded(self._ctx, _ptr(r_limbs), _ptr(s_limbs), C.c_void_p(z_ptr), flags, _ptr(out)))

    def prove_sharded_submit_raw(self, slot: int, r_limbs, s_limbs, z_ptr, flags: int):
        _check(self._lib.g16_prove_sharded_submit(self._ctx, slot, _ptr(r_limbs), _ptr(s_limbs), C.c_void_p(z_ptr), flags))

    def prove_sharded_wait_raw(self, slot: int, out: np.ndarray):
        _check(self._lib.g16_prove_sharded_wait(self._ctx, slot, _ptr(out)))

    def prove_assemble_prepare(self, r, s):
        """start the (r, s)-only scalar multiplications on a helper thread (overlaps GPU work and the gather)"""
        self._asm_keep = (self._fr_arg(r), self._fr_arg(s))
        _check(self._lib.g16_prove_assemble_prepare(self._ctx, _ptr(self._asm_keep[0]), _ptr(self._asm_keep[1])))

    def prove_assemble(self, r, s, partials: np.ndarray) -> Proof:
        rr, ss = self._fr_arg(r), self._fr_arg(s)
        pl = self._lib.g16_partial_limbs(self._ctx)
        p = np.ascontiguousarray(partials, dtype=np.uint64).reshape(-1, pl)
        nq, ng2 = self.nq, self.ng2
        out = np.zeros(4 * nq + ng2, dtype=np.uint64)
        _check(self._lib.g16_prove_assemble(self._ctx, _ptr(rr), _ptr(ss), _ptr(p), p.shape[0], _ptr(out)))
        return Proof(out[:2 * nq].copy(), out[2 * nq:2 * nq + ng2].copy(), out[2 * nq + ng2:].copy())

    def partial_limbs(self) -> int:
        return self._lib.g16_partial_limbs(self._ctx)

    def witness_map_from_matrices(self, matrices: Optional[ConstraintMatrices], num_inputs: int, num_constraints: int,
                                  full_assignment: np.ndarray, flags: int = 0) -> np.ndarray:
        """R1CSToQAP::witness_map_from_matrices (r1cs_to_qap.rs:172-235) -> domain_size Montgomery Fr coefficients; with
        qap="circom", CircomReduction's domain_size evaluations at the odd powers of omega_2n.  flags: 0 or CHECK_WITNESS."""
        if matrices is not None and matrices is not self._matrices:
            self.load_matrices(matrices)
        m = self._matrices
        z = np.ascontiguousarray(full_assignment, dtype=np.uint64).reshape(-1, self.nr)
        if z.shape[0] != m.num_instance_variables + m.num_witness_variables:
            raise ValueError("full_assignment has the wrong length")
        n = 1 << self._lib.g16_domain_log(self._ctx)
        h = np.zeros((n, self.nr), dtype=np.uint64)
        _check(self._lib.g16_witness_map(self._ctx, _ptr(z), flags, _ptr(h)))
        return h

    # ---- R1CS satisfiability (ark-relations ConstraintSystem::is_satisfied / which_is_unsatisfied), on the GPU ----
    def check_witness(self, full_assignments, count: Optional[int] = None, flags: int = 0) -> List[WitnessReport]:
        """g16_check_witness on the resident circuit: one report per assignment.  `full_assignments`: (nv, F) or (K, nv, F)
        Montgomery limbs, or a device address of `count` assignments together with flags = ASSIGNMENT_ON_DEVICE."""
        m = self._matrices
        if m is None:
            raise ValueError("load_matrices must come first")
        nv = m.num_instance_variables + m.num_witness_variables
        if isinstance(full_assignments, np.ndarray):
            z = np.ascontiguousarray(full_assignments, dtype=np.uint64)
            if z.ndim == 2:
                z = z.reshape(1, *z.shape)
            if z.ndim != 3 or z.shape[1:] != (nv, self.nr):
                raise ValueError(f"full_assignments must have shape (nv, {self.nr}) or (K, {nv}, {self.nr})")
            count, ptr = z.shape[0], z.ctypes.data
        else:
            if count is None:
                raise ValueError("a device address needs `count`")
            ptr = int(full_assignments)
        out = (_lib.WitnessReport * max(count, 1))()
        _check(self._lib.g16_check_witness(self._ctx, count, C.c_void_p(ptr), flags, out))
        none = lambda v: None if v == _lib.NONE else int(v)
        return [WitnessReport(none(w.first_unsatisfied), int(w.num_unsatisfied), none(w.first_malformed)) for w in out[:count]]

    def is_satisfied(self, full_assignment: np.ndarray) -> bool:
        """ConstraintSystem::is_satisfied for one assignment (a malformed element counts as unsatisfied)"""
        return self.check_witness(full_assignment)[0].ok

    def which_is_unsatisfied(self, full_assignment: np.ndarray) -> Optional[int]:
        """ConstraintSystem::which_is_unsatisfied: the lowest unsatisfied constraint, or None (there are no constraint
        names at this boundary).  A malformed assignment raises Unsatisfiable naming the element."""
        w = self.check_witness(full_assignment)[0]
        if w.first_malformed is not None:
            raise Unsatisfiable(f"assignment element {w.first_malformed} is " +
                                ("not One" if w.first_malformed == 0 else "not a canonical Fr"))
        return w.first_unsatisfied

    def timings(self) -> dict:
        t = _lib.Timings()
        _check(self._lib.g16_get_timings(self._ctx, C.byref(t)))
        names = ["h", "l", "a", "b_g1", "b_g2"]
        return dict(total_ms=t.total_ms, h2d_ms=t.h2d_ms, witness_map_ms=t.witness_map_ms,
                    msm_ms={n: t.msm_ms[i] for i, n in enumerate(names)},
                    msm_accum_ms={n: t.msm_accum_ms[i] for i, n in enumerate(names)},
                    msm_pairs={n: int(t.msm_pairs[i]) for i, n in enumerate(names)},
                    msm_entries={n: int(t.msm_entries[i]) for i, n in enumerate(names)},
                    msm_begin_ms={n: t.msm_begin_ms[i] for i, n in enumerate(names)},
                    msm_end_ms={n: t.msm_end_ms[i] for i, n in enumerate(names)},
                    host_finish_ms=t.host_finish_ms, launches=int(t.launches), h2d_bytes=int(t.h2d_bytes),
                    d2h_bytes=int(t.d2h_bytes))

    def set_option(self, key: str, value: int):
        """MSM launch-geometry knobs (g16_set_option; results never depend on them)."""
        _check(self._lib.g16_set_option(self._ctx, key.encode(), int(value)))

    def get_option(self, key: str) -> int:
        """g16_get_option: the value `key` holds now; set_option(key, get_option(key)) changes nothing."""
        v = C.c_int64()
        _check(self._lib.g16_get_option(self._ctx, key.encode(), C.byref(v)))
        return int(v.value)

    def config(self) -> dict:
        """Launch geometry of the resident key's MSMs plus two derived figures bench.py reports: the field products per
        bucket entry of the G1 accumulation stage (XYZZ mixed addition = 10; batched-affine addition = 6 + the combine's
        share) and the stage's name."""
        c = _lib.Config()
        _check(self._lib.g16_get_config(self._ctx, C.byref(c)))
        d = {n: int(getattr(c, n)) for n, _ in _lib.Config._fields_ if n != "reserved"}
        R = d["ba_rounds_g1"]
        ba_mul = 6.0 + 3.0 / max(1, d["ba_m"])            # forward 1 + backward 5 + combine 3 per thread product
        frac = 1.0 - 0.5 ** R
        d["imad_per_g1_entry_mul"] = frac * ba_mul + (1.0 - frac) * 10.0 if R > 0 else 10.0
        d["g1_accum_stage"] = (f"G1 bucket accumulation: {R} batched-affine rounds (ba_forward / ba_combine / ba_backward) + "
                               "msm_accum_l0<Fq> on the last list; one stage per G1 MSM" if R > 0 else
                               "msm_accum_l0<Fq> (G1 bucket accumulation, XYZZ mixed additions); one launch per G1 MSM")
        return d

    def _fr_arg(self, x) -> np.ndarray:
        if isinstance(x, (int, np.integer)):
            return np.ascontiguousarray(self.codec.fr.enc1(int(x)))
        return np.ascontiguousarray(x, dtype=np.uint64).reshape(self.nr)

    def _fr_args(self, xs) -> np.ndarray:
        """a sequence of ints, or a (K, nr) array of Montgomery limbs -> (K, nr) contiguous limbs"""
        if isinstance(xs, np.ndarray):
            a = np.ascontiguousarray(xs, dtype=np.uint64)
            if a.ndim != 2 or a.shape[1] != self.nr:
                raise ValueError(f"scalar limbs must have shape (K, {self.nr})")
            return a
        xs = list(xs)
        if not xs:
            return np.zeros((0, self.nr), dtype=np.uint64)
        return np.ascontiguousarray(np.stack([self._fr_arg(x) for x in xs]), dtype=np.uint64)
