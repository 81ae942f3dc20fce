"""GPU tier of CircomReduction (Groth16(curve, qap="circom") / g16_circuit_load_qap; run on an H100 with `pytest -m gpu`).

g16_witness_map against the oracle restatement (qap_circom_ref.py) from log n = 1 to 13 and on the three-pass NTT plan
(2^18, 2^20), satisfying and unsatisfying assignments, three curves.  Keys and proofs against the LibsnarkReduction path,
which the rest of the suite pins to the CPU oracle: with the same toxic waste every query but H is the same bytes, H is the
oracle's scalars times G1, and the proof of a satisfying witness is byte-identical under the two reductions (see
test_qap_circom.py) on every prover path -- single, two slots, batch, host-plumbed shards -- and verifies under the pairing."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import orc
import pyref as P
import qap_circom_ref as Q
from groth16_b200 import ConstraintMatrices, Groth16, PolynomialDegreeTooLarge, _lib
from groth16_b200.params import GENERATORS
from groth16_b200.workload import dummy_r1cs, synthetic_r1cs
from util import ALL_CURVES, matrices_from_r1cs, proof_from_abi

pytestmark = pytest.mark.gpu

TOXIC = (0x1111111111111111111111, 0x2222222222222222222223, 0x3333333333333333333335, 0x4444444444444444444447,
         0x5555555555555555555559)
THREADS = 16
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_ENG = {}


def engine(curve, qap) -> Groth16:
    """one context per reduction, for one curve at a time (2^20 keys of three curves at once would crowd the device)"""
    for key in [k for k in _ENG if k[0] != curve]:
        _ENG.pop(key).close()
    if (curve, qap) not in _ENG:
        _ENG[(curve, qap)] = Groth16(curve, 0, qap=qap)
    return _ENG[(curve, qap)]


@pytest.fixture(scope="module", autouse=True)
def _engines():
    yield
    for g in _ENG.values():
        g.close()
    _ENG.clear()


def flat(pf):
    return np.concatenate([pf.a, pf.b, pf.c])


def setup(g, m, gens=None):
    G = GENERATORS[g.curve.name]
    g1, g2 = gens or (G["g1"], G["g2"])
    return g.generate_parameters_with_qap(m, *TOXIC, g1, g2, export=True)


def prove(g, m, z, r, s, flags=0):
    return flat(g.create_proof_with_reduction_and_matrices(None, r, s, None, m.num_instance_variables, m.num_constraints,
                                                          np.ascontiguousarray(z), flags))


def vk_from_abi(curve, pk):
    cd = engine(curve, "circom").codec
    vk = pk.vk
    return P.VerifyingKey(cd.dec_g1(vk.alpha_g1)[0], cd.dec_g2(vk.beta_g2)[0], cd.dec_g2(vk.gamma_g2)[0],
                          cd.dec_g2(vk.delta_g2)[0], cd.dec_g1(vk.gamma_abc_g1))


def perturbed(cd, z, idx):
    zi = cd.fr.dec(z)
    zi[idx] = (zi[idx] + 1) % cd.c.r
    return np.ascontiguousarray(cd.fr.enc(zi))


def small_circuit(c, log_n, seed):
    """a satisfying circuit whose domain is exactly 2^log_n"""
    if log_n == 1:
        return P.synthetic_circuit(c, 1, seed=seed, num_inputs=0)
    return P.synthetic_circuit(c, (1 << log_n) - 2, seed=seed, num_inputs=1)


@pytest.mark.parametrize("curve", ALL_CURVES)
@pytest.mark.parametrize("log_n", list(range(1, 14)))
def test_witness_map_small(curve, log_n):
    g = engine(curve, "circom")
    cd = g.codec
    cs = small_circuit(P.CURVES[curve], log_n, seed=60 + log_n)
    assert cs.is_satisfied()
    m = matrices_from_r1cs(cs)
    z = np.ascontiguousarray(cd.fr.enc(cs.assignment))
    for zz in (z, perturbed(cd, z, len(cs.assignment) - 1)):
        got = g.witness_map_from_matrices(m, m.num_instance_variables, m.num_constraints, zz)
        assert got.shape == (1 << log_n, 4)
        assert np.array_equal(got, Q.orc_witness_map(cd, m, zz, threads=THREADS)), (curve, log_n)
    if log_n <= 6:   # and the big-integer restatement directly
        assert cd.fr.dec(g.witness_map_from_matrices(m, m.num_instance_variables, m.num_constraints, z)) == Q.witness_map(cs)


@pytest.mark.parametrize("curve", ALL_CURVES)
@pytest.mark.parametrize("log_n", [18, 20])
def test_witness_map_three_pass_plan(curve, log_n):
    g = engine(curve, "circom")
    cd = g.codec
    m, z, _ = synthetic_r1cs(curve, log_n, seed=70 + log_n)
    zbad = perturbed(cd, z, 7)   # C z != a o b on the rows that read z[7]
    for zz in (z, zbad):
        got = g.witness_map_from_matrices(m, m.num_instance_variables, m.num_constraints, zz)
        assert np.array_equal(got, Q.orc_witness_map(cd, m, zz, threads=THREADS)), (curve, log_n)


@pytest.mark.parametrize("curve", ALL_CURVES)
def test_setup_and_proofs_2p20(curve):
    gl, gc = engine(curve, "libsnark"), engine(curve, "circom")
    cd = gc.codec
    c = P.CURVES[curve]
    m, z, pub = synthetic_r1cs(curve, 20, seed=80)
    n = 1 << 20
    pk_l, pk_c = setup(gl, m), setup(gc, m)
    for f in ("a_query", "b_g1_query", "b_g2_query", "l_query", "beta_g1", "delta_g1"):
        assert np.array_equal(getattr(pk_l, f), getattr(pk_c, f)), f
    for f in ("alpha_g1", "beta_g2", "gamma_g2", "delta_g2", "gamma_abc_g1"):
        assert np.array_equal(getattr(pk_l.vk, f), getattr(pk_c.vk, f)), f
    assert pk_l.h_query.shape[0] == n - 1 and pk_c.h_query.shape[0] == n
    hs = Q.orc_h_query_scalars(cd, 20, TOXIC[4], pow(TOXIC[3], -1, c.r), threads=THREADS)
    idx = [0, 1, 2, n // 2, n - 2, n - 1] + [int(i) for i in np.random.default_rng(81).integers(0, n, 10)]
    g1 = cd.enc_g1([GENERATORS[curve]["g1"]])[0]
    assert np.array_equal(pk_c.h_query[idx], orc.batch_mul_g1(c.cid, cd.nq, g1, hs[idx]))
    vk = vk_from_abi(curve, pk_c)
    rng = P.Rng(82)
    for r_, s_ in ((rng.fr(c.r), rng.fr(c.r)), (0, rng.fr(c.r))):   # r = 0: B in G1 skipped (prover.rs:98)
        pf_c = prove(gc, m, z, r_, s_)
        assert np.array_equal(pf_c, prove(gl, m, z, r_, s_)), (curve, r_)
    pf = proof_from_abi(curve, gc.create_proof_with_reduction_and_matrices(None, r_, s_, None, m.num_instance_variables,
                                                                         m.num_constraints, z))
    assert P.verify_proof(vk, c, pf, list(pub))
    assert not P.verify_proof(vk, c, pf, [(pub[0] + 1) % c.r])
    # an unsatisfying assignment: the circom proof differs from the libsnark one and is rejected
    zbad = perturbed(cd, z, 5)
    bad = prove(gc, m, zbad, 3, 4)
    assert not np.array_equal(bad, prove(gl, m, zbad, 3, 4))
    nq = gc.nq
    pfb = P.Proof(cd.dec_g1(bad[:2 * nq])[0], cd.dec_g2(bad[2 * nq:6 * nq])[0], cd.dec_g1(bad[6 * nq:])[0])
    assert not P.verify_proof(vk, c, pfb, list(pub))

    # two slots in flight, then a batch (groups of 1, 2 and all; the assignments also from device memory)
    k = 3
    rr = np.ascontiguousarray(cd.fr.enc([rng.fr(c.r) for _ in range(k)]))
    ss = np.ascontiguousarray(cd.fr.enc([rng.fr(c.r) for _ in range(k)]))
    zs = np.ascontiguousarray(np.stack([z, zbad, z]))
    singles = [prove(gc, m, zs[i], rr[i], ss[i]) for i in range(k)]
    outs = [np.zeros(8 * nq, dtype=np.uint64) for _ in range(2)]
    gc.prove_submit_raw(0, rr[0], ss[0], zs[0].ctypes.data, 0)
    gc.prove_submit_raw(1, rr[1], ss[1], zs[1].ctypes.data, 0)
    gc.prove_wait_raw(0, outs[0])
    gc.prove_wait_raw(1, outs[1])
    assert np.array_equal(outs[0], singles[0]) and np.array_equal(outs[1], singles[1])
    for group in (1, 2, 0):
        got = gc.create_proofs_batch(rr, ss, zs, group=group)
        for i in range(k):
            assert np.array_equal(flat(got[i]), singles[i]), (curve, group, i)
    import torch
    dz = torch.from_numpy(zs.view(np.int64).reshape(-1)).to("cuda:0")
    torch.cuda.synchronize()
    out = np.zeros((k, 8 * nq), dtype=np.uint64)
    gc.prove_batch_raw(k, rr, ss, dz.data_ptr(), 0, _lib.ASSIGNMENT_ON_DEVICE, out)
    for i in range(k):
        assert np.array_equal(out[i], singles[i])
    del dz


@pytest.mark.parametrize("curve", ALL_CURVES)
def test_dummy_circuit_2p20(curve):
    """benches/bench.rs's DummyCircuit: degenerate queries, constant witness; r = 0 included"""
    gl, gc = engine(curve, "libsnark"), engine(curve, "circom")
    m, z, _ = dummy_r1cs(curve, 1 << 19, (1 << 20) - 2, seed=83)
    setup(gl, m)
    setup(gc, m)
    for r_, s_ in ((11, 12), (0, 13)):
        assert np.array_equal(prove(gc, m, z, r_, s_), prove(gl, m, z, r_, s_)), (curve, r_)


@pytest.mark.parametrize("curve", ALL_CURVES)
def test_batch_three_vectors_per_launch_2p18(curve):
    """the three-pass plan with several vectors per launch (vstride)"""
    gc = engine(curve, "circom")
    cd = gc.codec
    c = P.CURVES[curve]
    m, z, _ = synthetic_r1cs(curve, 18, seed=84)
    setup(gc, m)
    rng = P.Rng(85)
    rr = np.ascontiguousarray(cd.fr.enc([rng.fr(c.r) for _ in range(3)]))
    ss = np.ascontiguousarray(cd.fr.enc([rng.fr(c.r) for _ in range(3)]))
    zs = np.ascontiguousarray(np.stack([z, perturbed(cd, z, 9), perturbed(cd, z, 100)]))
    got = gc.create_proofs_batch(rr, ss, zs, group=3)
    for i in range(3):
        assert np.array_equal(flat(got[i]), prove(gc, m, zs[i], rr[i], ss[i])), (curve, i)


def _edge_circuits(c):
    rng = P.Rng(86)
    a, b = rng.fr(c.r), rng.fr(c.r)
    no_public = P.R1CS(c, 1, 3, [[(1, 1)]] * 3, [[(1, 2)]] * 3, [[(1, 3)]] * 3, [1, a, b, a * b % c.r])
    single = P.R1CS(c, 2, 2, [[(1, 2)]], [[(1, 3)]], [[(1, 1)]], [1, a * b % c.r, a, b])
    return {"no_public_inputs": no_public, "exact_power_of_two": P.synthetic_circuit(c, 62, seed=87, num_inputs=1),
            "all_zero_witness": P.silly_circuit(c, 0, 0), "single_constraint": single}


@pytest.mark.parametrize("curve", ALL_CURVES)
@pytest.mark.parametrize("which", ["no_public_inputs", "exact_power_of_two", "all_zero_witness", "single_constraint"])
def test_edge_circuits(curve, which):
    c = P.CURVES[curve]
    cs = _edge_circuits(c)[which]
    assert cs.is_satisfied()
    gl, gc = engine(curve, "libsnark"), engine(curve, "circom")
    cd = gc.codec
    m = matrices_from_r1cs(cs)
    z = np.ascontiguousarray(cd.fr.enc(cs.assignment))
    cx = P.ctx(c)
    gens = (cx.g1_gen(), cx.g2_gen())   # pyref's generators, so that its key below is the same
    setup(gl, m, gens)
    pk_c = setup(gc, m, gens)
    assert cd.fr.dec(gc.witness_map_from_matrices(m, m.num_instance_variables, m.num_constraints, z)) == Q.witness_map(cs)
    # the key against the big-integer restatement
    want = Q.generate_parameters(cs, *TOXIC, qap="circom")
    assert cd.dec_g1(pk_c.h_query) == want.h_query
    rng = P.Rng(88)
    for r_, s_ in ((rng.fr(c.r), rng.fr(c.r)), (0, rng.fr(c.r))):
        pf_c = prove(gc, m, z, r_, s_)
        assert np.array_equal(pf_c, prove(gl, m, z, r_, s_)), (curve, which, r_)
    pf = proof_from_abi(curve, gc.create_proof_with_reduction_and_matrices(None, r_, s_, None, m.num_instance_variables,
                                                                         m.num_constraints, z))
    want_pf = Q.create_proof(want, cs, r_, s_, qap="circom")
    assert (pf.a, pf.b, pf.c) == (want_pf.a, want_pf.b, want_pf.c)
    assert P.verify_proof(want.vk, c, pf, cs.assignment[1:cs.num_instance])


@pytest.mark.parametrize("world", [2, 3])
def test_host_plumbed_shards(world):
    curve = "bls12_381"
    gc = engine(curve, "circom")
    cd = gc.codec
    m, z, _ = synthetic_r1cs(curve, 12, seed=89)
    pk = setup(gc, m)
    r_, s_ = 1234567, 7654321
    single = prove(gc, m, z, r_, s_)
    rl = np.ascontiguousarray(cd.fr.enc1(r_))
    parts = []
    for rank in range(world):
        gc.load_proving_key(pk, rank, world)
        out = np.zeros(gc.partial_limbs(), dtype=np.uint64)
        gc.prove_partial_raw(rl, z.ctypes.data, 0, out)
        parts.append(out)
    assert np.array_equal(flat(gc.prove_assemble(r_, s_, np.stack(parts))), single)
    gc.load_proving_key(pk, 0, 1)


def test_errors_and_switching_reductions():
    with pytest.raises(ValueError):
        Groth16("bn254", 0, qap="snarkjs")
    g = engine("bn254", "circom")
    cd = g.codec
    m, z, _ = synthetic_r1cs("bn254", 10, seed=90)
    setup(g, m)
    before = prove(g, m, z, 5, 6)
    # an unknown reduction at the C ABI, and BN254 at nc + ni > 2^27 (the size-2n domain would need two-adicity 29): both
    # refused from the sizes alone -- row_ptr is 2^27 + 1 zero pages never touched -- and the resident circuit survives
    nc = 1 << 27
    rp = np.zeros(nc + 1, dtype=np.uint32)
    empty = _lib.Csr()
    empty.row_ptr = rp.ctypes.data_as(_lib.u32p)
    empty.col = None
    empty.val = None
    for qap, rc in ((7, _lib.ERR_BAD_ARGUMENT), (-1, _lib.ERR_BAD_ARGUMENT), (_lib.QAP_CIRCOM, _lib.ERR_POLYNOMIAL_DEGREE_TOO_LARGE)):
        assert g._lib.g16_circuit_load_qap(g._ctx, qap, 2, nc, 1, C.byref(empty), C.byref(empty), C.byref(empty)) == rc, qap
    assert np.array_equal(prove(g, m, z, 5, 6), before)
    huge = ConstraintMatrices(2, 1, nc, (rp, np.zeros(0, np.uint32), np.zeros((0, 4), np.uint64)),
                              (rp, np.zeros(0, np.uint32), np.zeros((0, 4), np.uint64)),
                              (rp, np.zeros(0, np.uint32), np.zeros((0, 4), np.uint64)))
    with pytest.raises(PolynomialDegreeTooLarge):
        g.load_matrices(huge)
    # a LibsnarkReduction circuit loaded on the same context after a CircomReduction one proves exactly as before
    gl = engine("bn254", "libsnark")
    setup(gl, m)
    want = prove(gl, m, z, 5, 6)
    zbad = perturbed(cd, z, 3)
    want_bad = prove(gl, m, zbad, 5, 6)
    want_h = gl.witness_map_from_matrices(m, m.num_instance_variables, m.num_constraints, zbad)
    g.qap = "libsnark"
    try:
        pk = setup(g, m)
        assert pk.h_query.shape[0] == (1 << 10) - 1
        assert np.array_equal(prove(g, m, z, 5, 6), want)
        assert np.array_equal(prove(g, m, zbad, 5, 6), want_bad)
        assert np.array_equal(g.witness_map_from_matrices(m, m.num_instance_variables, m.num_constraints, zbad), want_h)
    finally:
        g.qap = "circom"
    setup(g, m)
    assert np.array_equal(prove(g, m, z, 5, 6), before)


def _ngpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def test_sharded_wm_split_over_nccl():
    """g16_prove_sharded with "wm_split": chains a, b, c on ranks 0, 1, 2 mod world, the pointwise step on rank 3 mod world"""
    n = min(_ngpus(), 4)
    if n < 2:
        pytest.skip("needs at least 2 GPUs (the witness-map exchange is NCCL send / recv between processes)")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29537", os.path.join(ROOT, "tools", "sharded_check.py"), "bn254", "14", "circom"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and f"SHARDED_OK world={n}" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
