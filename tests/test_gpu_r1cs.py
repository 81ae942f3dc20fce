"""GPU tier of circom .r1cs / .wtns loading (Groth16.load_r1cs / g16_r1cs_load, Groth16.read_wtns / g16_wtns_read, and
Groth16.load_zkey_key / g16_zkey_load with G16_ZKEY_KEY_ONLY; run on an H100 with `pytest -m gpu`).

Circuits are written as .r1cs by tests/r1cs_ref.py (an independent writer of the format) and loaded with g16_r1cs_load.
Everything must be bit-identical to a second context holding the same matrices through g16_circuit_load_qap: proofs on
every path, witness maps, witness checks, g16_setup and g16_setup_from_srs keys and g16_pk_verify_pairs outputs.  One
curve's contexts at a time.  PARITY UNPINNED BY CIRCOM: the format is pinned by r1cs_ref's restatement and by proofs that
verify under pyref's pairing."""
import ctypes as C
import gc
import struct

import numpy as np
import pytest

import pyref as P
import r1cs_ref as R
import zkey_ref as Z
from groth16_b200 import Groth16, MalformedKey, Unsatisfiable, _lib
from groth16_b200.params import GENERATORS
from groth16_b200.serialize import DeserializeError
from groth16_b200.workload import synthetic_r1cs
from util import matrices_from_r1cs, pk_from_abi, proof_from_abi

pytestmark = pytest.mark.gpu

CURVES = ["bn254", "bls12_381", "bls12_377", "bw6_761"]
QAPS = ["libsnark", "circom"]
TOXIC = (0x1111111111111111111111, 0x2222222222222222222223, 0x3333333333333333333335, 0x4444444444444444444447,
         0x5555555555555555555559)
CHUNK = 1 << 17   # terms per staging chunk (Engine::SER_CHUNK)
_ENG = {}


def engine(curve, qap, which) -> Groth16:
    """contexts of one curve and reduction at a time: "ref" holds matrices, "r1" loads .r1cs files, "zk" full .zkey files"""
    for key in [k for k in _ENG if k[:2] != (curve, qap)]:
        _ENG.pop(key).close()
    if (curve, qap, which) not in _ENG:
        _ENG[(curve, qap, which)] = Groth16(curve, 0, qap=qap)
    return _ENG[(curve, qap, which)]


@pytest.fixture(scope="module", autouse=True)
def _engines():
    yield
    for g in _ENG.values():
        g.close()
    _ENG.clear()


def flat(pf):
    return np.concatenate([pf.a, pf.b, pf.c])


def gens(curve):
    G = GENERATORS[curve]
    return G["g1"], G["g2"]


def circuit(curve, name):
    """(ConstraintMatrices, full assignment in limbs) of a named circuit; the pyref ones exist on the three pyref curves"""
    if name.isdigit():
        m, z, _ = synthetic_r1cs(curve, int(name), seed=40 + int(name))
        return m, np.ascontiguousarray(z)
    if curve not in P.CURVES:
        pytest.skip("pyref circuits are not defined on " + curve)
    c = P.CURVES[curve]
    if name == "silly":
        cs = P.silly_circuit(c, 3, 11)
    elif name == "mimc":
        rng = P.Rng(5)
        cs = P.mimc_circuit(c, rng.fr(c.r), rng.fr(c.r), [rng.fr(c.r) for _ in range(P.MIMC_ROUNDS)])
    else:
        cs = P.synthetic_circuit(c, 5, seed=7, num_inputs=0)
    assert cs.is_satisfied()
    return matrices_from_r1cs(cs), np.ascontiguousarray(_codec(curve).fr.enc(cs.assignment))


def _codec(curve):
    from groth16_b200 import CurveCodec, get_curve
    return CurveCodec(get_curve(curve))


def unsat(cd, z, k=-1):
    zi = cd.fr.dec(z)
    zi[k] = (zi[k] + 1) % cd.c.r
    return np.ascontiguousarray(cd.fr.enc(zi))


def all_paths(g, ni, nc, z, r_, s_):
    """proof bytes on every prover path: single, both slots, batch (one group, groups of 2 and 1)"""
    cd = g.codec
    out = {"single": flat(g.create_proof_with_reduction_and_matrices(None, r_, s_, None, ni, nc, z))}
    rl, sl = np.ascontiguousarray(cd.fr.enc1(r_)), np.ascontiguousarray(cd.fr.enc1(s_))
    for slot in (0, 1):
        buf = np.zeros_like(out["single"])
        g.prove_submit_raw(slot, rl, sl, z.ctypes.data, 0)
        g.prove_wait_raw(slot, buf)
        out[f"slot{slot}"] = buf
    zs = np.stack([z, z, z])
    for group in (0, 2, 1):
        out[f"batch{group}"] = np.stack([flat(p) for p in g.create_proofs_batch([r_] * 3, [s_] * 3, zs, group=group)])
    return out


def sharded(g, pk, r_, s_, z, world=3):
    """partial / assemble over `world` emulated ranks of the key pk"""
    rl = np.ascontiguousarray(g.codec.fr.enc1(r_))
    parts = []
    for rank in range(world):
        g.load_proving_key(pk, rank, world)
        out = np.zeros(g.partial_limbs(), dtype=np.uint64)
        g.prove_partial_raw(rl, z.ctypes.data, 0, out)
        parts.append(out)
    pf = flat(g.prove_assemble(r_, s_, np.stack(parts)))
    g.load_proving_key(pk)
    return pf


def setup_resident(g):
    """g16_setup of the resident circuit with TOXIC, exported"""
    cd = g.codec
    sc = [np.ascontiguousarray(cd.fr.enc1(x)) for x in TOXIC]
    g1, g2 = gens(g.curve.name)
    G1, G2 = np.ascontiguousarray(cd.enc_g1([g1])[0]), np.ascontiguousarray(cd.enc_g2([g2])[0])
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = g._lib.g16_setup(g._ctx, *[ptr(x) for x in sc], ptr(G1), ptr(G2))
    assert rc == 0, _lib.last_error()
    g._pk_resident = True
    return g.export_proving_key()


def same_key(a, b):
    for name in ("beta_g1", "delta_g1", "a_query", "b_g1_query", "b_g2_query", "h_query", "l_query"):
        assert np.array_equal(np.asarray(getattr(a, name)), np.asarray(getattr(b, name))), name
    for name in ("alpha_g1", "beta_g2", "gamma_g2", "delta_g2", "gamma_abc_g1"):
        assert np.array_equal(np.asarray(getattr(a.vk, name)), np.asarray(getattr(b.vk, name))), name


def reports(g, z):
    return [(w.first_unsatisfied, w.num_unsatisfied, w.first_malformed) for w in g.check_witness(z)]


def compare(curve, qap, m, z, data, deep=True):
    """load m as limbs ("ref") and `data` as .r1cs ("r1"); every output of both must be bit-identical"""
    gr, g1 = engine(curve, qap, "ref"), engine(curve, qap, "r1")
    pk = gr.generate_parameters_with_qap(m, *TOXIC, *gens(curve), export=True)
    info = g1.load_r1cs(data)
    assert (info.num_instance_variables, info.num_constraints, info.num_witness_variables) == \
        (m.num_instance_variables, m.num_constraints, m.num_witness_variables)
    assert info.log_n == gr._lib.g16_domain_log(gr._ctx)
    g1.load_proving_key(pk)
    cd = gr.codec
    rng = P.Rng(90)
    r_, s_ = rng.fr(cd.c.r), rng.fr(cd.c.r)
    ni, nc = m.num_instance_variables, m.num_constraints
    if not deep:
        assert np.array_equal(flat(g1.create_proof_with_reduction_and_matrices(None, r_, s_, None, ni, nc, z)),
                              flat(gr.create_proof_with_reduction_and_matrices(None, r_, s_, None, ni, nc, z)))
        assert np.array_equal(g1.witness_map_from_matrices(None, 0, 0, z), gr.witness_map_from_matrices(None, 0, 0, z))
        return info
    want, got = all_paths(gr, ni, nc, z, r_, s_), all_paths(g1, ni, nc, z, r_, s_)
    for k in want:
        assert np.array_equal(got[k], want[k]), k
    assert np.array_equal(sharded(g1, pk, r_, s_, z), sharded(gr, pk, r_, s_, z))
    bad = unsat(cd, z)
    for zz in (z, bad):
        assert np.array_equal(g1.witness_map_from_matrices(None, 0, 0, zz), gr.witness_map_from_matrices(None, 0, 0, zz))
        assert reports(g1, zz) == reports(gr, zz)
    assert reports(g1, z)[0][1] == 0
    if reports(gr, bad)[0][1]:
        msgs = []
        for g in (gr, g1):
            with pytest.raises(Unsatisfiable) as e:
                g.create_proof_with_reduction_and_matrices(None, r_, s_, None, ni, nc, bad, flags=_lib.CHECK_WITNESS)
            msgs.append(str(e.value))
        assert msgs[0] == msgs[1]
    # keys: g16_setup, g16_setup_from_srs, and the key check of the transcript key
    same_key(setup_resident(g1), setup_resident(gr))
    n = 1 << info.log_n
    srs = gr.srs_from_secrets(2 * n - 1, n, TOXIC[4], TOXIC[0], TOXIC[1], *gens(curve))
    ka, kb = g1.generate_parameters_from_srs(None, srs), gr.generate_parameters_from_srs(None, srs)
    same_key(ka, kb)
    gr.load_matrices(m)   # the key check wants a resident circuit and no key
    g1.load_r1cs(data)
    pa = g1.key_verification_pairs(ka, srs, 0x1234567, uncontributed=True)
    pb = gr.key_verification_pairs(kb, srs, 0x1234567, uncontributed=True)
    assert np.array_equal(pa.g1, pb.g1) and np.array_equal(pa.g2, pb.g2)
    return info


@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("qap", QAPS)
@pytest.mark.parametrize("name", ["silly", "mimc", "npub0", "6", "9", "12"])
def test_matches_limbs_path(curve, qap, name):
    m, z = circuit(curve, name)
    c = R.Circuit.from_matrices(curve, m)
    info = compare(curve, qap, m, z, R.write(c))
    assert (info.a_nnz, info.b_nnz, info.c_nnz) == tuple(int(t[0][-1]) for t in (m.a, m.b, m.c))
    if name in ("silly", "9"):
        for data in (R.write(c, order=[3, 2, 1]), R.write(c, extra=[(7, b"x" * 9), (99, b"")], npubin=1),
                     R.write(c.transformed(split_seed=3)), R.write(c.transformed(zero_seed=4))):
            compare(curve, qap, m, z, data, deep=False)
    if curve in P.CURVES and name == "silly":
        # the pairing equations of the .r1cs circuit's key hold under pyref
        g1 = engine(curve, qap, "r1")
        g1.load_r1cs(R.write(c))
        pk = setup_resident(g1)
        pf = proof_from_abi(curve, g1.create_proof_with_reduction_and_matrices(None, 5, 6, None, 2, m.num_constraints, z))
        assert P.verify_proof(pk_from_abi(curve, pk).vk, P.CURVES[curve], pf, [33 % P.CURVES[curve].r])


@pytest.mark.parametrize("curve", CURVES)
def test_long_constraint(curve):
    """one constraint longer than a staging chunk"""
    m, z = circuit(curve, "6")
    c = R.Circuit.from_matrices(curve, m).transformed(long_row=(3, CHUNK + 77))
    compare(curve, "circom", m, z, R.write(c), deep=False)


@pytest.mark.parametrize("curve", CURVES)
def test_2_20(curve):
    """a 2^20 circuit: the proof and witness map after load_r1cs equal those after load_matrices of the same circuit and
    key.  One context does both in turn, and every other context of this module is closed first, so the test needs the
    device memory of one 2^20 prover only."""
    for key in list(_ENG):
        _ENG.pop(key).close()
    gc.collect()   # contexts other tests left for the collector
    m, z = circuit(curve, "20")
    data = R.write(R.Circuit.from_matrices(curve, m))
    g = engine(curve, "circom", "big")
    pk = g.generate_parameters_with_qap(m, *TOXIC, *gens(curve), export=True)
    ni, nc = m.num_instance_variables, m.num_constraints
    rng = P.Rng(92)
    r_, s_ = rng.fr(g.curve.r), rng.fr(g.curve.r)
    want = flat(g.create_proof_with_reduction_and_matrices(None, r_, s_, None, ni, nc, z))
    want_h = g.witness_map_from_matrices(None, 0, 0, z)
    info = g.load_r1cs(data)
    assert (info.num_instance_variables, info.num_constraints, info.num_witness_variables, info.log_n) == (ni, nc, m.num_witness_variables, 20)
    assert (info.a_nnz, info.b_nnz, info.c_nnz) == tuple(int(t[0][-1]) for t in (m.a, m.b, m.c))
    g.load_proving_key(pk)
    assert np.array_equal(flat(g.create_proof_with_reduction_and_matrices(None, r_, s_, None, ni, nc, z)), want)
    assert np.array_equal(g.witness_map_from_matrices(None, 0, 0, z), want_h)
    assert reports(g, z)[0][1] == 0
    _ENG.pop((curve, "circom", "big")).close()


def _patch(data, off, raw):
    b = bytearray(data)
    b[off:off + len(raw)] = raw
    return bytes(b)


@pytest.mark.parametrize("curve", CURVES)
def test_device_refusals(curve):
    m, z = circuit(curve, "17")
    c = R.Circuit.from_matrices(curve, m)
    data = R.write(c)
    g = engine(curve, "libsnark", "r1")
    cp = g.curve
    n8 = 8 * cp.fr_limbs
    tp = c.term_prefix()
    total = int(tp[-1])
    assert total > CHUNK + 2
    # global term t -> (constraint, matrix, index in the combination)
    def place(t):
        i = int(np.searchsorted(tp, t, side="right") - 1)
        k = t - int(tp[i])
        for mi in range(3):
            cnt = int(c.mats[mi][0][i + 1] - c.mats[mi][0][i])
            if k < cnt:
                return i, mi, k
            k -= cnt
    pk = engine(curve, "libsnark", "ref").generate_parameters_with_qap(m, *TOXIC, *gens(curve), export=True)
    for t in (0, CHUNK - 1, CHUNK, total - 1):
        i, mi, k = place(t)
        off = R.term_offset(data, i, mi, k)
        for what, raw, msg in (("wire", struct.pack("<I", c.ni + c.nw), f"wire {c.ni + c.nw} >= nWires {c.ni + c.nw}"),
                               ("coef", cp.r.to_bytes(n8, "little"), "coefficient is not below r")):
            bad = _patch(data, off if what == "wire" else off + 4, raw)
            g.load_r1cs(data)
            g.load_proving_key(pk)
            with pytest.raises(DeserializeError) as e:
                g.load_r1cs(bad)
            assert str(e.value) == f"constraint {i}, {'ABC'[mi]} term {k} (byte {off}): {msg}", (t, what)
            # nothing resident: the C side refuses a proof and a witness check
            out = np.zeros(4 * g.nq + g.ng2, dtype=np.uint64)
            rl = np.ascontiguousarray(g.codec.fr.enc1(1))
            assert g._lib.g16_prove(g._ctx, rl.ctypes.data_as(C.c_void_p), rl.ctypes.data_as(C.c_void_p),
                                    z.ctypes.data_as(C.c_void_p), 0, out.ctypes.data_as(C.c_void_p)) == _lib.ERR_BAD_ARGUMENT
    # each matrix refuses in turn, and the next load succeeds
    seen = set()
    for t in range(total):
        i, mi, k = place(t)
        if mi in seen:
            continue
        seen.add(mi)
        off = R.term_offset(data, i, mi, k)
        with pytest.raises(DeserializeError, match=f"{'ABC'[mi]} term {k} "):
            g.load_r1cs(_patch(data, off, struct.pack("<I", 0xFFFFFFFF)))
        if len(seen) == 3:
            break
    assert g.load_r1cs(data).num_constraints == m.num_constraints


@pytest.mark.parametrize("curve", CURVES)
def test_host_refusals_keep_state(curve):
    m, z = circuit(curve, "9")
    data = R.write(R.Circuit.from_matrices(curve, m))
    gr, g = engine(curve, "libsnark", "ref"), engine(curve, "libsnark", "r1")
    pk = gr.generate_parameters_with_qap(m, *TOXIC, *gens(curve), export=True)
    g.load_r1cs(data)
    g.load_proving_key(pk)
    ni, nc = m.num_instance_variables, m.num_constraints
    want = flat(gr.create_proof_with_reduction_and_matrices(None, 7, 8, None, ni, nc, z))
    h1 = R.sections(data)[1][0]
    for bad, exc in ((data[:-3], DeserializeError), (R.write(R.Circuit.from_matrices(curve, m), extra=[(4, b"")]), DeserializeError),
                     (_patch(data, h1 + 4, b"\0"), DeserializeError)):
        with pytest.raises(exc):
            g.load_r1cs(bad)
        assert np.array_equal(flat(g.create_proof_with_reduction_and_matrices(None, 7, 8, None, ni, nc, z)), want)
    rc = g._lib.g16_r1cs_load(g._ctx, 7, data, len(data), None)
    assert rc == _lib.ERR_BAD_ARGUMENT
    rc = g._lib.g16_r1cs_load(g._ctx, 0, None, len(data), None)
    assert rc == _lib.ERR_BAD_ARGUMENT
    assert np.array_equal(flat(g.create_proof_with_reduction_and_matrices(None, 7, 8, None, ni, nc, z)), want)


@pytest.mark.parametrize("curve", Z.SNARKJS_CURVES)
@pytest.mark.parametrize("name", ["silly", "9"])
def test_key_only_zkey(curve, name):
    m, z = circuit(curve, name)
    gr, g1, gz = (engine(curve, "circom", w) for w in ("ref", "r1", "zk"))
    pk = gr.generate_parameters_with_qap(m, *TOXIC, *gens(curve), export=True)
    zk = Z.write(curve, m, pk, shuffle_seed=3)
    g1.load_r1cs(R.write(R.Circuit.from_matrices(curve, m)))
    vk = g1.load_zkey_key(zk)
    for got, want in ((vk.alpha_g1, pk.vk.alpha_g1), (vk.gamma_g2, pk.vk.gamma_g2), (vk.gamma_abc_g1, pk.vk.gamma_abc_g1),
                      (vk.delta_g1, pk.delta_g1)):
        assert np.array_equal(np.asarray(got).ravel(), np.asarray(want).ravel())
    gz.load_zkey(zk)
    ni, nc = m.num_instance_variables, m.num_constraints
    rng = P.Rng(91)
    r_, s_ = rng.fr(gr.curve.r), rng.fr(gr.curve.r)
    want = all_paths(gr, ni, nc, z, r_, s_)
    for g in (g1, gz):
        got = all_paths(g, ni, nc, z, r_, s_)
        for k in want:
            assert np.array_equal(got[k], want[k]), k
    # C is resident: CHECK_WITNESS and check_witness name the first unsatisfied constraint
    bad = unsat(gr.codec, z)
    first = reports(gr, bad)[0][0]
    assert reports(g1, bad)[0][0] == first
    if first != _lib.NONE:
        with pytest.raises(Unsatisfiable, match=f"constraint {first}"):
            g1.create_proof_with_reduction_and_matrices(None, r_, s_, None, ni, nc, bad, flags=_lib.CHECK_WITNESS)
    # MALFORMED_KEY (a well-formed .zkey of another circuit) and a malformed file keep the previous key
    m2, _ = circuit(curve, "mimc" if name == "silly" else "6")
    zk2 = Z.write(curve, m2, gr.generate_parameters_with_qap(m2, *TOXIC, *gens(curve), export=True))
    h = Z.header(zk)
    for bad, exc, msg in ((zk2, MalformedKey, "section 2: nVars = "), (zk[:-1], DeserializeError, "truncated input"),
                          (_patch(zk, h["points"] - 4, struct.pack("<I", 2 * h["domain_size"])), DeserializeError, r"section 9 \(H\)")):
        with pytest.raises(exc, match=msg):
            g1.load_zkey_key(bad)
        assert np.array_equal(flat(g1.create_proof_with_reduction_and_matrices(None, r_, s_, None, ni, nc, z)), want["single"])
    gl = Groth16(curve, 0, qap="libsnark")
    try:
        assert gl._lib.g16_zkey_load(gl._ctx, zk, len(zk), _lib.ZKEY_KEY_ONLY, 0, 1, None, None) == _lib.ERR_BAD_ARGUMENT
        gl.load_matrices(m)
        assert gl._lib.g16_zkey_load(gl._ctx, zk, len(zk), _lib.ZKEY_KEY_ONLY, 0, 1, None, None) == _lib.ERR_BAD_ARGUMENT
        assert gl._lib.g16_zkey_load(gl._ctx, zk, len(zk), 8, 0, 1, None, None) == _lib.ERR_BAD_ARGUMENT
    finally:
        gl.close()
    # a refused point: the circuit stays, no key
    hoff = Z.sections(zk)[9][0] + 2 * 8 * gr.nq   # H[1]: one G1 point is 2 nq limbs
    with pytest.raises(DeserializeError, match=r"^H\[1\] \(byte \d+\): non-canonical"):
        g1.load_zkey_key(_patch(zk, hoff, gr.curve.q.to_bytes(8 * gr.nq, "little")))
    out = np.zeros(4 * gr.nq + gr.ng2, dtype=np.uint64)
    rl = np.ascontiguousarray(gr.codec.fr.enc1(1))
    assert g1._lib.g16_prove(g1._ctx, rl.ctypes.data_as(C.c_void_p), rl.ctypes.data_as(C.c_void_p), z.ctypes.data_as(C.c_void_p),
                             0, out.ctypes.data_as(C.c_void_p)) == _lib.ERR_BAD_ARGUMENT
    assert reports(g1, z)[0][1] == 0
    g1.load_zkey_key(zk, validate=False)
    assert np.array_equal(flat(g1.create_proof_with_reduction_and_matrices(None, r_, s_, None, ni, nc, z)), want["single"])


@pytest.mark.parametrize("curve", CURVES)
def test_read_wtns(curve):
    m, z = circuit(curve, "9")
    g = engine(curve, "libsnark", "r1")
    data = R.wtns_from_limbs(curve, z)
    got = g.read_wtns(data)
    assert got.shape == z.shape and np.array_equal(got, z)
    n = C.c_uint64()
    assert g._lib.g16_wtns_read(g._ctx, data, len(data), None, 0, C.byref(n)) == 0 and n.value == z.shape[0]
    small = np.zeros((2, g.nr), dtype=np.uint64)
    assert g._lib.g16_wtns_read(g._ctx, data, len(data), small.ctypes.data_as(C.c_void_p), 2, C.byref(n)) == _lib.ERR_BAD_ARGUMENT
    assert n.value == z.shape[0]
    g.load_r1cs(R.write(R.Circuit.from_matrices(curve, m)))
    assert reports(g, got)[0][1] == 0
    pk = engine(curve, "libsnark", "ref").generate_parameters_with_qap(m, *TOXIC, *gens(curve), export=True)
    g.load_proving_key(pk)
    ni, nc = m.num_instance_variables, m.num_constraints
    assert np.array_equal(flat(g.create_proof_with_reduction_and_matrices(None, 3, 4, None, ni, nc, got, flags=_lib.CHECK_WITNESS)),
                          flat(g.create_proof_with_reduction_and_matrices(None, 3, 4, None, ni, nc, z)))
    vals = R.read_wtns(curve, data)
    for k in (0, 17, len(vals) - 1):
        bad = list(vals)
        bad[k] = g.curve.r + k
        d = R.write_wtns(curve, bad)
        off = R.sections(d, b"wtns")[2][0] + k * 8 * g.nr
        with pytest.raises(DeserializeError, match=rf"^witness\[{k}\] \(byte {off}\): not below r$"):
            g.read_wtns(d)
    assert g.read_wtns(R.write_wtns(curve, [])).shape == (0, g.nr)


@pytest.mark.parametrize("curve", Z.SNARKJS_CURVES)
def test_circom_ceremony(curve):
    """load_r1cs, transcript, key from it, a contribution, export, .zkey; the key check on the .r1cs circuit holds under
    pyref's pairing, and a proof from the key-only .zkey load with CHECK_WITNESS verifies"""
    c = P.CURVES[curve]
    cs = P.silly_circuit(c, 3, 11)
    m = matrices_from_r1cs(cs)
    g = engine(curve, "circom", "r1")
    info = g.load_r1cs(R.write(R.Circuit.from_r1cs(cs)))
    n = 1 << info.log_n
    srs = g.srs_from_secrets(2 * n - 1, n, 0xABCDEF, 0x1357, 0x2468, *gens(curve))
    g.generate_parameters_from_srs(None, srs)
    pk = g.contribute_delta(0x777777)
    zk = Z.write(curve, m, pk)
    g.load_r1cs(R.write(R.Circuit.from_r1cs(cs)))   # the key check wants a resident circuit and no key
    pairs = g.key_verification_pairs(pk, srs, 0x31415926)
    cx = P.ctx(c)
    cd = g.codec
    ps, qs = cd.dec_g1(pairs.g1), cd.dec_g2(pairs.g2)
    for k in range(4):
        assert cx.pairing_product_is_one([(ps[2 * k], qs[2 * k]), (cx.G1.neg(ps[2 * k + 1]), qs[2 * k + 1])]), k
    vk = g.load_zkey_key(zk)
    z = g.read_wtns(R.write_wtns(curve, cs.assignment))
    pf = g.create_proof_with_reduction_and_matrices(None, 11, 12, None, cs.num_instance, cs.num_constraints, z,
                                                    flags=_lib.CHECK_WITNESS)
    rvk = P.VerifyingKey(cd.dec_g1(vk.alpha_g1)[0], cd.dec_g2(vk.beta_g2)[0], cd.dec_g2(vk.gamma_g2)[0],
                         cd.dec_g2(vk.delta_g2)[0], cd.dec_g1(vk.gamma_abc_g1))
    assert P.verify_proof(rvk, c, proof_from_abi(curve, pf), [33 % c.r])
    assert not P.verify_proof(rvk, c, proof_from_abi(curve, pf), [34])
