"""GPU tier of snarkjs .zkey loading (Groth16.load_zkey / g16_zkey_load; run on an H100 with `pytest -m gpu`).

A CircomReduction key is made with g16_setup and exported, written as a .zkey by tests/zkey_ref.py (an independent writer
of the format), and loaded with g16_zkey_load.  Proofs and witness maps must be bit-identical to a second context holding
the same circuit and key through g16_circuit_load_qap(CIRCOM) + g16_pk_load, on every prover path.  PARITY UNPINNED BY
SNARKJS: the format is pinned by zkey_ref's restatement and by proofs that verify under pyref's pairing."""
import struct

import numpy as np
import pytest

import pyref as P
import zkey_ref as Z
from groth16_b200 import Groth16, _lib
from groth16_b200.params import GENERATORS
from groth16_b200.serialize import DeserializeError
from groth16_b200.workload import synthetic_r1cs
from util import matrices_from_r1cs, proof_from_abi

pytestmark = pytest.mark.gpu

CURVES = list(Z.SNARKJS_CURVES)
TOXIC = (0x1111111111111111111111, 0x2222222222222222222223, 0x3333333333333333333335, 0x4444444444444444444447,
         0x5555555555555555555559)
_ENG = {}


def engine(curve, which) -> Groth16:
    """contexts of one curve at a time: "ref" holds matrices + limbs key, "zk" loads .zkey files"""
    for key in [k for k in _ENG if k[0] != curve]:
        _ENG.pop(key).close()
    if (curve, which) not in _ENG:
        _ENG[(curve, which)] = Groth16(curve, 0, qap="circom")
    return _ENG[(curve, which)]


@pytest.fixture(scope="module", autouse=True)
def _engines():
    yield
    for g in _ENG.values():
        g.close()
    _ENG.clear()


def flat(pf):
    return np.concatenate([pf.a, pf.b, pf.c])


def make(curve, m):
    """the CircomReduction key of m by g16_setup, resident in the "ref" context through g16_pk_load"""
    g = engine(curve, "ref")
    G = GENERATORS[g.curve.name]
    pk = g.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=True)
    g.load_proving_key(pk)
    return pk


def circuit(curve, name):
    c = P.CURVES[curve]
    if name == "silly":
        cs = P.silly_circuit(c, 3, 11)
    elif name == "mimc":
        rng = P.Rng(5)
        cs = P.mimc_circuit(c, rng.fr(c.r), rng.fr(c.r), [rng.fr(c.r) for _ in range(P.MIMC_ROUNDS)])
    elif name == "npub0":
        cs = P.synthetic_circuit(c, 5, seed=7, num_inputs=0)
    else:
        m, z, _ = synthetic_r1cs(curve, int(name), seed=40 + int(name))
        return m, np.ascontiguousarray(z)
    assert cs.is_satisfied()
    return matrices_from_r1cs(cs), np.ascontiguousarray(engine(curve, "ref").codec.fr.enc(cs.assignment))


def unsat(cd, z):
    zi = cd.fr.dec(z)
    zi[-1] = (zi[-1] + 1) % cd.c.r
    return np.ascontiguousarray(cd.fr.enc(zi))


def all_paths(g, m, z, r_, s_):
    """proof bytes on every prover path: single, both slots, batch (one group, groups of 2 and 1), 3 emulated ranks"""
    cd = g.codec
    ni, nc = m.num_instance_variables, m.num_constraints
    single = flat(g.create_proof_with_reduction_and_matrices(None, r_, s_, None, ni, nc, z))
    out = {"single": single}
    rl, sl = np.ascontiguousarray(cd.fr.enc1(r_)), np.ascontiguousarray(cd.fr.enc1(s_))
    for slot in (0, 1):
        buf = np.zeros_like(single)
        g.prove_submit_raw(slot, rl, sl, z.ctypes.data, 0)
        g.prove_wait_raw(slot, buf)
        out[f"slot{slot}"] = buf
    zs = np.stack([z, z, z])
    for group in (0, 2, 1):
        pfs = g.create_proofs_batch([r_] * 3, [s_] * 3, zs, group=group)
        out[f"batch{group}"] = np.stack([flat(p) for p in pfs])
    return out


def sharded(g, load, r_, s_, z, world=3):
    """partial / assemble over `world` emulated ranks; load(rank, world) makes that rank's shard resident"""
    cd = g.codec
    rl = np.ascontiguousarray(cd.fr.enc1(r_))
    parts = []
    for rank in range(world):
        load(rank, world)
        out = np.zeros(g.partial_limbs(), dtype=np.uint64)
        g.prove_partial_raw(rl, z.ctypes.data, 0, out)
        parts.append(out)
    pf = flat(g.prove_assemble(r_, s_, np.stack(parts)))
    load(0, 1)
    return pf


@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("name", ["silly", "mimc", "npub0", "6", "9", "12"])
def test_proofs_match_limbs_path(curve, name):
    m, z = circuit(curve, name)
    pk = make(curve, m)
    data = Z.write(curve, m, pk)
    gr, gz = engine(curve, "ref"), engine(curve, "zk")
    vk, info = gz.load_zkey(data)
    assert (info.num_instance_variables, info.num_constraints, info.num_witness_variables) == \
        (m.num_instance_variables, m.num_constraints, m.num_witness_variables)
    assert info.log_n == gr._lib.g16_domain_log(gr._ctx)
    assert (info.a_nnz, info.b_nnz) == (int(m.a[0][-1]), int(m.b[0][-1]))
    for got, want in ((vk.alpha_g1, pk.vk.alpha_g1), (vk.beta_g2, pk.vk.beta_g2), (vk.gamma_g2, pk.vk.gamma_g2),
                      (vk.delta_g2, pk.vk.delta_g2), (vk.gamma_abc_g1, pk.vk.gamma_abc_g1), (vk.beta_g1, pk.beta_g1),
                      (vk.delta_g1, pk.delta_g1)):
        assert np.array_equal(np.asarray(got).ravel(), np.asarray(want).ravel())
    cd = gr.codec
    c = P.CURVES[curve]
    rng = P.Rng(90)
    r_, s_ = rng.fr(c.r), rng.fr(c.r)
    want, got = all_paths(gr, m, z, r_, s_), all_paths(gz, info, z, r_, s_)
    for k in want:
        assert np.array_equal(got[k], want[k]), (curve, name, k)
    for zz in (z, unsat(cd, z)):
        assert np.array_equal(gz.witness_map_from_matrices(None, 0, 0, zz), gr.witness_map_from_matrices(None, 0, 0, zz))
        assert np.array_equal(flat(gz.create_proof_with_reduction_and_matrices(None, r_, s_, None, info.num_instance_variables,
                                                                               info.num_constraints, zz)),
                              flat(gr.create_proof_with_reduction_and_matrices(None, r_, s_, None, m.num_instance_variables,
                                                                               m.num_constraints, zz)))
    # partial / assemble over three emulated ranks, against the single proof
    pf = sharded(gz, lambda rank, world: gz.load_zkey(data, rank=rank, world=world), r_, s_, z)
    assert np.array_equal(pf, want["single"])
    if name in ("silly", "6"):   # and the proof verifies under the pairing, a wrong public input does not
        from util import pk_from_abi
        opk = pk_from_abi(curve, pk)
        proof = proof_from_abi(curve, gz.create_proof_with_reduction_and_matrices(None, r_, s_, None, info.num_instance_variables,
                                                                                 info.num_constraints, z))
        pub = cd.fr.dec(z)[1:m.num_instance_variables]
        assert P.verify_proof(opk.vk, c, proof, pub)
        assert not P.verify_proof(opk.vk, c, proof, [(pub[0] + 1) % c.r] + pub[1:])


@pytest.mark.parametrize("curve", CURVES)
def test_2_20_and_timings(curve):
    m, z = circuit(curve, "20")
    pk = make(curve, m)
    r_, s_ = 1234567, 7654321
    want = flat(engine(curve, "ref").create_proof_with_reduction_and_matrices(None, r_, s_, None, m.num_instance_variables,
                                                                              m.num_constraints, z))
    # one 2^20 context of this module at a time: the limbs context goes before the .zkey is loaded, so that the test does
    # not depend on how much memory the contexts of other modules leave free
    _ENG.pop((curve, "ref")).close()
    data = Z.write(curve, m, pk, shuffle_seed=3)
    gz = engine(curve, "zk")
    for validate in (False, True):
        _, info = gz.load_zkey(data, validate=validate)
        t = gz.timings()
        assert t["total_ms"] > 0 and t["h2d_bytes"] >= len(data) - 4096 and t["launches"] > 0
        assert np.array_equal(flat(gz.create_proof_with_reduction_and_matrices(None, r_, s_, None, info.num_instance_variables,
                                                                               info.num_constraints, z)), want)


@pytest.mark.parametrize("curve", CURVES)
def test_file_variants_prove_the_same(curve):
    m, z = circuit(curve, "mimc")
    pk = make(curve, m)
    gz = engine(curve, "zk")
    r_, s_ = 99, 101
    proofs = []
    for kw in ({}, {"shuffle_seed": 1}, {"order": [9, 3, 1, 7, 5, 2, 8, 4, 6]}, {"split_seed": 2, "shuffle_seed": 4},
               {"junk10": b"\x01" * 333}):
        _, info = gz.load_zkey(Z.write(curve, m, pk, **kw))
        proofs.append(flat(gz.create_proof_with_reduction_and_matrices(None, r_, s_, None, info.num_instance_variables,
                                                                       info.num_constraints, z)))
    for p in proofs[1:]:
        assert np.array_equal(p, proofs[0])


# ---- rejections -----------------------------------------------------------------------------------------------------
def _fixture(curve):
    m, z = circuit(curve, "9")
    pk = make(curve, m)
    return m, z, pk, Z.write(curve, m, pk)


def _resident_ok(g, info, z):
    """a proof runs on the resident circuit and key"""
    g.create_proof_with_reduction_and_matrices(None, 5, 6, None, info.num_instance_variables, info.num_constraints, z)


def _patch(data, off, raw):
    b = bytearray(data)
    b[off:off + len(raw)] = raw
    return bytes(b)


def _with_section(curve, m, pk, sid, body):
    """the file with section sid's body replaced"""
    data = Z.write(curve, m, pk)
    off, size = Z.sections(data)[sid]
    hdr = off - 12
    return data[:hdr] + struct.pack("<IQ", sid, len(body)) + body + data[off + size:]


def host_cases(curve, m, pk, data):
    cp = engine(curve, "zk").curve
    h = Z.header(data)
    off2, _ = Z.sections(data)[2]
    nq = h["n8q"]
    yield "magic", b"zkex" + data[4:], "not a .zkey file"
    yield "version", _patch(data, 4, struct.pack("<I", 2)), "unsupported .zkey version 2"
    yield "truncated", data[:-1], "truncated input"
    yield "trailing", data + b"\0", "trailing bytes"
    yield "missing", Z.write(curve, m, pk, order=[1, 2, 3, 4, 5, 6, 7, 8]), "section 9 is missing"
    yield "duplicate", Z.write(curve, m, pk, order=[1, 2, 3, 4, 5, 6, 7, 8, 9, 6]), "section 6 appears twice"
    yield "protocol", _patch(data, Z.sections(data)[1][0], struct.pack("<I", 2)), "protocol 2 is not Groth16"
    yield "n8q", _patch(data, off2, struct.pack("<I", nq + 16)), "n8q = "
    yield "q", _patch(data, off2 + 4, (cp.q + 2).to_bytes(nq, "little")), "q is not the base field modulus"
    yield "r", _patch(data, off2 + 8 + nq, (cp.r + 2).to_bytes(h["n8r"], "little")), "r is not the scalar field modulus"
    yield "nvars", _patch(data, h["points"] - 12, struct.pack("<I", 0)), "nVars = 0 is below"
    yield "domain", _patch(data, h["points"] - 4, struct.pack("<I", h["domain_size"] + 1)), "is not a power of two"
    yield "size3", _with_section(curve, m, pk, 3, np.ascontiguousarray(pk.vk.gamma_abc_g1).tobytes()[:-8]), "section 3 (IC)"
    yield "size4", _with_section(curve, m, pk, 4, data[Z.sections(data)[4][0]:sum(Z.sections(data)[4])] + b"\0"), "section 4"
    yield "size9", _with_section(curve, m, pk, 9, np.ascontiguousarray(pk.h_query).tobytes()[:-2 * nq]), "section 9 (H)"


@pytest.mark.parametrize("curve", CURVES)
def test_host_refusals_keep_the_resident_state(curve):
    m, z, pk, data = _fixture(curve)
    gz = engine(curve, "zk")
    _, info = gz.load_zkey(data)
    for what, bad, msg in host_cases(curve, m, pk, data):
        with pytest.raises(DeserializeError) as ei:
            gz.load_zkey(bad)
        assert msg in str(ei.value), (what, str(ei.value))
        _resident_ok(gz, info, z)   # the previous circuit and key are still resident
    rc = gz._lib.g16_zkey_load(gz._ctx, None, 0, 8, 0, 1, None, None)   # unknown flag
    assert rc == _lib.ERR_BAD_ARGUMENT
    _resident_ok(gz, info, z)


def device_cases(curve, m, pk, data):
    cp = engine(curve, "zk").curve
    h = Z.header(data)
    nr, nq = h["n8r"], h["n8q"]
    ncoef = struct.unpack_from("<I", data, Z.sections(data)[4][0])[0]
    chunk = 1 << 17
    for k in sorted({0, ncoef - 1} | ({chunk - 1, chunk} if ncoef > chunk else set())):
        o = Z.coef_offset(data, k)
        yield f"matrix@{k}", _patch(data, o, struct.pack("<I", 2)), f"coefficient {k}: matrix 2"
        yield f"constraint@{k}", _patch(data, o + 4, struct.pack("<I", h["domain_size"])), f"coefficient {k}: constraint"
        yield f"signal@{k}", _patch(data, o + 8, struct.pack("<I", h["nvars"] + 5)), \
            f"coefficient {k}: signal {h['nvars'] + 5} >= nVars {h['nvars']}"
        yield f"value@{k}", _patch(data, o + 12, cp.r.to_bytes(nr, "little")), f"coefficient {k}: value"
    # the public-input rows: the last record is row nc + nPublic of A
    o = Z.coef_offset(data, ncoef - 1)
    npub = h["npub"]
    yield "pubrow-col", _patch(data, o + 8, struct.pack("<I", (npub + 1) % h["nvars"])), \
        f"public-input row {npub} of A is not {{({npub}, 1)}}"
    yield "pubrow-B", _patch(data, o, struct.pack("<I", 1)), f"public-input row {npub} of"
    # points: non-canonical, off the curve, in every point section at the first and last index
    secs = Z.sections(data)
    G1, G2 = 2 * nq, 4 * nq
    single = {"alpha1": h["points"], "beta1": h["points"] + G1, "beta2": h["points"] + 2 * G1,
              "gamma2": h["points"] + 2 * G1 + G2, "delta1": h["points"] + 2 * G1 + 2 * G2, "delta2": h["points"] + 3 * G1 + 2 * G2}
    items = [(k, v, 1, k.endswith("2")) for k, v in single.items()]
    nv, nw = h["nvars"], h["nvars"] - npub - 1
    items += [("IC", secs[3][0], npub + 1, False), ("A", secs[5][0], nv, False), ("B1", secs[6][0], nv, False),
              ("B2", secs[7][0], nv, True), ("C", secs[8][0], nw, False), ("H", secs[9][0], h["domain_size"], False)]
    for name, off, cnt, g2 in items:
        ps = G2 if g2 else G1
        for i in sorted({0, cnt - 1}):
            at = off + i * ps
            label = name if name in single else f"{name}[{i}]"
            yield f"{label}-noncanon", _patch(data, at, cp.q.to_bytes(nq, "little")), f"{label} (byte {at}): non-canonical"
            yield f"{label}-offcurve", _patch(data, at, (1).to_bytes(nq, "little")), f"{label} (byte {at}): point is not on the curve"


@pytest.mark.parametrize("curve", CURVES)
def test_device_refusals_leave_nothing_resident(curve):
    m, z, pk, data = _fixture(curve)
    gz = engine(curve, "zk")
    for what, bad, msg in device_cases(curve, m, pk, data):
        _, info = gz.load_zkey(data)
        with pytest.raises(DeserializeError) as ei:
            gz.load_zkey(bad)
        assert msg in str(ei.value), (what, str(ei.value))
        rl = np.ascontiguousarray(gz.codec.fr.enc1(5))
        out = np.zeros(4 * gz.nq + gz.ng2, dtype=np.uint64)
        rc = gz._lib.g16_prove(gz._ctx, rl.ctypes.data, rl.ctypes.data, z.ctypes.data, 0, out.ctypes.data)
        assert rc == _lib.ERR_BAD_ARGUMENT, what        # neither circuit nor key
    _, info = gz.load_zkey(data)                        # and the next load succeeds
    _resident_ok(gz, info, z)


@pytest.mark.parametrize("curve", CURVES)
def test_subgroup_only_with_validate(curve):
    if curve == "bn254":   # G1 has cofactor 1: the point to refuse is in B2
        name, sid, g2 = "B2", 7, True
    else:
        name, sid, g2 = "A", 5, False
    m, z, pk, data = _fixture(curve)
    gz = engine(curve, "zk")
    c = P.CURVES[curve]
    cx = P.ctx(c)
    cd = gz.codec
    G, F = (cx.G2, cx.Fq2) if g2 else (cx.G1, cx.Fq)
    # a curve point outside the prime-order subgroup: the first x whose curve equation has a root, cofactor not cleared
    x = 1
    while True:
        xx = (x, 1) if g2 else x
        y = F.sqrt(F.add(F.mul(F.mul(xx, xx), xx), G.b))
        if y is not None and G.mul((xx, y), c.r) is not None:
            pt = (xx, y)
            break
        x += 1
    enc = (cd.enc_g2([pt]) if g2 else cd.enc_g1([pt]))[0]
    secs = Z.sections(data)
    at = secs[sid][0] + 3 * len(enc.tobytes())
    bad = _patch(data, at, enc.tobytes())
    _, info = gz.load_zkey(bad, validate=False)     # accepted without the check
    with pytest.raises(DeserializeError, match=rf"{name}\[3\] \(byte {at}\): point is not in the prime-order subgroup"):
        gz.load_zkey(bad, validate=True)


@pytest.mark.parametrize("curve", ["bls12_377", "bw6_761"])
def test_other_curves_refuse(curve):
    g = Groth16(curve, 0)
    try:
        with pytest.raises(ValueError, match="BN254 and BLS12-381 only"):
            g.load_zkey(b"zkey")
    finally:
        g.close()


@pytest.mark.parametrize("curve", CURVES)
def test_calls_that_need_c_refuse(curve):
    m, z, pk, data = _fixture(curve)
    gz = engine(curve, "zk")
    _, info = gz.load_zkey(data)
    cd = gz.codec
    rl = np.ascontiguousarray(cd.fr.enc1(5))
    out = np.zeros(4 * gz.nq + gz.ng2, dtype=np.uint64)
    h = np.zeros(((1 << info.log_n), gz.nr), dtype=np.uint64)
    rep = (_lib.WitnessReport * 1)()
    L = gz._lib
    calls = {
        "check_witness": lambda: L.g16_check_witness(gz._ctx, 1, z.ctypes.data, 0, rep),
        "prove+check": lambda: L.g16_prove(gz._ctx, rl.ctypes.data, rl.ctypes.data, z.ctypes.data, _lib.CHECK_WITNESS, out.ctypes.data),
        "submit+check": lambda: L.g16_prove_submit(gz._ctx, 0, rl.ctypes.data, rl.ctypes.data, z.ctypes.data, _lib.CHECK_WITNESS),
        "batch+check": lambda: L.g16_prove_batch(gz._ctx, 1, rl.ctypes.data, rl.ctypes.data, z.ctypes.data, 0, _lib.CHECK_WITNESS,
                                                 out.ctypes.data),
        "partial+check": lambda: L.g16_prove_partial(gz._ctx, rl.ctypes.data, z.ctypes.data, _lib.CHECK_WITNESS, out.ctypes.data),
        "witness_map+check": lambda: L.g16_witness_map(gz._ctx, z.ctypes.data, _lib.CHECK_WITNESS, h.ctypes.data),
        "setup": lambda: L.g16_setup(gz._ctx, *([rl.ctypes.data] * 7)),
        "setup_from_srs": lambda: L.g16_setup_from_srs(gz._ctx, _lib.SrsDesc(), 0),
        "pk_verify_pairs": lambda: L.g16_pk_verify_pairs(gz._ctx, _lib.SrsDesc(), _lib.PkCheckDesc(), rl.ctypes.data, 0,
                                                         out.ctypes.data, out.ctypes.data),
    }
    for name, call in calls.items():
        assert call() == _lib.ERR_BAD_ARGUMENT, name
        assert "holds no C matrix" in _lib.last_error(), name
        _resident_ok(gz, info, z)
    # a later g16_circuit_load_qap clears the state
    gz.qap = "circom"
    gz.load_matrices(m)
    rep = gz.check_witness(z)
    assert rep[0].num_unsatisfied == 0
