"""GPU tier of ark-serialized proving keys (g16_pk_load_serialized / g16_pk_export_serialized; run on an H100 with
`pytest -m gpu`).  groth16_b200.serialize.ArkCodec, with its subgroup check on exactly when `validate` is, is the oracle:
  * keys made by g16_setup, encoded by ArkCodec, load in both encodings with and without validation, give the verifying key
    back and prove bit for bit as the same key in limbs; the export equals ArkCodec's bytes;
  * every committed ark fixture's pk.bin loads as it is and reproduces proof.bin;
  * 2^20 keys on each curve round-trip (export, validated load, same proof) and load sharded over 3 emulated ranks;
  * rejections name the first bad item in stream order, with serialize.py's reason: every malformation in every member at
    its first and last index, and in every query at a chunk boundary of a 2^20 key; no key is resident afterwards;
  * small-order and cofactor-torsion points fail the subgroup check and pass without it."""
import io
import os

import numpy as np
import pytest

import pyref as P
from groth16_b200 import Groth16, MalformedKey, Proof
from groth16_b200.params import GENERATORS
from groth16_b200.serialize import ArkCodec, DeserializeError
from groth16_b200.workload import synthetic_r1cs
from test_ser_host import _special_points, _torsion_points
from util import ALL_CURVES, matrices_from_r1cs, pk_from_abi, proof_from_abi, toxic

pytestmark = pytest.mark.gpu

SER_CHUNK = 1 << 17   # points per decode chunk (Engine::SER_CHUNK): index SER_CHUNK starts the second chunk of a member
MEMBERS = ["vk.alpha_g1", "vk.beta_g2", "vk.gamma_g2", "vk.delta_g2", "vk.gamma_abc_g1", "beta_g1", "delta_g1", "a_query",
           "b_g1_query", "b_g2_query", "h_query", "l_query"]
G2_MEMBERS = {"vk.beta_g2", "vk.gamma_g2", "vk.delta_g2", "b_g2_query"}
VECS = {"vk.gamma_abc_g1", "a_query", "b_g1_query", "b_g2_query", "h_query", "l_query"}
_ENG = {}
_KEYS = {}


@pytest.fixture(scope="module", autouse=True)
def _release_contexts():
    """the contexts of this module hold keys resident: free their device memory for the modules that run after it"""
    yield
    for g in _ENG.values():
        g.close()
    _ENG.clear()
    _KEYS.clear()


def engine(curve, qap="libsnark") -> Groth16:
    if (curve, qap) not in _ENG:
        _ENG[(curve, qap)] = Groth16(curve, 0, qap=qap)
    return _ENG[(curve, qap)]


def layout(k: ArkCodec, data: bytes, compress: bool):
    """member -> (byte offset of element 0, length, bytes per point), from the length prefixes"""
    out, pos = {}, 0
    for name in MEMBERS:
        ps = k.fq_bytes * (2 if name in G2_MEMBERS else 1) * (1 if compress else 2)
        n = 1
        if name in VECS:
            n = int.from_bytes(data[pos:pos + 8], "little")
            pos += 8
        out[name] = (pos, n, ps)
        pos += n * ps
    assert pos == len(data)
    return out


def ark_bytes(curve, pk_abi, compress):
    opk = pk_from_abi(curve, pk_abi)
    k = ArkCodec(curve)
    vk = opk.vk
    return k.proving_key((vk.alpha_g1, vk.beta_g2, vk.gamma_g2, vk.delta_g2, vk.gamma_abc_g1), opk.beta_g1, opk.delta_g1,
                         opk.a_query, opk.b_g1_query, opk.b_g2_query, opk.h_query, opk.l_query, compress=compress)


def prove(g, m, z, r, s):
    out = np.zeros(8 * g.nq, dtype=np.uint64)
    g.prove_raw(g.codec.fr.enc1(r), g.codec.fr.enc1(s), np.ascontiguousarray(z).ctypes.data, 0, out)
    return out


def small_key(curve, kind):
    """(engine, matrices, assignment, setup key limbs, oracle circuit or None) for one of the small circuits"""
    key = (curve, kind)
    if key not in _KEYS:
        c = P.CURVES[curve]
        cx = P.ctx(c)
        qap = "circom" if kind == "circom" else "libsnark"
        g = engine(curve, qap)
        cs = None
        if kind == "silly":
            rng = P.Rng(5)
            cs = P.silly_circuit(c, rng.fr(c.r), rng.fr(c.r))
            m = matrices_from_r1cs(cs)
            z = np.ascontiguousarray(g.codec.fr.enc(cs.assignment))
        else:
            m, z, _ = synthetic_r1cs(curve, {"2p6": 6, "2p10": 10, "circom": 6}[kind], seed=9)
        tw = toxic(c, 31)
        pk = g.generate_parameters_with_qap(m, *tw, cx.g1_gen(), cx.g2_gen())
        _KEYS[key] = (g, m, z, pk, cs, tw)
    g, m = _KEYS[key][0], _KEYS[key][1]
    if g._matrices is not m:   # another test made another circuit resident on this context
        g.load_matrices(m)
    return _KEYS[key]


# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["silly", "2p6", "2p10", "circom"])
@pytest.mark.parametrize("curve", ALL_CURVES)
def test_setup_key_round_trip(curve, kind):
    g, m, z, pk, cs, tw = small_key(curve, kind)
    c = P.CURVES[curve]
    r, s = 0x1234567 % c.r, 0x7654321 % c.r
    g.load_proving_key(pk)
    want = prove(g, m, z, r, s)                       # the key in limbs
    for compress in (True, False):
        data = ark_bytes(curve, pk, compress)
        g.generate_parameters_with_qap(m, *tw, P.ctx(c).g1_gen(), P.ctx(c).g2_gen(), export=False)
        assert g.export_proving_key_bytes(compress) == data, (curve, kind, compress)
        for validate in (True, False):
            vk = g.load_proving_key_bytes(data, compress=compress, validate=validate)
            for name in ("alpha_g1", "beta_g2", "gamma_g2", "delta_g2", "gamma_abc_g1"):
                assert np.array_equal(getattr(vk, name), getattr(pk.vk, name)), name
            assert np.array_equal(vk.beta_g1, pk.beta_g1) and np.array_equal(vk.delta_g1, pk.delta_g1)
            assert np.array_equal(prove(g, m, z, r, s), want), (curve, kind, compress, validate)
    if cs is not None:   # and the oracle
        opk = pk_from_abi(curve, pk)
        pf = proof_from_abi(curve, Proof(want[:2 * g.nq], want[2 * g.nq:6 * g.nq], want[6 * g.nq:]))
        ref = P.create_proof(opk, cs, r, s)
        assert (pf.a, pf.b, pf.c) == (ref.a, ref.b, ref.c)


def _fixture_dirs():
    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ark")
    return sorted(os.path.join(here, d) for d in os.listdir(here) if os.path.isfile(os.path.join(here, d, "meta.json")))


@pytest.mark.parametrize("d", _fixture_dirs(), ids=os.path.basename)
def test_fixture_pk_bin_loads_directly(d):
    from test_ark_fixture import load_fixture
    fx = load_fixture(d)
    meta = fx["meta"]
    g = engine(fx["curve"])
    g.load_matrices(fx["m"])
    pk_bin = open(os.path.join(d, "pk.bin"), "rb").read()
    g.load_proving_key_bytes(pk_bin, compress=(meta["pk"] == "compressed"), validate=True)
    cd = fx["cd"]
    z = np.ascontiguousarray(cd.fr.enc(fx["z"]))
    out = prove(g, fx["m"], z, fx["r"], fx["s"])
    a, b, c = cd.dec_g1(out[:2 * g.nq])[0], cd.dec_g2(out[2 * g.nq:6 * g.nq])[0], cd.dec_g1(out[6 * g.nq:])[0]
    assert fx["codec"].proof(a, b, c, compress=True) == fx["proof_bytes"]


@pytest.mark.parametrize("curve", ALL_CURVES)
def test_2p20_round_trip_and_sharded_load(curve):
    g = Groth16(curve, 0)   # its own context, closed at the end: a 2^20 key with its precomputed copies holds ~10 GB
    try:
        _round_trip_2p20(g, curve)
    finally:
        g.close()


def _round_trip_2p20(g, curve):
    G = GENERATORS[curve]
    m, z, _ = synthetic_r1cs(curve, 20, seed=3)
    c = P.CURVES[curve]
    zz = g.codec.fr.dec(z)
    assert all(v != 0 for v in zz[1:]), "every base must enter the MSMs"
    g.generate_parameters_with_qap(m, 11, 13, 17, 19, 23, G["g1"], G["g2"], export=False)
    r, s = 0xabcdef % c.r, 0xfedcba % c.r
    want = prove(g, m, z, r, s)
    blobs = {cp: g.export_proving_key_bytes(cp) for cp in (True, False)}
    k = ArkCodec(curve)
    for cp, data in blobs.items():
        lay = layout(k, data, cp)
        assert lay["a_query"][1] > SER_CHUNK and lay["h_query"][1] > 2 * SER_CHUNK   # several chunks per query
        g.load_proving_key_bytes(data, compress=cp, validate=True)
        assert np.array_equal(prove(g, m, z, r, s), want), (curve, cp)
    # each malformation in each vector member at a chunk boundary (index SER_CHUNK starts a member's second chunk), both
    # encodings: reported with the member, that index and serialize.py's reason for the point
    for cp, data in blobs.items():
        lay = layout(k, data, cp)
        buf = bytearray(data)
        for name in ("a_query", "b_g1_query", "b_g2_query", "h_query", "l_query"):
            off, n, ps = lay[name]
            at = off + SER_CHUNK * ps
            orig = bytes(buf[at:at + ps])
            for fn in _corruptions(k, cp, name in G2_MEMBERS):
                buf[at:at + ps] = fn(orig)
                with pytest.raises(DeserializeError) as want_e:
                    k.read_point(io.BytesIO(bytes(buf[at:at + ps])), name in G2_MEMBERS, cp)
                with pytest.raises(DeserializeError) as e:
                    g.load_proving_key_bytes(buf, compress=cp, validate=False)
                label = f"{name}[{SER_CHUNK}]"
                assert label in str(e.value) and str(want_e.value) in str(e.value), (label, str(e.value), str(want_e.value))
            buf[at:at + ps] = orig
    # world = 3, emulated sequentially: the partial sums assemble into the same proof
    data = blobs[True]
    parts = []
    rl = np.ascontiguousarray(g.codec.fr.enc1(r))
    for rank in range(3):
        g.load_proving_key_bytes(data, compress=True, validate=True, rank=rank, world=3)
        out = np.zeros(g.partial_limbs(), dtype=np.uint64)
        g.prove_partial_raw(rl, z.ctypes.data, 0, out)
        parts.append(out)
    pf = g.prove_assemble(r, s, np.stack(parts))
    assert np.array_equal(np.concatenate([pf.a, pf.b, pf.c]), want)
    # a corruption at a chunk boundary and at the last index; with both present the earlier one is reported
    lay = layout(k, data, True)
    bad = bytearray(data)
    off, n, ps = lay["a_query"]
    at = off + SER_CHUNK * ps
    bad[at:at + k.fq_bytes] = _noncanonical(k, c.q)
    with pytest.raises(DeserializeError, match=r"a_query\[%d\].*non-canonical" % SER_CHUNK):
        g.load_proving_key_bytes(bytes(bad), compress=True, validate=True)
    off2, n2, ps2 = lay["l_query"]
    at2 = off2 + (n2 - 1) * ps2
    bad2 = bytearray(data)
    bad2[at2:at2 + k.fq_bytes] = _noncanonical(k, c.q)
    with pytest.raises(DeserializeError, match=r"l_query\[%d\]" % (n2 - 1)):
        g.load_proving_key_bytes(bytes(bad2), compress=True, validate=False)
    bad[at2:at2 + k.fq_bytes] = _noncanonical(k, c.q)
    with pytest.raises(DeserializeError, match=r"a_query\[%d\]" % SER_CHUNK):
        g.load_proving_key_bytes(bytes(bad), compress=True, validate=True)
    g.load_proving_key_bytes(data, compress=True, validate=False)
    assert np.array_equal(prove(g, m, z, r, s), want)


def _noncanonical(k, q):
    """the first field element of a compressed point set to q, flag bits kept as a valid compressed encoding would have"""
    if k.zcash:
        b = bytearray(q.to_bytes(k.fq_bytes, "big"))
        b[0] |= 0x80
        return bytes(b)
    return q.to_bytes(k.fq_bytes, "little")


def _corruptions(k, compress, g2):
    """functions (bytes of one point) -> bad bytes: a coordinate >= q, a flag error, and (uncompressed) a y off the curve"""
    q, nb = k.q, k.fq_bytes
    if k.zcash:
        qb = q.to_bytes(nb, "big")
        out = [lambda b: bytes([qb[0] | (b[0] & 0xE0)]) + qb[1:] + b[nb:], lambda b: bytes([b[0] ^ 0x80]) + b[1:]]
    else:
        out = [lambda b: q.to_bytes(nb, "little") + b[nb:], lambda b: b[:-1] + bytes([b[-1] | 0xC0])]
    if not compress:
        out.append(lambda b: b[:-1] + bytes([b[-1] ^ 1]) if k.zcash else b[:len(b) // 2] + bytes([b[len(b) // 2] ^ 1]) + b[len(b) // 2 + 1:])
    return out


@pytest.mark.parametrize("compress", [True, False])
@pytest.mark.parametrize("curve", ALL_CURVES)
def test_rejections_name_the_first_bad_item(curve, compress):
    g, m, z, pk, cs, tw = small_key(curve, "2p6")
    c = P.CURVES[curve]
    k = ArkCodec(curve)
    data = ark_bytes(curve, pk, compress)
    lay = layout(k, data, compress)
    r, s = 3, 5
    g.load_proving_key_bytes(data, compress=compress)
    want = prove(g, m, z, r, s)
    for name in MEMBERS:
        off, n, ps = lay[name]
        for idx in sorted({0, n - 1}):
            for fn in _corruptions(k, compress, name in G2_MEMBERS):
                bad = bytearray(data)
                at = off + idx * ps
                bad[at:at + ps] = fn(bytes(data[at:at + ps]))
                with pytest.raises(DeserializeError) as want_e:      # serialize.py's verdict and reason
                    k.read_proving_key(bytes(bad), compress=compress)
                label = f"{name}[{idx}]"
                with pytest.raises(DeserializeError) as e:
                    g.load_proving_key_bytes(bytes(bad), compress=compress, validate=False)
                assert label in str(e.value) and str(want_e.value) in str(e.value), (label, str(e.value), str(want_e.value))
    # no key is resident after a rejection; a good load proves again
    with pytest.raises(ValueError):
        prove(g, m, z, r, s)
    g.load_proving_key_bytes(data, compress=compress)
    assert np.array_equal(prove(g, m, z, r, s), want)
    # structure: truncated, trailing bytes, absurd length prefix, gamma_abc_g1 of the wrong length
    for bad, reason in ((data[:-1], "truncated input"), (data + b"\0", "trailing bytes"),
                        (data[:lay["a_query"][0] - 8] + (1 << 40).to_bytes(8, "little") + data[lay["a_query"][0]:], "exceeds the limit")):
        with pytest.raises(DeserializeError, match=reason):
            g.load_proving_key_bytes(bad, compress=compress)
    off, n, ps = lay["vk.gamma_abc_g1"]
    short = data[:off - 8] + (n - 1).to_bytes(8, "little") + data[off:off + (n - 1) * ps] + data[off + n * ps:]
    with pytest.raises(MalformedKey):
        g.load_proving_key_bytes(short, compress=compress)
    with pytest.raises(ValueError):
        prove(g, m, z, r, s)


@pytest.mark.parametrize("curve", ALL_CURVES)
def test_subgroup_check_small_order_and_torsion(curve):
    g, m, z, pk, cs, tw = small_key(curve, "2p6")
    for compress in (True, False):
        k = ArkCodec(curve)
        kv = ArkCodec(curve, check_subgroup=True)
        data = ark_bytes(curve, pk, compress)
        lay = layout(k, data, compress)
        for g2 in (False, True):
            member = "b_g2_query" if g2 else "a_query"
            off, n, ps = lay[member]
            at = off + 1 * ps
            pts = _torsion_points(curve, g2) + [p for p in _special_points(curve, g2)]
            if curve == "bn254" and not g2:
                assert not _torsion_points(curve, g2)
                x = 1
                while True:
                    try:
                        pts = [(x, k._solve_y(x, False))]
                        break
                    except DeserializeError:
                        x += 1
            for pt in pts:
                bad = data[:at] + k.point(pt, g2, compress) + data[at + ps:]
                in_sub = kv._in_subgroup(pt, g2)
                if in_sub:
                    g.load_proving_key_bytes(bad, compress=compress, validate=True)
                else:
                    with pytest.raises(DeserializeError, match=r"%s\[1\].*prime-order subgroup" % member):
                        g.load_proving_key_bytes(bad, compress=compress, validate=True)
                g.load_proving_key_bytes(bad, compress=compress, validate=False)
            if curve == "bn254" and not g2:
                assert all(kv._in_subgroup(p, False) for p in pts)
