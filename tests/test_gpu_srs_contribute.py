"""GPU tier of g16_srs_contribute (phase-1 contributions to a powers-of-tau transcript).  T(tau, alpha, beta) is
g16_srs_from_secrets, which reaches the same transcript by another route (fixed-base tables): contributing (tau2, alpha2,
beta2) to T(tau1, alpha1, beta1) must give T(tau1 tau2, alpha1 alpha2, beta1 beta2) in every limb.  The CPU oracle
(liboracle's batch multiplication), tests/bw6_ref.py and pyref's pairing check the result independently of the device."""
import ctypes as C

import numpy as np
import pytest

import pyref as P
from groth16_b200 import Groth16, Srs, _lib
from groth16_b200.params import GENERATORS
from groth16_b200.serialize import DeserializeError
from groth16_b200.workload import synthetic_r1cs
from util import matrices_from_r1cs, proof_from_abi

pytestmark = pytest.mark.gpu

CURVES4 = ["bls12_381", "bn254", "bls12_377", "bw6_761"]
TAU, ALPHA, BETA = 0x1234567890ABCDEF1234567, 0x2222222222222222222223, 0x3333333333333333333335
TAU2, ALPHA2, BETA2 = 0x7777777777777777777779ABC, 0x6666666666666666666661, 0x5555555555555555555557
TAU3, ALPHA3, BETA3 = 0x99999999999999999999999B, 0x8888888888888888888885, 0xAAAAAAAAAAAAAAAAAAAAAD
D1 = 0x4444444444444444444447
VECS = ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1")
MEMBERS = VECS + ("beta_g2",)
KEY_MEMBERS = ("a_query", "b_g1_query", "b_g2_query", "h_query", "l_query", "beta_g1", "delta_g1")
VK_MEMBERS = ("alpha_g1", "beta_g2", "gamma_g2", "delta_g2", "gamma_abc_g1")

_ENG = {}


def engine(curve, qap="libsnark") -> Groth16:
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


def gens(curve):
    G = GENERATORS[curve]
    return G["g1"], G["g2"]


def T(g, n1, n2, tau, alpha, beta) -> Srs:
    return g.srs_from_secrets(n1, n2, tau, alpha, beta, *gens(g.curve.name))


def prod(g, *xs):
    r = g.curve.r
    out = 1
    for x in xs:
        out = out * x % r
    return out


def assert_same_srs(a: Srs, b: Srs):
    for k in MEMBERS:
        x, y = np.asarray(getattr(a, k)), np.asarray(getattr(b, k))
        assert x.shape == y.shape and np.array_equal(x, y), k


def copy_srs(s: Srs) -> Srs:
    return Srs(**{k: np.array(getattr(s, k), copy=True) for k in MEMBERS})


# ---- 1-3: composition, identity transcript, two contributions ---------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES4)
def test_composition(curve):
    g = engine(curve)
    for log_n in range(4, 13):
        n = 1 << log_n
        got = g.contribute_srs(T(g, 2 * n - 1, n, TAU, ALPHA, BETA), TAU2, ALPHA2, BETA2)
        assert_same_srs(got, T(g, 2 * n - 1, n, prod(g, TAU, TAU2), prod(g, ALPHA, ALPHA2), prod(g, BETA, BETA2)))
    for n1, n2 in ((1, 1), (2, 2), (3, 3), (1000, 1000), (1, 3), (1000, 2)):
        got = g.contribute_srs(T(g, n1, n2, TAU, ALPHA, BETA), TAU2, ALPHA2, BETA2)
        assert_same_srs(got, T(g, n1, n2, prod(g, TAU, TAU2), prod(g, ALPHA, ALPHA2), prod(g, BETA, BETA2)))
    # one member of length 0 (None or an empty array): skipped, the others unchanged in meaning
    want = T(g, 31, 16, prod(g, TAU, TAU2), prod(g, ALPHA, ALPHA2), prod(g, BETA, BETA2))
    for k in VECS:
        s = T(g, 31, 16, TAU, ALPHA, BETA)
        setattr(s, k, None if k == "tau_g2" else getattr(s, k)[:0])
        got = g.contribute_srs(s, TAU2, ALPHA2, BETA2)
        assert getattr(got, k).shape[0] == 0
        for j in MEMBERS:
            if j != k:
                assert np.array_equal(getattr(got, j), getattr(want, j)), (k, j)


@pytest.mark.parametrize("curve", CURVES4)
def test_identity_transcript_and_two_contributions(curve):
    g = engine(curve)
    n = 1 << 7
    assert_same_srs(g.contribute_srs(T(g, 2 * n - 1, n, 1, 1, 1), TAU, ALPHA, BETA), T(g, 2 * n - 1, n, TAU, ALPHA, BETA))
    two = g.contribute_srs(g.contribute_srs(T(g, 2 * n - 1, n, TAU, ALPHA, BETA), TAU2, ALPHA2, BETA2), TAU3, ALPHA3, BETA3)
    one = g.contribute_srs(T(g, 2 * n - 1, n, TAU, ALPHA, BETA), prod(g, TAU2, TAU3), prod(g, ALPHA2, ALPHA3),
                           prod(g, BETA2, BETA3))
    assert_same_srs(two, one)
    assert_same_srs(two, T(g, 2 * n - 1, n, prod(g, TAU, TAU2, TAU3), prod(g, ALPHA, ALPHA2, ALPHA3),
                           prod(g, BETA, BETA2, BETA3)))


# ---- 4: chunking and aliasing, and the call's timings -----------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES4)
def test_chunking_and_in_place(curve):
    g = engine(curve)
    n = 300
    src = T(g, 2 * n - 1, n, TAU, ALPHA, BETA)
    want = g.contribute_srs(src, TAU2, ALPHA2, BETA2)
    # chunks of one point (one launch per point) on a prefix: the contribution of a prefix is the prefix of the contribution
    head = lambda s, k: Srs(*(getattr(s, m)[:k] for m in VECS), s.beta_g2)
    for chunk in (1, 7, 128, 0):
        for in_place in (False, True):
            k = 24 if chunk == 1 else 2 * n
            s = copy_srs(head(src, k))
            got = g.contribute_srs(s, TAU2, ALPHA2, BETA2, chunk_points=chunk, in_place=in_place)
            assert (got is s) == in_place
            assert_same_srs(got, head(want, k))
            if not in_place:
                assert_same_srs(s, head(src, k))   # the input is only read
    assert_same_srs(g.contribute_srs(src, TAU2, ALPHA2, BETA2, validate=True, chunk_points=7), want)


@pytest.mark.parametrize("curve", ["bn254", "bw6_761"])
def test_timings_describe_the_call(curve):
    g = engine(curve)
    lens = dict(tau_g1=1001, tau_g2=300, alpha_tau_g1=299, beta_tau_g1=7)
    s = T(g, 1001, 300, TAU, ALPHA, BETA)
    s.alpha_tau_g1, s.beta_tau_g1 = s.alpha_tau_g1[:299], s.beta_tau_g1[:7]
    chunk = 64
    g.contribute_srs(s, TAU2, ALPHA2, BETA2, chunk_points=chunk)
    tm = _lib.Timings()
    assert g._lib.g16_get_timings(g._ctx, C.byref(tm)) == 0
    esz = dict(tau_g1=16 * g.nq, tau_g2=8 * g.ng2, alpha_tau_g1=16 * g.nq, beta_tau_g1=16 * g.nq)
    chunks = {k: -(-v // chunk) for k, v in lens.items()}
    vec_bytes = sum(lens[k] * esz[k] for k in VECS)
    assert tm.launches == 2 * sum(chunks.values()) + 1   # check + transform per chunk, and beta_g2's check
    assert tm.h2d_bytes == 2 * vec_bytes + 8 * g.ng2 + 32 * 8 * g.nr
    assert tm.d2h_bytes == vec_bytes + 8 * (sum(chunks.values()) + 1)
    assert tm.total_ms > 0 and tm.h2d_ms > 0 and all(tm.msm_ms[m] > 0 for m in range(4))
    assert tm.total_ms >= tm.h2d_ms + sum(tm.msm_ms[m] for m in range(4)) * 0.99
    assert tm.msm_ms[4] == 0 and tm.witness_map_ms == 0 and tm.host_finish_ms == 0
    assert all(tm.msm_pairs[m] == 0 and tm.msm_entries[m] == 0 for m in range(5))


# ---- 5, 6: independent references ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", ["bls12_381", "bn254", "bls12_377"])
def test_against_cpu_oracle(curve):
    import orc
    g = engine(curve)
    cd, r = g.codec, g.curve.r
    n = 1 << 16
    got = g.contribute_srs(T(g, 2 * n - 1, n, TAU, ALPHA, BETA), TAU2, ALPHA2, BETA2)
    t, a, b = prod(g, TAU, TAU2), prod(g, ALPHA, ALPHA2), prod(g, BETA, BETA2)
    pw = [1] * (2 * n - 1)
    for i in range(1, 2 * n - 1):
        pw[i] = pw[i - 1] * t % r
    g1, g2 = (np.ascontiguousarray(x) for x in (cd.enc_g1([gens(curve)[0]])[0], cd.enc_g2([gens(curve)[1]])[0]))
    cid, th = P.CURVES[curve].cid, 8
    assert np.array_equal(got.tau_g1, orc.batch_mul_g1(cid, cd.nq, g1, cd.fr.enc(pw), th))
    assert np.array_equal(got.tau_g2, orc.batch_mul_g2(cid, cd.nq, g2, cd.fr.enc(pw[:n]), th))
    assert np.array_equal(got.alpha_tau_g1, orc.batch_mul_g1(cid, cd.nq, g1, cd.fr.enc([a * x % r for x in pw[:n]]), th))
    assert np.array_equal(got.beta_tau_g1, orc.batch_mul_g1(cid, cd.nq, g1, cd.fr.enc([b * x % r for x in pw[:n]]), th))
    assert np.array_equal(got.beta_g2, orc.batch_mul_g2(cid, cd.nq, g2, cd.fr.enc([b]), 1)[0])


def test_bw6_against_reference():
    import bw6_ref as B
    g = engine("bw6_761")
    cd, r = g.codec, g.curve.r
    n = 1 << 12
    got = g.contribute_srs(T(g, 2 * n - 1, n, TAU, ALPHA, BETA), TAU2, ALPHA2, BETA2, chunk_points=1000)
    t, a, b = prod(g, TAU, TAU2), prod(g, ALPHA, ALPHA2), prod(g, BETA, BETA2)
    g1, g2 = gens("bw6_761")
    for i in (0, 1, 2, 999, 1000, n - 1, 2 * n - 2):
        assert cd.dec_g1(got.tau_g1[i])[0] == B.mul(pow(t, i, r), g1), i
    for i in (0, 1, 1000, n - 1):
        assert cd.dec_g2(got.tau_g2[i])[0] == B.mul(pow(t, i, r), g2), i
        assert cd.dec_g1(got.alpha_tau_g1[i])[0] == B.mul(a * pow(t, i, r) % r, g1), i
        assert cd.dec_g1(got.beta_tau_g1[i])[0] == B.mul(b * pow(t, i, r) % r, g1), i
    assert cd.dec_g2(got.beta_g2)[0] == B.mul(b, g2)


@pytest.mark.parametrize("curve", ["bn254", "bls12_381"])
def test_phase1_pairing_checks(curve):
    """the pairing equations a phase-1 verifier checks, on a contributed transcript"""
    g = engine(curve)
    cx = P.ctx(P.CURVES[curve])
    cd = g.codec
    got = g.contribute_srs(T(g, 7, 4, TAU, ALPHA, BETA), TAU2, ALPHA2, BETA2)
    g1, g2 = gens(curve)
    t1 = [cd.dec_g1(x)[0] for x in got.tau_g1]
    t2 = [cd.dec_g2(x)[0] for x in got.tau_g2]
    bt1 = [cd.dec_g1(x)[0] for x in got.beta_tau_g1]
    bg2 = cd.dec_g2(got.beta_g2)[0]
    eq = lambda p, q, p2, q2: cx.pairing_product_is_one([(p, q), (cx.G1.neg(p2), q2)])
    for i in (1, 2):
        assert eq(t1[i + 1], g2, t1[i], t2[1]), i
        assert eq(t1[i], g2, g1, t2[i]), i
        assert eq(bt1[i], g2, t1[i], bg2), i
    assert not eq(t1[3], g2, t1[1], t2[1])   # the check has teeth


# ---- 7, 8: the whole ceremony, and a production-size transcript ---------------------------------------------------------
def _key_and_bytes(g):
    return g.export_proving_key(), g.export_proving_key_bytes(compress=False)


def _assert_same_key(a, b):
    (k1, b1), (k2, b2) = a, b
    for name in KEY_MEMBERS:
        assert np.array_equal(getattr(k1, name), getattr(k2, name)), name
    for name in VK_MEMBERS:
        assert np.array_equal(getattr(k1.vk, name), getattr(k2.vk, name)), "vk." + name
    assert b1 == b2


def _n_of(m):
    need = m.num_constraints + m.num_instance_variables
    return 1 << max(need - 1, 0).bit_length()


def _ceremony(g, m, n):
    srs = g.contribute_srs(T(g, 2 * n - 1, n, TAU, ALPHA, BETA), TAU2, ALPHA2, BETA2, chunk_points=100)
    g.generate_parameters_from_srs(m, srs, export=False)
    g.contribute_delta(D1, export=False)
    got = _key_and_bytes(g)
    g.generate_parameters_with_qap(m, prod(g, ALPHA, ALPHA2), prod(g, BETA, BETA2), 1, D1, prod(g, TAU, TAU2),
                                   *gens(g.curve.name), export=False)
    _assert_same_key(got, _key_and_bytes(g))
    return srs


@pytest.mark.parametrize("qap", ["libsnark", "circom"])
@pytest.mark.parametrize("curve", CURVES4)
def test_whole_ceremony_key(curve, qap):
    g = engine(curve, qap)
    m, _, _ = synthetic_r1cs(curve, 6, seed=500)
    _ceremony(g, m, _n_of(m))


@pytest.mark.parametrize("qap", ["libsnark", "circom"])
@pytest.mark.parametrize("curve", ["bn254", "bls12_381"])
def test_whole_ceremony_proof_verifies(curve, qap):
    c = P.CURVES[curve]
    rng = P.Rng(21)
    a, b = rng.fr(c.r), rng.fr(c.r)
    cs = P.silly_circuit(c, a, b)
    m = matrices_from_r1cs(cs)
    g = engine(curve, qap)
    cd = g.codec
    srs = _ceremony(g, m, _n_of(m))   # leaves the matching g16_setup key resident: derive the ceremony's key again
    g.generate_parameters_from_srs(None, srs, export=False)
    pk = g.contribute_delta(D1)
    z = np.ascontiguousarray(cd.fr.enc(cs.assignment))
    pf = g.create_proof_with_reduction_and_matrices(None, rng.fr(c.r), rng.fr(c.r), None, cs.num_instance,
                                                    cs.num_constraints, z)
    vk = P.VerifyingKey(cd.dec_g1(pk.vk.alpha_g1)[0], cd.dec_g2(pk.vk.beta_g2)[0], cd.dec_g2(pk.vk.gamma_g2)[0],
                        cd.dec_g2(pk.vk.delta_g2)[0], cd.dec_g1(pk.vk.gamma_abc_g1))
    pub = cd.fr.dec(z)[1:cs.num_instance]
    assert P.verify_proof(vk, c, proof_from_abi(curve, pf), pub)
    assert not P.verify_proof(vk, c, proof_from_abi(curve, pf), [(pub[0] + 1) % c.r] + pub[1:])


@pytest.mark.parametrize("curve", ["bls12_381", "bn254"])
def test_production_size(curve):
    g = engine(curve)
    n = 1 << 20
    got = g.contribute_srs(T(g, 2 * n - 1, n, TAU, ALPHA, BETA), TAU2, ALPHA2, BETA2, in_place=True)
    assert_same_srs(got, T(g, 2 * n - 1, n, prod(g, TAU, TAU2), prod(g, ALPHA, ALPHA2), prod(g, BETA, BETA2)))


# ---- 9: refusals --------------------------------------------------------------------------------------------------------
def _desc(cls, arrs, lens=None):
    d = cls()
    for k in VECS:
        v = arrs.get(k)
        setattr(d, k, None if v is None else v.ctypes.data_as(_lib.u64p))
        setattr(d, k + "_len", (lens or {}).get(k, 0 if v is None else v.shape[0]))
    v = arrs.get("beta_g2")
    d.beta_g2 = None if v is None else v.ctypes.data_as(_lib.u64p)
    return d


def _raw(g, ins, outs, secrets=(TAU2, ALPHA2, BETA2), flags=0, chunk=0, in_lens=None, out_lens=None, null=()):
    """g16_srs_contribute on explicit arrays: (status, g16_last_error())"""
    sc = [None if x is None else np.ascontiguousarray(g.codec.fr.enc1(x)) for x in secrets]
    d_in = None if "in" in null else C.byref(_desc(_lib.SrsDesc, ins, in_lens))
    d_out = None if "out" in null else C.byref(_desc(_lib.SrsOut, outs, out_lens))
    rc = g._lib.g16_srs_contribute(g._ctx, d_in, *[None if x is None else x.ctypes.data_as(C.c_void_p) for x in sc], flags,
                                   chunk, d_out)
    return rc, _lib.last_error()


def _arrays(s: Srs):
    return {k: np.ascontiguousarray(getattr(s, k)) for k in MEMBERS}


SENTINEL = np.uint64(0xABABABABABABABAB)


def _sentinel_like(ins):
    return {k: np.full_like(v, SENTINEL) for k, v in ins.items()}


@pytest.mark.parametrize("curve", ["bls12_381", "bw6_761"])
def test_argument_errors(curve):
    g = engine(curve)
    ins = _arrays(T(g, 15, 8, TAU, ALPHA, BETA))
    keep = {k: v.copy() for k, v in ins.items()}
    outs = _sentinel_like(ins)
    bad = _lib.ERR_BAD_ARGUMENT

    def refused(match, **kw):
        rc, msg = _raw(g, kw.pop("ins", ins), kw.pop("outs", outs), **kw)
        assert rc == bad and match in msg, (rc, msg)
        for k in MEMBERS:
            assert np.array_equal(ins[k], keep[k]), k
            assert (outs[k] == SENTINEL).all(), k

    assert _raw(g, ins, _sentinel_like(ins))[0] == 0   # the arguments below are the only thing wrong
    for which in ("in", "out"):
        refused("null argument", null=(which,))
    for i in range(3):
        sec = [TAU2, ALPHA2, BETA2]
        sec[i] = None
        refused("null argument", secrets=sec)
    for k in MEMBERS:
        ln = None if k == "beta_g2" else {k: ins[k].shape[0]}
        refused(f"null srs member {k}", ins={**ins, k: None}, in_lens=ln)
        refused(f"null srs member {k}", outs={**outs, k: None}, out_lens=ln)
    for flags in (1, 4, 3, 1 << 31):
        refused("takes 0 or G16_SER_VALIDATE", flags=flags)
    for i in range(3):
        for zero in (0, g.curve.r):
            sec = [TAU2, ALPHA2, BETA2]
            sec[i] = zero
            refused("UnexpectedIdentity", secrets=sec)
    for k in VECS:
        refused("lengths must be equal", out_lens={k: ins[k].shape[0] - 1})
        refused("at most 2^32 - 1", in_lens={k: 1 << 32}, out_lens={k: 1 << 32})
    # overlaps: an output shifted by one point from its own input, an output over another member's input, two outputs
    big = np.concatenate([ins["tau_g1"], ins["tau_g1"][:2]])
    refused("out tau_g1 overlaps in tau_g1", ins={**ins, "tau_g1": big[:-1]}, outs={**outs, "tau_g1": big[1:]})
    refused("out alpha_tau_g1 overlaps in tau_g1", outs={**outs, "alpha_tau_g1": ins["tau_g1"][3:3 + 8]})
    refused("out beta_g2 overlaps in tau_g2", outs={**outs, "beta_g2": ins["tau_g2"][5]})
    both = np.full((16, ins["tau_g1"].shape[1]), SENTINEL, dtype=np.uint64)
    refused("out alpha_tau_g1 overlaps out beta_tau_g1", outs={**outs, "alpha_tau_g1": both[:8], "beta_tau_g1": both[7:15]})
    # in place is fine, and so is an empty member pointing anywhere
    inp = {k: v.copy() for k, v in ins.items()}
    assert _raw(g, inp, inp)[0] == 0
    e = {**_sentinel_like(ins), "beta_tau_g1": ins["tau_g1"][4:4]}
    assert _raw(g, {**ins, "beta_tau_g1": ins["tau_g1"][2:2]}, e)[0] == 0


def _off_curve(arr, idx):
    a = arr[idx] if arr.ndim == 2 else arr
    a[-1] ^= np.uint64(1)   # y's top limb: off the curve, still below q


@pytest.mark.parametrize("curve", ["bls12_381", "bw6_761"])
def test_refused_point_in_a_late_chunk(curve):
    g = engine(curve)
    n = 1 << 17
    src = T(g, 2 * n - 1, n, TAU, ALPHA, BETA)
    k = 70001
    s = copy_srs(src)
    _off_curve(s.beta_tau_g1, k)
    _off_curve(s.beta_tau_g1, k + 5)     # a later bad point in the same chunk is not the one named
    _off_curve(s.beta_tau_g1, 120000)    # nor one in a later chunk
    ins = _arrays(s)
    outs = _sentinel_like(ins)
    rc, msg = _raw(g, ins, outs, chunk=1000)
    assert rc == _lib.ERR_INVALID_DATA and msg == f"beta_tau_g1[{k}]: point is not on the curve", msg
    assert all((outs[m] == SENTINEL).all() for m in MEMBERS)
    # the same through Python, in place: the transcript is intact
    before = copy_srs(s)
    with pytest.raises(DeserializeError, match=rf"^beta_tau_g1\[{k}\]: point is not on the curve$"):
        g.contribute_srs(s, TAU2, ALPHA2, BETA2, chunk_points=1000, in_place=True)
    assert_same_srs(s, before)
    # an earlier member is named first, whatever the index
    _off_curve(s.tau_g2, n - 1)
    with pytest.raises(DeserializeError, match=rf"^tau_g2\[{n - 1}\]: point is not on the curve$"):
        g.contribute_srs(s, TAU2, ALPHA2, BETA2, chunk_points=7)
    for m, idx in (("tau_g1", 2 * n - 2), ("beta_g2", 0)):
        s = copy_srs(src)
        _off_curve(getattr(s, m), idx)
        before = copy_srs(s)
        with pytest.raises(DeserializeError, match=rf"^{m}\[{idx}\]: point is not on the curve$"):
            g.contribute_srs(s, TAU2, ALPHA2, BETA2, in_place=True)
        assert_same_srs(s, before)


@pytest.mark.parametrize("curve", ["bls12_381", "bn254", "bls12_377"])
def test_torsion_point_needs_validate(curve):
    """a G2 point on the curve but outside the prime-order subgroup: refused with G16_SER_VALIDATE only"""
    g = engine(curve)
    c = P.CURVES[curve]
    Gp = P.ctx(c).G2
    F = Gp.F
    x = F.from_int(1)
    while True:
        y = F.sqrt(F.add(F.mul(F.mul(x, x), x), Gp.b))
        if y is not None:
            break
        x = F.add(x, F.from_int(1))
    Tp = (x, y)
    assert Gp.mul(Tp, c.r) is not None
    s = T(g, 15, 8, TAU, ALPHA, BETA)
    s.tau_g2[5] = g.codec.enc_g2([Tp])[0]
    with pytest.raises(DeserializeError, match=r"^tau_g2\[5\]: point is not in the prime-order subgroup$"):
        g.contribute_srs(s, TAU2, ALPHA2, BETA2, validate=True, chunk_points=3)
    got = g.contribute_srs(s, TAU2, ALPHA2, BETA2)
    assert g.codec.dec_g2(got.tau_g2[5])[0] == Gp.mul(Tp, pow(TAU2, 5, c.r))


# ---- 10: the resident circuit and key are untouched ------------------------------------------------------------------
@pytest.mark.parametrize("curve", ["bn254", "bw6_761"])
def test_residency_untouched(curve):
    g = engine(curve)
    m, z, _ = synthetic_r1cs(curve, 6, seed=510)
    g.generate_parameters_with_qap(m, ALPHA, BETA, 1, D1, TAU, *gens(curve), export=False)
    prove = lambda: g.create_proof_with_reduction_and_matrices(None, 5, 7, None, m.num_instance_variables,
                                                               m.num_constraints, z)
    before = prove()
    key_before = g.export_proving_key_bytes(compress=False)
    s = T(g, 1 << 12, 1 << 11, TAU, ALPHA, BETA)
    g.contribute_srs(s, TAU2, ALPHA2, BETA2, chunk_points=1000)
    g.contribute_srs(s, TAU2, ALPHA2, BETA2, in_place=True, validate=True)
    after = prove()
    assert all(np.array_equal(getattr(before, k), getattr(after, k)) for k in "abc")
    assert g.export_proving_key_bytes(compress=False) == key_before
    # a proof in flight refuses the call, and it stays in flight
    r_, s_ = (np.ascontiguousarray(g.codec.fr.enc1(v)) for v in (5, 7))
    g.prove_submit_raw(0, r_, s_, z.ctypes.data, 0)
    try:
        with pytest.raises(ValueError, match="in flight"):
            g.contribute_srs(s, TAU2, ALPHA2, BETA2)
    finally:
        out = np.zeros_like(np.concatenate([before.a, before.b, before.c]))
        g.prove_wait_raw(0, out)
    assert np.array_equal(out, np.concatenate([before.a, before.b, before.c]))
