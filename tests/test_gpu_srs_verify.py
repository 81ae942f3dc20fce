"""GPU tier of g16_srs_verify_pairs (the transcript check).  T(tau, alpha, beta) comes from g16_srs_from_secrets; every one
of the twenty output points is compared limb for limb with its closed-form scalar times the generator, formed by the CPU
oracle (liboracle's batch multiplication) or tests/bw6_ref.py, never by the device.  Which equations hold is decided in
the exponent (srs_verify_ref) on all four curves and with pyref's pairing where it has one."""
import ctypes as C

import numpy as np
import pytest

import pyref as P
from groth16_b200 import Groth16, Srs, _lib
from groth16_b200.params import GENERATORS
from groth16_b200.serialize import DeserializeError
from groth16_b200.workload import synthetic_r1cs
from srs_verify_ref import MEMBERS, VECS, closed_exponents, expected_failures, failing, pair_exponents, \
    transcript_exponents

pytestmark = pytest.mark.gpu

CURVES4 = ["bls12_381", "bn254", "bls12_377", "bw6_761"]
PAIRING = ["bn254", "bls12_381", "bls12_377"]
TAU, ALPHA, BETA = 0x1234567890ABCDEF1234567, 0x2222222222222222222223, 0x3333333333333333333335
TAU2, ALPHA2, BETA2 = 0x7777777777777777777779ABC, 0x6666666666666666666661, 0x5555555555555555555557
RHO, RHO2 = 0x5EED5EED5EED5EED5EED5EED5EED5EED1, 0xC0FFEE0C0FFEE0C0FFEE0C0FFEE01
D1 = 0x4444444444444444444447

_ENG = {}


def engine(curve) -> Groth16:
    for key in [k for k in _ENG if k != curve]:
        _ENG.pop(key).close()
    if curve not in _ENG:
        _ENG[curve] = Groth16(curve, 0)
    return _ENG[curve]


@pytest.fixture(scope="module", autouse=True)
def _engines():
    yield
    for g in _ENG.values():
        g.close()
    _ENG.clear()


def gens(curve):
    G = GENERATORS[curve]
    return G["g1"], G["g2"]


def T(g, lens, tau=TAU, alpha=ALPHA, beta=BETA) -> Srs:
    """T(tau, alpha, beta) with lens = (tau_g1, tau_g2, alpha_tau_g1, beta_tau_g1) points"""
    n1, n2, na, nb = lens
    s = g.srs_from_secrets(n1, max(n2, na, nb), tau, alpha, beta, *gens(g.curve.name))
    return Srs(s.tau_g1, np.ascontiguousarray(s.tau_g2[:n2]), np.ascontiguousarray(s.alpha_tau_g1[:na]),
               np.ascontiguousarray(s.beta_tau_g1[:nb]), s.beta_g2)


def copy_srs(s: Srs) -> Srs:
    return Srs(**{k: np.array(getattr(s, k), copy=True) for k in MEMBERS})


def closed(g, p, q):
    """[p_j]g1 and [q_j]g2 as limbs, by the CPU oracle or bw6_ref"""
    curve, cd = g.curve.name, g.codec
    g1, g2 = gens(curve)
    if curve == "bw6_761":
        import bw6_ref as B
        return cd.enc_g1([B.mul(k, g1) for k in p]), cd.enc_g2([B.mul(k, g2) for k in q])
    import orc
    cid = P.CURVES[curve].cid
    G1, G2 = (np.ascontiguousarray(x) for x in (cd.enc_g1([g1])[0], cd.enc_g2([g2])[0]))
    return orc.batch_mul_g1(cid, cd.nq, G1, cd.fr.enc(p), 4), orc.batch_mul_g2(cid, cd.nq, G2, cd.fr.enc(q), 4)


def assert_pairs(got, want, what=""):
    assert np.array_equal(got.g1, want[0]), ("g1", what)
    assert np.array_equal(got.g2, want[1]), ("g2", what)


def pairing_failures(g, pairs) -> set:
    cx = P.ctx(P.CURVES[g.curve.name])
    cd = g.codec
    ps, qs = cd.dec_g1(pairs.g1), cd.dec_g2(pairs.g2)
    return {k for k in range(5)
            if not cx.pairing_product_is_one([(ps[2 * k], qs[2 * k]), (cx.G1.neg(ps[2 * k + 1]), qs[2 * k + 1])])}


def point_of(g, m, k):
    """[k]g1 (G1 members) or [k]g2 (G2 members) as limbs, by g16_srs_from_secrets (tau_g1[1] / tau_g2[1] of tau = k)"""
    s = g.srs_from_secrets(2, 2, k, 1, 1, *gens(g.curve.name))
    return (s.tau_g2 if m in ("tau_g2", "beta_g2") else s.tau_g1)[1]


# ---- 1: closed form ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES4)
def test_closed_form(curve):
    g = engine(curve)
    r = g.curve.r
    sizes = [(2 * (1 << k) - 1, 1 << k, 1 << k, 1 << k) for k in range(4, 13, 2)] + [(2, 2, 1, 1), (1000, 3, 999, 7)]
    for lens in sizes:
        got = g.srs_verification_pairs(T(g, lens), RHO, validate=(lens[0] < 600))
        assert_pairs(got, closed(g, *closed_exponents(r, lens, TAU, ALPHA, BETA, RHO)), lens)


# ---- 2: pairing acceptance --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", PAIRING)
def test_honest_transcripts_pass_the_pairing(curve):
    g = engine(curve)
    honest = T(g, (33, 17, 17, 17))
    two = g.contribute_srs(g.contribute_srs(honest, TAU2, ALPHA2, BETA2), TAU, ALPHA2, BETA)
    for s in (honest, two):
        for rho in (RHO, RHO2):
            assert pairing_failures(g, g.srs_verification_pairs(s, rho)) == set()


# ---- 3: tampering -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES4)
def test_tampering(curve):
    g = engine(curve)
    r = g.curve.r
    lens, chunk = (300, 150, 150, 150), 64
    e = transcript_exponents(r, lens, TAU, ALPHA, BETA)
    src = T(g, lens)
    cases = []
    for m in VECS:
        n = len(e[m])
        for idx in (1, n // 2, chunk, n - 1):
            cases.append((m, idx))
    cases += [("beta_tau_g1", 0), ("beta_g2", 0)]
    for m, idx in cases:
        s, t = copy_srs(src), {k: (list(v) if k != "beta_g2" else v) for k, v in e.items()}
        if m == "beta_g2":
            t[m] = t[m] * TAU % r
            s.beta_g2[:] = point_of(g, m, t[m])
        else:
            t[m][idx] = t[m][idx] * TAU % r   # a subgroup point, one power of tau too high
            getattr(s, m)[idx] = point_of(g, m, t[m][idx])
        p, q = pair_exponents(t, RHO, r)
        want = expected_failures(m, idx)
        assert failing(p, q, r) == want, (m, idx)
        got = g.srs_verification_pairs(s, RHO, chunk_points=chunk)
        assert_pairs(got, closed(g, p, q), (m, idx))
        if curve in PAIRING and (m, idx) in (("tau_g1", 1), ("tau_g2", chunk), ("alpha_tau_g1", 149), ("beta_g2", 0)):
            assert pairing_failures(g, got) == want, (m, idx)
    # tau_g2 from another tau than tau_g1, and beta_g2 of another beta
    s = copy_srs(src)
    s.tau_g2 = np.ascontiguousarray(T(g, lens, tau=TAU2).tau_g2)
    t = {**e, "tau_g2": transcript_exponents(r, lens, TAU2, ALPHA, BETA)["tau_g2"]}
    got = g.srs_verification_pairs(s, RHO)
    assert_pairs(got, closed(g, *pair_exponents(t, RHO, r)), "mixed tau")
    assert failing(*pair_exponents(t, RHO, r), r) == {0, 1, 2, 3}
    s = copy_srs(src)
    s.beta_g2 = T(g, (2, 2, 1, 1), beta=BETA2).beta_g2
    t = {**e, "beta_g2": BETA2}
    got = g.srs_verification_pairs(s, RHO)
    assert_pairs(got, closed(g, *pair_exponents(t, RHO, r)), "beta_g2")
    assert failing(*pair_exponents(t, RHO, r), r) == {4}
    if curve in PAIRING:
        assert pairing_failures(g, got) == {4}


# ---- 4: refusals --------------------------------------------------------------------------------------------------------
def _desc(arrs, lens=None):
    d = _lib.SrsDesc()
    for k in VECS:
        v = arrs.get(k)
        setattr(d, k, None if v is None else v.ctypes.data_as(_lib.u64p))
        setattr(d, k + "_len", (lens or {}).get(k, 0 if v is None else v.shape[0]))
    v = arrs.get("beta_g2")
    d.beta_g2 = None if v is None else v.ctypes.data_as(_lib.u64p)
    return d


SENTINEL = np.uint64(0xABABABABABABABAB)


def _raw(g, arrs, rho=RHO, flags=0, chunk=0, lens=None, null=(), outs=None):
    """g16_srs_verify_pairs on explicit arrays: (status, g16_last_error(), out_g1, out_g2)"""
    cd = g.codec
    o1 = np.full((10, 2 * g.nq), SENTINEL, dtype=np.uint64) if outs is None else outs[0]
    o2 = np.full((10, g.ng2), SENTINEL, dtype=np.uint64) if outs is None else outs[1]
    g1, g2 = (np.ascontiguousarray(x) for x in (cd.enc_g1([gens(g.curve.name)[0]])[0], cd.enc_g2([gens(g.curve.name)[1]])[0]))
    rr = np.ascontiguousarray(cd.fr.enc1(rho))
    ptr = lambda name, a: None if name in null else a.ctypes.data_as(C.c_void_p)
    d = None if "srs" in null else C.byref(_desc(arrs, lens))
    rc = g._lib.g16_srs_verify_pairs(g._ctx, d, ptr("g1", g1), ptr("g2", g2), ptr("rho", rr), flags, chunk, ptr("o1", o1),
                                     ptr("o2", o2))
    return rc, _lib.last_error(), o1, o2


def _arrays(s: Srs):
    return {k: np.ascontiguousarray(getattr(s, k)) for k in MEMBERS}


def _untouched(o1, o2):
    return (o1 == SENTINEL).all() and (o2 == SENTINEL).all()


@pytest.mark.parametrize("curve", ["bls12_381", "bw6_761"])
def test_argument_errors(curve):
    g = engine(curve)
    arrs = _arrays(T(g, (15, 8, 8, 8)))
    bad = _lib.ERR_BAD_ARGUMENT

    def refused(match, **kw):
        rc, msg, o1, o2 = _raw(g, kw.pop("arrs", arrs), **kw)
        assert rc == bad and match in msg, (rc, msg)
        assert _untouched(o1, o2)

    assert _raw(g, arrs)[0] == 0   # the arguments below are the only thing wrong
    for which in ("srs", "g1", "g2", "rho", "o1", "o2"):
        refused("null argument", null=(which,))
    for k in MEMBERS:
        refused(f"null srs member {k}", arrs={**arrs, k: None}, lens=None if k == "beta_g2" else {k: arrs[k].shape[0]})
    for flags in (1, 4, 3, 1 << 8, 1 << 31):
        refused("takes 0 or G16_SER_VALIDATE", flags=flags)
    for zero in (0, g.curve.r):
        refused("rho must be non-zero", rho=zero)
    for k, need in (("tau_g1", 2), ("tau_g2", 2), ("alpha_tau_g1", 1), ("beta_tau_g1", 1)):
        refused(f"{k} holds {need - 1} points, at least {need} are needed", lens={k: need - 1})
        refused(f"{k} holds {1 << 32} points, at most 2^32 - 1", lens={k: 1 << 32})


def _off_curve(a):
    a[-1] ^= np.uint64(1)   # y's top limb: off the curve, still below q


def _non_canonical(a, nq):
    a[nq - 1] = np.uint64(0xFFFFFFFFFFFFFFFF) >> np.uint64(1)   # x's top limb: x >= q


@pytest.mark.parametrize("curve", CURVES4)
def test_refused_points(curve):
    g = engine(curve)
    lens = (300, 150, 150, 150)
    src = T(g, lens)
    for m in MEMBERS:
        for idx in ((0,) if m == "beta_g2" else (0, 1, 77, lens[VECS.index(m)] - 1)):
            for how, reason in (("identity", "point is the identity"), ("off", "point is not on the curve"),
                                ("big", "non-canonical field element (>= q)")):
                s = copy_srs(src)
                a = getattr(s, m)
                pt = a if m == "beta_g2" else a[idx]
                if how == "identity":
                    pt[:] = 0
                elif how == "off":
                    _off_curve(pt)
                else:
                    _non_canonical(pt, g.nq)
                rc, msg, o1, o2 = _raw(g, _arrays(s), chunk=64)
                assert rc == _lib.ERR_INVALID_DATA and msg == f"{m}[{idx}]: {reason}", (m, idx, how, msg)
                assert _untouched(o1, o2)
    # the first bad point by member, then index; later chunks are not needed to name it
    s = copy_srs(src)
    s.alpha_tau_g1[100][:] = 0
    _off_curve(s.alpha_tau_g1[120])
    _off_curve(s.beta_tau_g1[3])
    with pytest.raises(DeserializeError, match=r"^alpha_tau_g1\[100\]: point is the identity$"):
        g.srs_verification_pairs(s, RHO, chunk_points=7)
    # a wrong generator at index 0 of either group, as a transcript point or as the agreed generator
    for m in ("tau_g1", "tau_g2"):
        s = copy_srs(src)
        getattr(s, m)[0] = point_of(g, m, 2)
        grp = "g1" if m == "tau_g1" else "g2"
        with pytest.raises(DeserializeError, match=rf"^{m}\[0\]: not the generator {grp}$"):
            g.srs_verification_pairs(s, RHO)
    g1 = gens(curve)[0]
    if curve == "bw6_761":
        import bw6_ref as B
        two = B.mul(2, g1)
    else:
        two = P.ctx(P.CURVES[curve]).G1.mul(g1, 2)
    with pytest.raises(DeserializeError, match=r"^tau_g1\[0\]: not the generator g1$"):
        g.srs_verification_pairs(src, RHO, g1=two)
    # the identity stays accepted by the other transcript calls
    s = copy_srs(src)
    s.tau_g2[5][:] = 0
    g.contribute_srs(s, TAU2, ALPHA2, BETA2)


@pytest.mark.parametrize("curve", PAIRING)
def test_torsion_point_needs_validate(curve):
    """a G2 point on the curve but outside the prime-order subgroup: refused with validate only"""
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
    assert Gp.mul((x, y), c.r) is not None
    s = T(g, (15, 8, 8, 8))
    s.tau_g2[5] = g.codec.enc_g2([(x, y)])[0]
    with pytest.raises(DeserializeError, match=r"^tau_g2\[5\]: point is not in the prime-order subgroup$"):
        g.srs_verification_pairs(s, RHO, chunk_points=3)
    g.srs_verification_pairs(s, RHO, validate=False)   # on the curve: only the subgroup check refuses it


# ---- 5: chunking, and the challenge -----------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES4)
def test_chunking(curve):
    g = engine(curve)
    src = T(g, (599, 300, 300, 300))
    want = g.srs_verification_pairs(src, RHO)
    for chunk in (7, 128, 0, 1 << 40):
        assert_pairs(g.srs_verification_pairs(src, RHO, chunk_points=chunk), (want.g1, want.g2), chunk)
    assert_pairs(g.srs_verification_pairs(src, RHO, validate=False, chunk_points=128), (want.g1, want.g2), "no validate")
    # chunks of one point (one MSM per point) on a prefix
    head = Srs(*(getattr(src, m)[:24] for m in VECS), src.beta_g2)
    ref = g.srs_verification_pairs(head, RHO)
    assert_pairs(g.srs_verification_pairs(head, RHO, chunk_points=1), (ref.g1, ref.g2), "chunk 1")
    other = g.srs_verification_pairs(src, RHO2)
    assert not np.array_equal(other.g1, want.g1) and not np.array_equal(other.g2, want.g2)
    r = g.curve.r
    assert_pairs(other, closed(g, *closed_exponents(r, (599, 300, 300, 300), TAU, ALPHA, BETA, RHO2)), "rho2")
    if curve in PAIRING:
        assert pairing_failures(g, other) == set()


# ---- 6: isolation -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", ["bn254", "bw6_761"])
def test_isolation(curve):
    fresh = Groth16(curve, 0)   # no circuit, no key
    try:
        got = fresh.srs_verification_pairs(T(fresh, (31, 16, 16, 16)), RHO)
        assert_pairs(got, closed(fresh, *closed_exponents(fresh.curve.r, (31, 16, 16, 16), TAU, ALPHA, BETA, RHO)))
    finally:
        fresh.close()
    g = engine(curve)
    m, z, _ = synthetic_r1cs(curve, 6, seed=520)
    g.generate_parameters_with_qap(m, ALPHA, BETA, 1, D1, TAU, *gens(curve), export=False)
    prove = lambda: g.create_proof_with_reduction_and_matrices(None, 5, 7, None, m.num_instance_variables,
                                                               m.num_constraints, z)
    before = prove()
    key_before = g.export_proving_key_bytes(compress=False)
    s = T(g, (1 << 12, 1 << 11, 1 << 11, 1 << 11))
    g.srs_verification_pairs(s, RHO, chunk_points=1000)
    g.srs_verification_pairs(s, RHO2)
    after = prove()
    assert all(np.array_equal(getattr(before, k), getattr(after, k)) for k in "abc")
    assert g.export_proving_key_bytes(compress=False) == key_before
    # a proof in flight refuses the call, and it stays in flight
    r_, s_ = (np.ascontiguousarray(g.codec.fr.enc1(v)) for v in (5, 7))
    g.prove_submit_raw(0, r_, s_, z.ctypes.data, 0)
    try:
        rc, msg, o1, o2 = _raw(g, _arrays(s))
        assert rc == _lib.ERR_BAD_ARGUMENT and "in flight" in msg and _untouched(o1, o2)
    finally:
        out = np.zeros_like(np.concatenate([before.a, before.b, before.c]))
        g.prove_wait_raw(0, out)
    assert np.array_equal(out, np.concatenate([before.a, before.b, before.c]))


# ---- 7: a production-size transcript ------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", ["bn254", "bls12_381"])
def test_production_size(curve):
    g = engine(curve)
    n = 1 << 20
    lens = (2 * n - 1, n, n, n)
    s = T(g, lens)
    want = closed(g, *closed_exponents(g.curve.r, lens, TAU, ALPHA, BETA, RHO))
    auto = g.srs_verification_pairs(s, RHO)
    assert_pairs(auto, want, "auto")
    assert_pairs(g.srs_verification_pairs(s, RHO, chunk_points=1 << 18), want, "2^18")


# ---- 8: timings ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", ["bn254", "bw6_761"])
def test_timings_describe_the_call(curve):
    """h2d bytes exactly; per chunk of a group a fixed number of launches and d2h bytes (the check's error word, the MSM's
    slot total and leaf arrays), found from three calls and confirmed by a fourth"""
    g = engine(curve)
    chunk = 64
    src = T(g, (256, 128, 128, 128))
    esz1, esz2, fr = 16 * g.nq, 8 * g.ng2, 8 * g.nr

    def call(lens):
        s = Srs(*(np.ascontiguousarray(getattr(src, m)[:n]) for m, n in zip(VECS, lens)), src.beta_g2)
        g.srs_verification_pairs(s, RHO, chunk_points=chunk)
        tm = _lib.Timings()
        assert g._lib.g16_get_timings(g._ctx, C.byref(tm)) == 0
        c1 = sum(-(-n // chunk) for m, n in zip(VECS, lens) if m != "tau_g2")
        c2 = -(-lens[1] // chunk)
        assert tm.h2d_bytes == (lens[0] + lens[2] + lens[3]) * esz1 + (lens[1] + 1) * esz2 + 32 * fr
        assert [tm.msm_pairs[m] for m in range(5)] == list(lens) + [0]
        assert all(tm.msm_ms[m] > 0 for m in range(4)) and tm.msm_ms[4] == 0
        assert tm.total_ms >= sum(tm.msm_ms[m] for m in range(4))
        assert tm.h2d_ms == 0 and tm.witness_map_ms == 0 and tm.host_finish_ms == 0
        assert all(tm.msm_entries[m] == 0 for m in range(5))
        return c1, c2, tm.launches - 1, tm.d2h_bytes - 8   # beta_g2's check: one launch, one error word
    # every chunk below holds exactly `chunk` points
    (a1, a2, la, da), (b1, b2, lb, db), (c1, c2, lc, dc) = (call(x) for x in ((128, 64, 64, 64), (256, 64, 64, 64),
                                                                             (128, 128, 64, 64)))
    per1, dper1 = (lb - la) // (b1 - a1), (db - da) // (b1 - a1)
    per2, dper2 = (lc - la) // (c2 - a2), (dc - da) // (c2 - a2)
    assert per1 >= 3 and per2 >= 3 and dper1 > 12 and dper2 > 12
    for (x1, x2, lx, dx) in ((a1, a2, la, da), (b1, b2, lb, db), (c1, c2, lc, dc), call((256, 128, 128, 128))):
        assert lx == x1 * per1 + x2 * per2
        assert dx == x1 * dper1 + x2 * dper2
