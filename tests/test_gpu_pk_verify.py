"""GPU tier of g16_pk_verify_pairs (the key check).  Keys come from g16_setup(alpha, beta, gamma, delta, tau) with gamma !=
delta, transcripts from g16_srs_from_secrets(tau, alpha, beta).  Every output point is compared limb for limb with its
closed-form scalar (pk_verify_ref.verdict on the key's exponents) times the generator, formed by the CPU oracle or
tests/bw6_ref.py, never by the device; which equations hold is decided in the exponent on all four curves and with pyref's
pairing on BN254 and BLS12-381."""
import ctypes as C

import numpy as np
import pytest

import bw6_ref as B
import pyref as P
from groth16_b200 import ConstraintMatrices, Groth16, Srs, _lib
from groth16_b200.api import key_members
from groth16_b200.params import GENERATORS
from groth16_b200.serialize import DeserializeError
from groth16_b200.workload import synthetic_r1cs
from pk_verify_ref import (G2_MEMBERS, POINTS, VECTORS, edited_rows, failing, key_exponents, key_sums, tamperings,
                           transcript_sums, verdict)
from util import proof_from_abi

pytestmark = pytest.mark.gpu

CURVES4 = ["bls12_381", "bn254", "bls12_377", "bw6_761"]
PAIRING = ["bn254", "bls12_381"]
TAU, ALPHA, BETA, GAMMA, DELTA = (0x1234567890ABCDEF1234567, 0x2222222222222222222223, 0x3333333333333333333335,
                                  0x6666666666666666666661, 0x4444444444444444444447)
TAU2, ALPHA2, BETA2 = 0x7777777777777777777779ABC, 0x6666666666666666666665, 0x5555555555555555555557
D1, D2 = 0x4444444444444444444449, 0x5555555555555555555559
RHO, RHO2 = 0x5EED5EED5EED5EED5EED5EED5EED5EED1, 0xC0FFEE0C0FFEE0C0FFEE0C0FFEE01
MEMBERS = VECTORS + POINTS

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


def root_of(curve):
    if curve == "bw6_761":
        return B.domain_root
    c = P.CURVES[curve]
    return lambda L: P.Domain(c, 1 << L).omega


def rows_of(g, m):
    out = []
    for rp, col, val in (m.a, m.b, m.c):
        vals = g.codec.fr.dec(val) if len(col) else []
        out.append([[(vals[e], int(col[e])) for e in range(int(rp[i]), int(rp[i + 1]))] for i in range(len(rp) - 1)])
    return out


class Case:
    """a circuit on the engine, its key g16_setup(ALPHA, BETA, GAMMA, DELTA, TAU) and the reference's view of both"""

    def __init__(self, g, log_n, seed, gamma=GAMMA, delta=DELTA):
        self.g, self.curve, self.r = g, g.curve.name, g.curve.r
        self.m, self.z, _ = synthetic_r1cs(self.curve, log_n, seed=seed)
        self.rows, self.ni, self.nw = rows_of(g, self.m), self.m.num_instance_variables, self.m.num_witness_variables
        self.n = 1 << log_n
        self.circom = g.qap == "circom"
        self.pk = g.generate_parameters_with_qap(self.m, ALPHA, BETA, gamma, delta, TAU, *gens(self.curve))
        self.k = key_exponents(self.r, root_of(self.curve), self.rows, self.ni, self.nw, ALPHA, BETA, gamma, delta, TAU,
                               self.circom)

    def sums(self, rho=RHO):
        """S_X(T) from the key's own exponents: the transcript's key has gamma = delta = 1 (test_pk_verify_cpu proves that
        the library's transcript-side weights give exactly these sums)"""
        ks, r = key_sums(self.k, rho, self.r, self.ni), self.r
        return dict(ks, h=ks["h"] * DELTA % r, l=ks["l"] * DELTA % r, ic=ks["ic"] * GAMMA % r)

    def srs(self, extra=0, tau=TAU):
        return self.g.srs_from_secrets(2 * self.n - 1 + extra, self.n + extra, tau, ALPHA, BETA, *gens(self.curve))


def closed(g, p, q):
    """[p_j]g1 and [q_j]g2 as limbs, by the CPU oracle or bw6_ref"""
    curve, cd = g.curve.name, g.codec
    g1, g2 = gens(curve)
    if curve == "bw6_761":
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
    return {k for k in range(4)
            if not cx.pairing_product_is_one([(ps[2 * k], qs[2 * k]), (cx.G1.neg(ps[2 * k + 1]), qs[2 * k + 1])])}


def point_of(g, g2, k):
    """[k]g1 or [k]g2 as limbs (the identity for k = 0), by g16_srs_from_secrets"""
    if k % g.curve.r == 0:
        return np.zeros(g.ng2 if g2 else 2 * g.nq, dtype=np.uint64)
    s = g.srs_from_secrets(2, 2, k, 1, 1, *gens(g.curve.name))
    return (s.tau_g2 if g2 else s.tau_g1)[1]


def copy_pk(pk):
    import copy
    return copy.deepcopy(pk)


def set_point(g, pk, m, idx, k):
    """member m (index idx of a vector) of pk := [k] times its group's generator"""
    pt = point_of(g, m in G2_MEMBERS, k)
    holder = pk.vk if m in ("gamma_abc_g1", "alpha_g1", "beta_g2", "gamma_g2", "delta_g2") else pk
    v = getattr(holder, m)
    if m in VECTORS:
        v[idx] = pt
    else:
        setattr(holder, m, pt)


def expect(g, pk, srs, k, ts, rho=RHO, uncontributed=False, what=""):
    """run the call and compare with pk_verify_ref.verdict: the same refusal, or the closed-form outputs; returns the
    refusal or the set of broken equations"""
    bad, p, q = verdict(k, (TAU, ALPHA, BETA), ts, rho, g.curve.r, len(k["gamma_abc_g1"]), uncontributed)
    if bad is not None:
        with pytest.raises(DeserializeError, match=rf"^{bad}[: ]"):
            g.key_verification_pairs(pk, srs, rho, uncontributed=uncontributed)
        return bad
    got = g.key_verification_pairs(pk, srs, rho, uncontributed=uncontributed)
    assert_pairs(got, closed(g, p, q), what)
    return failing(p, q, g.curve.r)


# ---- 1: closed form -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("qap", ["libsnark", "circom"])
@pytest.mark.parametrize("curve", CURVES4)
def test_closed_form(curve, qap):
    g = engine(curve, qap)
    for log_n in (4, 8, 12):
        c = Case(g, log_n, 600 + log_n)
        ts = c.sums()
        for srs in (c.srs(), c.srs(extra=3)):
            assert expect(g, c.pk, srs, c.k, ts, what=log_n) == set()
        if log_n == 4:
            tm = g.timings()
            nv = c.ni + c.nw
            assert tm["msm_pairs"]["h"] == 3 * nv + len(c.k["h_query"]) + c.nw + c.ni
            assert tm["msm_pairs"]["l"] == 11 * c.n - 1
            assert tm["total_ms"] >= tm["h2d_ms"] > 0 and tm["witness_map_ms"] > 0 and tm["msm_ms"]["h"] > 0
            if curve in PAIRING:
                assert pairing_failures(g, g.key_verification_pairs(c.pk, c.srs(), RHO2)) == set()


# ---- 2: the whole ceremony ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES4)
def test_ceremony(curve):
    g = engine(curve)
    r = g.curve.r
    pc = P.CURVES["bls12_377" if curve == "bw6_761" else curve]
    rng = P.Rng(17)
    a, b = rng.fr(pc.r), rng.fr(pc.r)
    cs = P.silly_circuit(pc, a, b)
    m = ConstraintMatrices.from_rows(curve, cs.num_instance, cs.num_witness, cs.a, cs.b, cs.c)
    srs0 = g.srs_from_secrets(63, 32, TAU, ALPHA, BETA, *gens(curve))
    srs = g.contribute_srs(srs0, TAU2, ALPHA2, BETA2)
    if curve in PAIRING:
        cx, cd = P.ctx(pc), g.codec
        sp = g.srs_verification_pairs(srs, RHO)
        ps, qs = cd.dec_g1(sp.g1), cd.dec_g2(sp.g2)
        assert all(cx.pairing_product_is_one([(ps[2 * k], qs[2 * k]), (cx.G1.neg(ps[2 * k + 1]), qs[2 * k + 1])])
                   for k in range(5))
    k0 = g.generate_parameters_from_srs(m, srs)
    with pytest.raises(DeserializeError, match=r"^gamma_g2 equals delta_g2: "):
        g.key_verification_pairs(k0, srs, RHO)
    p0 = g.key_verification_pairs(k0, srs, RHO, uncontributed=True)
    g.contribute_delta(D1)
    k2 = g.contribute_delta(D2)
    p2 = g.key_verification_pairs(k2, srs, RHO)
    # in the exponent: the transcript is T(TAU TAU2, ALPHA ALPHA2, BETA BETA2)
    t, al, be = TAU * TAU2 % r, ALPHA * ALPHA2 % r, BETA * BETA2 % r
    rows, ni, nw = [cs.a, cs.b, cs.c], cs.num_instance, cs.num_witness
    root = root_of(curve)
    ts = transcript_sums(r, root, rows, ni, nw, t, al, be, RHO, False)
    for pairs, dl in ((p0, 1), (p2, D1 * D2 % r)):
        k = key_exponents(r, root, rows, ni, nw, al, be, 1, dl, t, False)
        bad, p, q = verdict(k, (t, al, be), ts, RHO, r, ni, uncontributed=True)
        assert bad is None and failing(p, q, r) == set()
        assert_pairs(pairs, closed(g, p, q), dl)
        if curve in PAIRING:
            assert pairing_failures(g, pairs) == set()
    if curve in PAIRING:   # proofs under the final key verify
        cd = g.codec
        z = np.ascontiguousarray(cd.fr.enc(cs.assignment))
        pf = g.create_proof_with_reduction_and_matrices(None, 5, 7, None, cs.num_instance, cs.num_constraints, z)
        vk = P.VerifyingKey(cd.dec_g1(k2.vk.alpha_g1)[0], cd.dec_g2(k2.vk.beta_g2)[0], cd.dec_g2(k2.vk.gamma_g2)[0],
                            cd.dec_g2(k2.vk.delta_g2)[0], cd.dec_g1(k2.vk.gamma_abc_g1))
        pub = cd.fr.dec(z)[1:cs.num_instance]
        assert P.verify_proof(vk, pc, proof_from_abi(curve, pf), pub)


# ---- 3: tampering -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES4)
def test_tampering(curve):
    g = engine(curve)
    r = g.curve.r
    c = Case(g, 6, 610)
    srs, ts = c.srs(), c.sums()
    seen = {}
    for what, t, want in tamperings(c.k, r):
        pk = copy_pk(c.pk)
        for m in MEMBERS:
            if m in VECTORS:
                for idx, (x, y) in enumerate(zip(t[m], c.k[m])):
                    if x != y:
                        set_point(g, pk, m, idx, x)
            elif t[m] != c.k[m]:
                set_point(g, pk, m, 0, t[m])
        got = expect(g, pk, srs, t, ts, what=what)
        assert got == want, (what, got, want)
        seen[what] = got
        if curve in PAIRING and what in ("h_query[0] changed", "delta_g2 changed", "gamma_g2 changed"):
            assert pairing_failures(g, g.key_verification_pairs(pk, srs, RHO)) == want, what
    assert len(seen) >= 24
    # a key for another tau
    other = engine(curve).generate_parameters_with_qap(c.m, ALPHA, BETA, GAMMA, DELTA, TAU2, *gens(curve))
    with pytest.raises(DeserializeError, match=r"^a_query: not the key of the resident circuit under this transcript$"):
        g.key_verification_pairs(other, srs, RHO)
    # keys of circuits with one coefficient changed (made resident, then the original circuit again)
    for which in range(4):
        try:
            edited, want = edited_rows(c.rows, which, c.ni)
        except ValueError:   # the synthetic circuit's C reads no instance variable
            continue
        em = ConstraintMatrices.from_rows(curve, c.ni, c.nw, *edited)
        ek = g.generate_parameters_with_qap(em, ALPHA, BETA, GAMMA, DELTA, TAU, *gens(curve))
        g.load_matrices(c.m)
        kx = key_exponents(r, root_of(curve), edited, c.ni, c.nw, ALPHA, BETA, GAMMA, DELTA, TAU, False)
        assert expect(g, ek, srs, kx, ts, what=("edited", which)) == want, which
    # a key made under the other reduction
    gc = engine(curve, "circom")
    ck = gc.generate_parameters_with_qap(c.m, ALPHA, BETA, GAMMA, DELTA, TAU, *gens(curve))
    kx = key_exponents(r, root_of(curve), c.rows, c.ni, c.nw, ALPHA, BETA, GAMMA, DELTA, TAU, True)
    ck.h_query = ck.h_query[:c.n - 1]   # the lengths of the libsnark key; the points are the circom key's
    kx["h_query"] = kx["h_query"][:c.n - 1]
    assert expect(g, ck, srs, kx, ts, what="circom key") == {1}
    ts_c = transcript_sums(r, root_of(curve), c.rows, c.ni, c.nw, TAU, ALPHA, BETA, RHO, True)
    lk = copy_pk(c.pk)
    lk.h_query = np.concatenate([lk.h_query, point_of(g, False, 0)[None]])   # a libsnark key padded to n points
    kx = dict(c.k, h_query=c.k["h_query"] + [0])
    assert expect(gc, lk, srs, kx, ts_c, what="libsnark key") == {1}


# ---- 4: bad points -------------------------------------------------------------------------------------------------------
SENTINEL = np.uint64(0xABABABABABABABAB)


def _raw(g, keys, arrs, rho=RHO, flags=0, null=(), lens=None, outs=None):
    """g16_pk_verify_pairs on explicit arrays: (status, g16_last_error(), out_g1, out_g2)"""
    d = _lib.PkCheckDesc()
    for k, v in keys.items():
        setattr(d, k, None if k in null or v is None else v.ctypes.data_as(_lib.u64p))
    s = _lib.SrsDesc()
    for k in ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1"):
        setattr(s, k, None if k in null else arrs[k].ctypes.data_as(_lib.u64p))
        setattr(s, k + "_len", (lens or {}).get(k, arrs[k].shape[0]))
    s.beta_g2 = None if "beta_g2_srs" in null else arrs["beta_g2"].ctypes.data_as(_lib.u64p)
    o1 = np.full((8, 2 * g.nq), SENTINEL, dtype=np.uint64) if outs is None else outs[0]
    o2 = np.full((8, g.ng2), SENTINEL, dtype=np.uint64) if outs is None else outs[1]
    rr = np.ascontiguousarray(g.codec.fr.enc1(rho))
    ptr = lambda name, a: None if name in null else a.ctypes.data_as(C.c_void_p)
    rc = g._lib.g16_pk_verify_pairs(g._ctx, None if "srs" in null else C.byref(s), None if "pk" in null else C.byref(d),
                                    ptr("rho", rr), flags, ptr("o1", o1), ptr("o2", o2))
    return rc, _lib.last_error(), o1, o2


def _keys(g, pk):
    out = {}
    for k, v in key_members(pk).items():
        w = g.ng2 if k in G2_MEMBERS else 2 * g.nq
        out[k] = np.ascontiguousarray(v, dtype=np.uint64).reshape(-1, w)
    return out


def _arrays(s: Srs):
    return {k: np.ascontiguousarray(getattr(s, k)) for k in ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1", "beta_g2")}


def _untouched(o1, o2):
    return (o1 == SENTINEL).all() and (o2 == SENTINEL).all()


def _off_curve(a):
    a[-1] ^= np.uint64(1)   # y's top limb: off the curve, still below q


def _non_canonical(a, nq):
    a[nq - 1] = np.uint64(0xFFFFFFFFFFFFFFFF) >> np.uint64(1)   # x's top limb: x >= q


@pytest.mark.parametrize("curve", CURVES4)
def test_bad_points(curve):
    g = engine(curve)
    c = Case(g, 5, 620)
    keys, arrs = _keys(g, c.pk), _arrays(c.srs(extra=5))
    cases = [("a_query", 0), ("b_g2_query", 3), ("h_query", 30), ("l_query", 17), ("gamma_abc_g1", 1), ("delta_g2", 0),
             ("alpha_g1", 0), ("tau_g1", 3), ("tau_g1", 62), ("tau_g2", 31), ("beta_tau_g1", 0), ("beta_g2", 0)]
    for m, idx in cases:
        for how, reason in (("off", "point is not on the curve"), ("big", "non-canonical field element (>= q)")):
            k2 = {x: v.copy() for x, v in keys.items()}
            a2 = {x: v.copy() for x, v in arrs.items()}
            src = k2 if m in k2 else a2
            pt = src[m].reshape(-1, src[m].shape[-1])[idx]
            _off_curve(pt) if how == "off" else _non_canonical(pt, g.nq)
            rc, msg, o1, o2 = _raw(g, k2, a2, flags=_lib.SER_VALIDATE)
            assert rc == _lib.ERR_INVALID_DATA and msg == f"{m}[{idx}]: {reason}", (m, idx, how, msg)
            assert _untouched(o1, o2)
    # key points before transcript points, then by member and index
    k2, a2 = {x: v.copy() for x, v in keys.items()}, {x: v.copy() for x, v in arrs.items()}
    _off_curve(a2["tau_g1"][1])
    _off_curve(k2["l_query"][9])
    _off_curve(k2["l_query"][4])
    assert _raw(g, k2, a2)[1] == "l_query[4]: point is not on the curve"
    # the identity is valid in the key's vectors: a key whose a_query[5] is the identity is refused by its sum only
    k2 = {x: v.copy() for x, v in keys.items()}
    k2["a_query"][5] = 0
    rc, msg, _, _ = _raw(g, k2, arrs)
    assert rc == _lib.ERR_INVALID_DATA and msg.startswith("a_query: not the key"), msg
    a2 = {x: v.copy() for x, v in arrs.items()}
    a2["tau_g2"][0] = 0
    assert _raw(g, keys, a2)[1] == "tau_g2[0]: point is the identity"


@pytest.mark.parametrize("curve", PAIRING)
def test_torsion_point_needs_validate(curve):
    """a G2 point on the curve but outside the prime-order subgroup: refused with validate only"""
    g = engine(curve)
    cc = P.CURVES[curve]
    Gp = P.ctx(cc).G2
    F = Gp.F
    x = F.from_int(1)
    while True:
        y = F.sqrt(F.add(F.mul(F.mul(x, x), x), Gp.b))
        if y is not None:
            break
        x = F.add(x, F.from_int(1))
    assert Gp.mul((x, y), cc.r) is not None
    c = Case(g, 4, 630)
    srs = c.srs()
    pk = copy_pk(c.pk)
    pk.b_g2_query[3] = g.codec.enc_g2([(x, y)])[0]
    with pytest.raises(DeserializeError, match=r"^b_g2_query\[3\]: point is not in the prime-order subgroup$"):
        g.key_verification_pairs(pk, srs, RHO)
    with pytest.raises(DeserializeError, match=r"^b_g2_query: not the key"):
        g.key_verification_pairs(pk, srs, RHO, validate=False)
    srs.tau_g2[7] = g.codec.enc_g2([(x, y)])[0]
    with pytest.raises(DeserializeError, match=r"^tau_g2\[7\]: point is not in the prime-order subgroup$"):
        g.key_verification_pairs(c.pk, srs, RHO)


# ---- 5: argument errors, and no key resident ----------------------------------------------------------------------------
@pytest.mark.parametrize("curve", ["bls12_381", "bw6_761"])
def test_argument_errors(curve):
    g = engine(curve)
    c = Case(g, 4, 640)
    keys, arrs = _keys(g, c.pk), _arrays(c.srs())
    bad = _lib.ERR_BAD_ARGUMENT

    def refused(match, gg=g, **kw):
        rc, msg, o1, o2 = _raw(gg, kw.pop("keys", keys), arrs, **kw)
        assert rc == bad and match in msg, (rc, msg)
        assert _untouched(o1, o2)

    assert _raw(g, keys, arrs)[0] == 0   # the arguments below are the only thing wrong
    for which in ("srs", "pk", "rho", "o1", "o2"):
        refused("null argument", null=(which,))
    for k in MEMBERS:
        refused(f"null pk member {k}", null=(k,))
    for k in ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1"):
        refused(f"null srs member {k}", null=(k,))
    refused("null srs member beta_g2", null=("beta_g2_srs",))
    for flags in (1, 8, 3, 1 << 8, 1 << 31):
        refused("takes G16_SER_VALIDATE and G16_PK_UNCONTRIBUTED only", flags=flags)
    for zero in (0, g.curve.r):
        refused("rho must be non-zero", rho=zero)
    n = c.n
    for k, need in (("tau_g1", 2 * n - 1), ("tau_g2", n), ("alpha_tau_g1", n), ("beta_tau_g1", n)):
        refused(f"{k} holds {need - 1} points, the circuit (domain 2^4) needs at least {need}", lens={k: need - 1})
    fresh = Groth16(curve, 0)   # no circuit
    try:
        refused("g16_circuit_load must precede g16_pk_verify_pairs", gg=fresh)
        # a circuit and no key: the call works
        fresh.load_matrices(c.m)
        rc, msg, o1, o2 = _raw(fresh, keys, arrs)
        assert rc == 0, msg
        ts = c.sums()
        _, p, q = verdict(c.k, (TAU, ALPHA, BETA), ts, RHO, g.curve.r, c.ni)
        want = closed(g, p, q)
        assert np.array_equal(o1, want[0]) and np.array_equal(o2, want[1])
    finally:
        fresh.close()


# ---- 6: isolation -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", ["bn254", "bw6_761"])
def test_isolation(curve):
    g = engine(curve)
    c = Case(g, 6, 650)
    prove = lambda: g.create_proof_with_reduction_and_matrices(None, 5, 7, None, c.ni, c.m.num_constraints, c.z)
    before = prove()
    key_before = g.export_proving_key_bytes(compress=False)
    limbs_before = g.export_proving_key()
    srs = c.srs()
    g.key_verification_pairs(c.pk, srs, RHO)
    other = copy_pk(c.pk)   # a key that is not the resident one, refused
    other.a_query[1] = other.a_query[2]
    with pytest.raises(DeserializeError, match="^a_query: not the key"):
        g.key_verification_pairs(other, srs, RHO)
    after = prove()
    assert all(np.array_equal(getattr(before, k), getattr(after, k)) for k in "abc")
    assert g.export_proving_key_bytes(compress=False) == key_before
    limbs_after = g.export_proving_key()
    for k, v in key_members(limbs_before).items():
        assert np.array_equal(v, key_members(limbs_after)[k]), k
    # a proof in flight refuses the call, and it stays in flight
    r_, s_ = (np.ascontiguousarray(g.codec.fr.enc1(v)) for v in (5, 7))
    g.prove_submit_raw(0, r_, s_, c.z.ctypes.data, 0)
    try:
        rc, msg, o1, o2 = _raw(g, _keys(g, c.pk), _arrays(srs))
        assert rc == _lib.ERR_BAD_ARGUMENT and "in flight" in msg and _untouched(o1, o2)
    finally:
        out = np.zeros_like(np.concatenate([before.a, before.b, before.c]))
        g.prove_wait_raw(0, out)
    assert np.array_equal(out, np.concatenate([before.a, before.b, before.c]))


# ---- 7: production size -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("qap", ["libsnark", "circom"])
@pytest.mark.parametrize("curve", PAIRING)
def test_production_size(curve, qap):
    g = engine(curve, qap)
    r = g.curve.r
    c = Case(g, 20, 660)
    srs, ts = c.srs(), c.sums()
    assert expect(g, c.pk, srs, c.k, ts, what="2^20") == set()
    idx = 12345
    pk = copy_pk(c.pk)
    t = dict(c.k, l_query=list(c.k["l_query"]))
    t["l_query"][idx] = t["l_query"][idx] * 3 % r
    set_point(g, pk, "l_query", idx, t["l_query"][idx])
    assert key_sums(t, RHO, r, c.ni)["l"] != key_sums(c.k, RHO, r, c.ni)["l"]
    assert expect(g, pk, srs, t, ts, what="2^20 l_query") == {2}
