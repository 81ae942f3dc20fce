"""GPU tier of the phase-2 ceremony calls: g16_pk_contribute (a delta contribution to a key held in host memory) and
g16_contribution_chain_pairs (the contributions' proofs of knowledge).  A contribution delta to an exported
g16_setup(alpha, beta, gamma, delta0, tau) key must be g16_setup(alpha, beta, gamma, delta0 delta, tau) in every limb and
what g16_setup_contribute makes of the resident key; chain outputs are compared limb for limb with closed-form multiples
of the generators (the CPU oracle or tests/bw6_ref.py, never the device).  The multi-party ceremony runs end to end, its
equations decided by pyref's pairing on BN254 and BLS12-381 and in the exponent on BLS12-377 and BW6-761."""
import copy
import ctypes as C

import numpy as np
import pytest

import pyref as P
from contribution_chain_ref import MEMBERS as REC_MEMBERS
from contribution_chain_ref import chain, failing, tamperings, verdict
from groth16_b200 import ContributionRecord, Groth16, _lib
from groth16_b200.params import GENERATORS
from groth16_b200.serialize import DeserializeError
from groth16_b200.workload import synthetic_r1cs
from test_gpu_pk_verify import closed
from util import matrices_from_r1cs, pk_from_abi, proof_from_abi

pytestmark = pytest.mark.gpu

CURVES4 = ["bls12_381", "bn254", "bls12_377", "bw6_761"]
PAIRING = ["bn254", "bls12_381"]
TAU, ALPHA, BETA, GAMMA, DELTA0 = (0x1234567890ABCDEF1234567, 0x2222222222222222222223, 0x3333333333333333333335,
                                   0x6666666666666666666661, 0x4444444444444444444447)
XS = (0x4444444444444444444449, 0x5555555555555555555559, 0x77777777777777777777771)
PHASE1 = [(0x7777777777777777777779ABC, 0x6666666666666666666665, 0x5555555555555555555557),
          (0x99999999999999999999999B, 0x8888888888888888888885, 0xAAAAAAAAAAAAAAAAAAAAAD),
          (0x1357913579135791357913, 0x2468024680246802468021, 0x3691236912369123691237)]
RHO = 0x5EED5EED5EED5EED5EED5EED5EED5EED1
KEY = ("a_query", "b_g1_query", "b_g2_query", "h_query", "l_query", "beta_g1", "delta_g1")
VK = ("alpha_g1", "beta_g2", "gamma_g2", "delta_g2", "gamma_abc_g1")

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


def prod(r, *xs):
    out = 1
    for x in xs:
        out = out * x % r
    return out


def assert_same_key(a, b, what=""):
    for k in KEY:
        assert np.array_equal(np.asarray(getattr(a, k)).reshape(-1), np.asarray(getattr(b, k)).reshape(-1)), (k, what)
    for k in VK:
        assert np.array_equal(np.asarray(getattr(a.vk, k)).reshape(-1), np.asarray(getattr(b.vk, k)).reshape(-1)), (k, what)


def setup_key(g, m, delta):
    return g.generate_parameters_with_qap(m, ALPHA, BETA, GAMMA, delta, TAU, *gens(g.curve.name))


# ---- contribution equals the closed form --------------------------------------------------------------------------------
@pytest.mark.parametrize("qap", ["libsnark", "circom"])
@pytest.mark.parametrize("curve", CURVES4)
def test_contribution_is_setup_of_the_product(curve, qap):
    g = engine(curve, qap)
    r = g.curve.r
    for log_n in range(4, 13):
        m, _, _ = synthetic_r1cs(curve, log_n, seed=600 + log_n)
        pk0 = setup_key(g, m, DELTA0)
        got = g.contribute_key(pk0, XS[0])
        resident = g.contribute_delta(XS[0])   # the resident key is pk0: g16_setup_contribute on it
        assert_same_key(got, resident, ("resident", log_n))
        assert_same_key(got, setup_key(g, m, prod(r, DELTA0, XS[0])), log_n)
        # untouched members are the input's own arrays
        assert got.a_query is pk0.a_query and got.vk.gamma_abc_g1 is pk0.vk.gamma_abc_g1 and got.beta_g1 is pk0.beta_g1


@pytest.mark.parametrize("curve", PAIRING)
def test_production_size(curve):
    g = engine(curve)
    m, _, _ = synthetic_r1cs(curve, 20, seed=620)
    pk = setup_key(g, m, DELTA0)
    got = g.contribute_key(pk, XS[1], in_place=True)
    assert got is pk
    assert_same_key(got, setup_key(g, m, prod(g.curve.r, DELTA0, XS[1])))


# ---- chunking, in place, identity points --------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES4)
def test_chunking_and_layout(curve):
    g = engine(curve)
    m, _, _ = synthetic_r1cs(curve, 9, seed=630)
    pk = setup_key(g, m, DELTA0)
    want = setup_key(g, m, prod(g.curve.r, DELTA0, XS[2]))
    for j in (0, 5, len(pk.l_query) - 1):   # identity points stay the identity
        pk.l_query[j] = 0
        want.l_query[j] = 0
    outs = []
    for chunk in (1, 7, 128, 0):
        for in_place in (False, True):
            k = copy.deepcopy(pk)
            outs.append(g.contribute_key(k, XS[2], chunk_points=chunk, in_place=in_place, validate=chunk == 7))
    for got in outs:
        assert_same_key(got, want)


def test_empty_queries():
    """h_query and l_query of no points: only delta_g1 and delta_g2 change"""
    g = engine("bn254")
    m, _, _ = synthetic_r1cs("bn254", 4, seed=640)
    pk = setup_key(g, m, DELTA0)
    want = setup_key(g, m, prod(g.curve.r, DELTA0, XS[0]))
    pk.h_query, pk.l_query = pk.h_query[:0], None
    with pytest.raises(ValueError, match="no l_query"):
        g.contribute_key(pk, XS[0])
    pk.l_query = np.zeros((0, 2 * g.nq), dtype=np.uint64)
    got = g.contribute_key(pk, XS[0])
    assert got.h_query.shape == (0, 2 * g.nq) and got.l_query.shape == (0, 2 * g.nq)
    assert np.array_equal(got.delta_g1, want.delta_g1) and np.array_equal(got.vk.delta_g2, want.vk.delta_g2)


# ---- refusals ----------------------------------------------------------------------------------------------------------
def _off_curve(a):
    a[-1] ^= np.uint64(1)   # y's top limb: off the curve, still below q


def _raw(g, pk, delta=XS[0], flags=0, chunk=0, out_lens=None, alias=None, null=()):
    """g16_pk_contribute on pk's arrays into fresh sentinel arrays: (status, g16_last_error(), outputs)"""
    ins = dict(h_query=np.ascontiguousarray(pk.h_query), l_query=np.ascontiguousarray(pk.l_query),
               delta_g1=np.ascontiguousarray(pk.delta_g1), delta_g2=np.ascontiguousarray(pk.vk.delta_g2))
    outs = {k: np.full_like(v, 0xA5A5A5A5A5A5A5A5) for k, v in ins.items()}
    if alias:
        outs[alias[0]] = ins[alias[1]]
    d_in, d_out = _lib.PkDeltaDesc(), _lib.PkDeltaOut()
    for d, arrs, lens in ((d_in, ins, None), (d_out, outs, out_lens)):
        for k in ("h_query", "l_query"):
            setattr(d, k, None if k in null else arrs[k].ctypes.data_as(_lib.u64p))
            setattr(d, k.replace("_query", "_len"), (lens or {}).get(k, arrs[k].shape[0]))
        d.delta_g1, d.delta_g2 = (arrs[k].ctypes.data_as(_lib.u64p) for k in ("delta_g1", "delta_g2"))
    dl = np.ascontiguousarray(g.codec.fr.enc1(delta))
    rc = g._lib.g16_pk_contribute(g._ctx, C.byref(d_in), dl.ctypes.data_as(C.c_void_p), flags, chunk, C.byref(d_out))
    return rc, _lib.last_error(), outs


def test_argument_errors():
    g = engine("bls12_377")
    m, _, _ = synthetic_r1cs("bls12_377", 6, seed=650)
    pk = setup_key(g, m, DELTA0)
    nh = len(pk.h_query)
    cases = [
        (dict(flags=8), "takes 0 or G16_SER_VALIDATE"),
        (dict(delta=0), "UnexpectedIdentity"),
        (dict(delta=g.curve.r), "UnexpectedIdentity"),
        (dict(out_lens={"h_query": nh - 1}), "the lengths must be equal"),
        (dict(null=("l_query",)), "null key member l_query"),
        (dict(alias=("l_query", "h_query"), out_lens={"l_query": len(pk.l_query)}), "overlaps in h_query"),
        (dict(alias=("delta_g1", "h_query")), "overlaps in h_query"),
    ]
    for kw, match in cases:
        rc, msg, outs = _raw(g, pk, **kw)
        assert rc == _lib.ERR_BAD_ARGUMENT and match in msg, (kw, msg)
        assert all((v == 0xA5A5A5A5A5A5A5A5).all() for k, v in outs.items() if not kw.get("alias") or k != kw["alias"][0])
    with pytest.raises(ValueError, match="UnexpectedIdentity"):
        g.contribute_key(pk, 0)


@pytest.mark.parametrize("curve", ["bls12_381", "bw6_761"])
def test_refused_point_writes_nothing(curve):
    g = engine(curve)
    m, _, _ = synthetic_r1cs(curve, 17, seed=660)
    src = setup_key(g, m, DELTA0)
    k = 70001
    pk = copy.deepcopy(src)
    _off_curve(pk.l_query[k])
    _off_curve(pk.l_query[k + 5])          # a later bad point in the same chunk is not the one named
    _off_curve(pk.l_query[k + 40000])      # nor one in a later chunk
    _off_curve(pk.vk.delta_g2)             # nor a later member
    rc, msg, outs = _raw(g, pk, chunk=1000)
    assert rc == _lib.ERR_INVALID_DATA and msg == f"l_query[{k}]: point is not on the curve", msg
    assert all((v == 0xA5A5A5A5A5A5A5A5).all() for v in outs.values())
    before = copy.deepcopy(pk)
    with pytest.raises(DeserializeError, match=rf"^l_query\[{k}\]: point is not on the curve$"):
        g.contribute_key(pk, XS[0], chunk_points=1000, in_place=True)
    assert_same_key(pk, before)
    for member, match in (("delta_g2", "delta_g2: point is the identity"), ("delta_g1", "delta_g1: point is the identity")):
        pk = copy.deepcopy(src)
        holder = pk.vk if member == "delta_g2" else pk
        getattr(holder, member)[:] = 0
        before = copy.deepcopy(pk)
        with pytest.raises(DeserializeError, match=rf"^{match}$"):
            g.contribute_key(pk, XS[0], in_place=True, chunk_points=7)
        assert_same_key(pk, before)
    pk = copy.deepcopy(src)
    _off_curve(pk.h_query[len(pk.h_query) - 1])
    with pytest.raises(DeserializeError, match=rf"^h_query\[{len(pk.h_query) - 1}\]: point is not on the curve$"):
        g.contribute_key(pk, XS[0], chunk_points=7)


@pytest.mark.parametrize("curve", ["bls12_381", "bls12_377"])
def test_torsion_point_needs_validate(curve):
    """a G1 point on the curve but outside the prime-order subgroup: refused with validate only"""
    g = engine(curve)
    c = P.CURVES[curve]
    Gp = P.ctx(c).G1
    F = Gp.F
    x = F.from_int(1)
    while True:
        y = F.sqrt(F.add(F.mul(F.mul(x, x), x), Gp.b))
        if y is not None:
            break
        x = F.add(x, F.from_int(1))
    Tp = (x, y)
    assert Gp.mul(Tp, c.r) is not None
    m, _, _ = synthetic_r1cs(curve, 6, seed=670)
    pk = setup_key(g, m, DELTA0)
    pk.h_query[9] = g.codec.enc_g1([Tp])[0]
    with pytest.raises(DeserializeError, match=r"^h_query\[9\]: point is not in the prime-order subgroup$"):
        g.contribute_key(pk, XS[0], validate=True, chunk_points=4)
    got = g.contribute_key(pk, XS[0])
    assert g.codec.dec_g1(got.h_query[9])[0] == Gp.mul(Tp, pow(XS[0], -1, c.r))
    # and in a chain, where end_g1 is named before the records
    start, tp = pk.delta_g1, pk.h_query[9]
    rec = ContributionRecord(tp, tp, tp, pk.vk.delta_g2, pk.vk.delta_g2)
    with pytest.raises(DeserializeError, match=r"^end_g1: point is not in the prime-order subgroup$"):
        g.contribution_chain_pairs(start, tp, [rec])
    with pytest.raises(DeserializeError, match=r"^records\[0\]\.after_g1: point is not in the prime-order subgroup$"):
        g.contribution_chain_pairs(start, start, [rec])
    assert len(g.contribution_chain_pairs(start, tp, [rec], validate=False)) == 2


# ---- the chain check ---------------------------------------------------------------------------------------------------
def chain_points(g, start, end, recs):
    """the exponents of a chain as limbs: (start, end, [ContributionRecord]) by the CPU oracle or bw6_ref"""
    e1 = [start, end] + [c[m] for c in recs for m in REC_MEMBERS[:3]]
    e2 = [c[m] for c in recs for m in REC_MEMBERS[3:]]
    p1, p2 = closed(g, [x % g.curve.r for x in e1], [x % g.curve.r for x in e2])
    p1[[i for i, x in enumerate(e1) if x % g.curve.r == 0]] = 0
    p2[[i for i, x in enumerate(e2) if x % g.curve.r == 0]] = 0
    records = [ContributionRecord(p1[2 + 3 * i], p1[3 + 3 * i], p1[4 + 3 * i], p2[2 * i], p2[2 * i + 1])
               for i in range(len(recs))]
    return p1[0], p1[1], records


@pytest.mark.parametrize("curve", CURVES4)
def test_chain_pairs_closed_form(curve):
    """honest chains of 1 to 5 records, and every tampering of a chain of three: the refusal the reference names, or the
    output points of the reference's exponents, limb for limb"""
    g = engine(curve)
    r = g.curve.r
    xs = XS + (0x1111111111111111111113, 0x2222222222222222222229)
    cases = [(f"honest {n}", TAU, *chain(TAU, xs[:n], r), set()) for n in range(1, 6)]
    cases += list(tamperings(TAU, xs[:3], r, other_start=ALPHA))
    for name, start, end, recs, want in cases:
        s, e, records = chain_points(g, start, end, recs)
        v = verdict(start, end, recs, r)
        if isinstance(want, str):
            with pytest.raises(DeserializeError, match="^" + want.replace("[", r"\[").replace("]", r"\]") + "$"):
                g.contribution_chain_pairs(s, e, records)
            continue
        got = g.contribution_chain_pairs(s, e, records)
        assert failing(v[1], v[2], r) == want, name
        assert len(got) == 2 * len(recs)
        p, q = closed(g, v[1], v[2])
        assert np.array_equal(got.g1, p) and np.array_equal(got.g2, q), name


def test_chain_argument_errors():
    g = engine("bn254")
    r = g.curve.r
    end, recs = chain(TAU, XS, r)
    s, e, records = chain_points(g, TAU, end, recs)
    with pytest.raises(ValueError, match="1 to 2\\^30 - 1 records"):
        g.contribution_chain_pairs(s, e, [])
    with pytest.raises(ValueError, match=r"records\[1\]\.r_g2 is missing"):
        g.contribution_chain_pairs(s, e, records[:1] + [ContributionRecord(records[1].after_g1, records[1].s_g1,
                                                                           records[1].s_x_g1, None, records[1].r_x_g2)])
    descs = (_lib.ContributionRecord * 3)()
    for d, c in zip(descs, records):
        for m in REC_MEMBERS:
            setattr(d, m, np.ascontiguousarray(getattr(c, m)).ctypes.data_as(_lib.u64p))
    o1, o2 = np.full((12, 8), 7, dtype=np.uint64), np.full((12, 16), 7, dtype=np.uint64)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)
    keep = [np.ascontiguousarray(getattr(c, m)) for c in records for m in REC_MEMBERS]
    for d, i in zip(descs, range(3)):
        for j, m in enumerate(REC_MEMBERS):
            setattr(d, m, keep[5 * i + j].ctypes.data_as(_lib.u64p))
    for args, match in (((ptr(s), ptr(e), descs, 0, 0), "count is 0"), ((ptr(s), ptr(e), descs, 3, 4), "takes 0 or"),
                        ((None, ptr(e), descs, 3, 0), "null argument")):
        rc = g._lib.g16_contribution_chain_pairs(g._ctx, *args, ptr(o1), ptr(o2))
        assert rc == _lib.ERR_BAD_ARGUMENT and match in _lib.last_error()
    descs[2].s_x_g1 = None
    rc = g._lib.g16_contribution_chain_pairs(g._ctx, ptr(s), ptr(e), descs, 3, 0, ptr(o1), ptr(o2))
    assert rc == _lib.ERR_BAD_ARGUMENT and "records[2].s_x_g1 is null" in _lib.last_error()
    assert (o1 == 7).all() and (o2 == 7).all()


# ---- resident state ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", ["bn254", "bw6_761"])
def test_resident_state_untouched(curve):
    g = engine(curve)
    m, z, _ = synthetic_r1cs(curve, 8, seed=680)
    pk = setup_key(g, m, DELTA0)
    prove = lambda: g.create_proof_with_reduction_and_matrices(None, 5, 7, None, m.num_instance_variables,
                                                               m.num_constraints, z)
    before = prove()
    key_before = g.export_proving_key_bytes(compress=False)
    g.contribute_key(pk, XS[0], chunk_points=100)
    g.contribute_key(copy.deepcopy(pk), XS[1], in_place=True, validate=True)
    end, recs = chain(1, XS, g.curve.r)
    g.contribution_chain_pairs(*chain_points(g, 1, end, recs))
    after = prove()
    assert all(np.array_equal(getattr(before, k), getattr(after, k)) for k in "abc")
    assert g.export_proving_key_bytes(compress=False) == key_before
    r_, s_ = (np.ascontiguousarray(g.codec.fr.enc1(v)) for v in (5, 7))
    g.prove_submit_raw(0, r_, s_, z.ctypes.data, 0)
    try:
        with pytest.raises(ValueError, match="in flight"):
            g.contribute_key(pk, XS[0])
        with pytest.raises(ValueError, match="in flight"):
            g.contribution_chain_pairs(*chain_points(g, 1, end, recs))
    finally:
        out = np.zeros_like(np.concatenate([before.a, before.b, before.c]))
        g.prove_wait_raw(0, out)
    assert np.array_equal(out, np.concatenate([before.a, before.b, before.c]))


# ---- the multi-party ceremony, end to end ------------------------------------------------------------------------------
def _point(g, k, g2=False):
    """[k] times the generator as limbs, by the CPU oracle or bw6_ref"""
    p1, p2 = closed(g, [k % g.curve.r], [k % g.curve.r])
    return p2[0] if g2 else p1[0]


def _record(g, x, after, s, rr):
    """contributor's published record: s and r as exponents, after the point it computed"""
    return ContributionRecord(np.ascontiguousarray(after), _point(g, s), _point(g, s * x), _point(g, rr, True),
                              _point(g, rr * x, True))


def _holds(g, pairs) -> set:
    """the failing equations of pairs, by pyref's pairing"""
    cx = P.ctx(P.CURVES[g.curve.name])
    ps, qs = g.codec.dec_g1(pairs.g1), g.codec.dec_g2(pairs.g2)
    n = len(ps) // 2
    return {k for k in range(n)
            if not cx.pairing_product_is_one([(ps[2 * k], qs[2 * k]), (cx.G1.neg(ps[2 * k + 1]), qs[2 * k + 1])])}


@pytest.mark.parametrize("curve", CURVES4)
def test_multi_party_ceremony(curve):
    g = engine(curve)
    r = g.curve.r
    pc = P.CURVES["bls12_377" if curve == "bw6_761" else curve]
    rng = P.Rng(31)
    a, b = rng.fr(pc.r), rng.fr(pc.r)
    cs = P.silly_circuit(pc, a, b) if curve != "bw6_761" else None
    m = matrices_from_r1cs(cs) if cs else synthetic_r1cs(curve, 4, seed=690)[0]
    need = m.num_constraints + m.num_instance_variables
    n = 1 << max(need - 1, 0).bit_length()
    # phase 1: three contributions, each with a record per chain
    srs = g.srs_from_secrets(2 * n - 1, n, TAU, ALPHA, BETA, *gens(curve))
    heads = lambda s: (s.tau_g1[1], s.alpha_tau_g1[0], s.beta_tau_g1[0])
    starts = [np.array(h) for h in heads(srs)]
    p1_recs = [[], [], []]
    for k, secrets in enumerate(PHASE1):
        srs = g.contribute_srs(srs, *secrets)
        for j, after in enumerate(heads(srs)):
            p1_recs[j].append(_record(g, secrets[j], after, 0x51 + 3 * k + j, 0x61 + 5 * k + j))
    srs_pairs = g.srs_verification_pairs(srs, RHO)
    p1_pairs = [g.contribution_chain_pairs(starts[j], heads(srs)[j], p1_recs[j]) for j in range(3)]
    # phase 2: the key with delta = 1, then three parties, each in its own context, contributing to the key it was sent
    g.generate_parameters_from_srs(m, srs)
    pk = g.export_proving_key()
    p2_recs = []
    for k, x in enumerate(XS):
        party = Groth16(curve, 0)
        try:
            pk = party.contribute_key(pk, x, validate=True)
        finally:
            party.close()
        p2_recs.append(_record(g, x, pk.delta_g1, 0x71 + k, 0x81 + k))
    key_pairs = g.key_verification_pairs(pk, srs, RHO)
    p2_pairs = g.contribution_chain_pairs(srs.tau_g1[0], pk.delta_g1, p2_recs)
    t1, a1, b1 = (prod(r, TAU, *[s[0] for s in PHASE1]), prod(r, ALPHA, *[s[1] for s in PHASE1]),
                  prod(r, BETA, *[s[2] for s in PHASE1]))
    if curve in PAIRING:
        assert _holds(g, srs_pairs) == set()
        assert all(_holds(g, p) == set() for p in p1_pairs)
        assert _holds(g, key_pairs) == set()
        assert _holds(g, p2_pairs) == set()
    else:   # in the exponent: the outputs are the closed-form points of honest chains, and the key is the product's setup
        for j, x0 in enumerate((TAU, ALPHA, BETA)):
            end, recs = chain(x0, [s[j] for s in PHASE1], r)
            for k, c in enumerate(recs):   # the same s and r as _record
                c.update(s_g1=0x51 + 3 * k + j, s_x_g1=(0x51 + 3 * k + j) * PHASE1[k][j], r_g2=0x61 + 5 * k + j,
                         r_x_g2=(0x61 + 5 * k + j) * PHASE1[k][j])
            _, p, q = verdict(x0, end, recs, r)
            assert failing(p, q, r) == set()
            assert (np.array_equal(p1_pairs[j].g1, closed(g, p, q)[0]) and np.array_equal(p1_pairs[j].g2, closed(g, p, q)[1]))
        end, recs = chain(1, XS, r)
        for k, c in enumerate(recs):
            c.update(s_g1=0x71 + k, s_x_g1=(0x71 + k) * XS[k], r_g2=0x81 + k, r_x_g2=(0x81 + k) * XS[k])
        _, p, q = verdict(1, end, recs, r)
        assert failing(p, q, r) == set()
        pp, qq = closed(g, p, q)
        assert np.array_equal(p2_pairs.g1, pp) and np.array_equal(p2_pairs.g2, qq)
    # the final key is the setup of the product secrets, with gamma = 1 as g16_setup_from_srs leaves it
    want = g.generate_parameters_with_qap(m, a1, b1, 1, prod(r, *XS), t1, *gens(curve))
    assert_same_key(pk, want)
    # a tampered record fails exactly its equation
    bad = list(p2_recs)
    bad[1] = ContributionRecord(bad[1].after_g1, bad[1].s_g1, _point(g, 12345), bad[1].r_g2, bad[1].r_x_g2)
    tp = g.contribution_chain_pairs(srs.tau_g1[0], pk.delta_g1, bad)
    if curve in PAIRING:
        assert _holds(g, tp) == {2}
    else:
        diff = {k for k in range(len(tp)) if not all(np.array_equal(x, y) for x, y in zip(tp.equation(k), p2_pairs.equation(k)))}
        assert diff == {2}
    # proofs under the final key verify, and a wrong input is rejected
    if cs is not None:
        g.load_matrices(m)
        g.load_proving_key(pk)
        cd = g.codec
        z = np.ascontiguousarray(cd.fr.enc(cs.assignment))
        pf = g.create_proof_with_reduction_and_matrices(None, rng.fr(pc.r), rng.fr(pc.r), None, cs.num_instance,
                                                        cs.num_constraints, z)
        vk = pk_from_abi(curve, pk).vk
        pub = cd.fr.dec(z)[1:cs.num_instance]
        assert P.verify_proof(vk, pc, proof_from_abi(curve, pf), pub)
        assert not P.verify_proof(vk, pc, proof_from_abi(curve, pf), [(pub[0] + 1) % pc.r] + pub[1:])
