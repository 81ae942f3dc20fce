"""GPU tier of g16_setup_from_srs / g16_setup_contribute / g16_srs_from_secrets: a key derived from a powers-of-tau
transcript, after delta contributions, must equal g16_setup(alpha, beta, 1, prod delta, tau, g1, g2) in every limb of
g16_pk_export and every byte of g16_pk_export_serialized; proofs under it must equal the matching g16_setup key's."""
import numpy as np
import pytest

import pyref as P
from groth16_b200 import ConstraintMatrices, Groth16, _lib
from groth16_b200.params import GENERATORS
from groth16_b200.serialize import DeserializeError
from groth16_b200.workload import synthetic_r1cs
from util import matrices_from_r1cs, proof_from_abi

pytestmark = pytest.mark.gpu

CURVES4 = ["bls12_381", "bn254", "bls12_377", "bw6_761"]
TAU, ALPHA, BETA = 0x1234567890ABCDEF1234567, 0x2222222222222222222223, 0x3333333333333333333335
D1, D2 = 0x4444444444444444444447, 0x5555555555555555555559
KEY_MEMBERS = ("a_query", "b_g1_query", "b_g2_query", "h_query", "l_query", "beta_g1", "delta_g1")
VK_MEMBERS = ("alpha_g1", "beta_g2", "gamma_g2", "delta_g2", "gamma_abc_g1")

_ENG = {}


def engine(curve, qap) -> Groth16:
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


def transcript(g, n, extra=0):
    return g.srs_from_secrets(2 * n - 1 + extra, n + extra, TAU, ALPHA, BETA, *gens(g.curve.name))


def assert_same_key(g, k1, k2, b1, b2):
    for name in KEY_MEMBERS:
        assert np.array_equal(getattr(k1, name), getattr(k2, name)), name
    for name in VK_MEMBERS:
        assert np.array_equal(getattr(k1.vk, name), getattr(k2.vk, name)), "vk." + name
    assert b1 == b2


def setup_key(g, m, delta):
    k = g.generate_parameters_with_qap(m, ALPHA, BETA, 1, delta, TAU, *gens(g.curve.name))
    return k, g.export_proving_key_bytes(compress=False)


def srs_key(g, m, srs, deltas=(), validate=False):
    k = g.generate_parameters_from_srs(m, srs, validate=validate)
    for d in deltas:
        k = g.contribute_delta(d)
    return k, g.export_proving_key_bytes(compress=False)


def n_of(m):
    need = m.num_constraints + m.num_instance_variables
    return 1 << max(need - 1, 0).bit_length()


@pytest.mark.parametrize("qap", ["libsnark", "circom"])
@pytest.mark.parametrize("log_n", [4, 9, 14])
@pytest.mark.parametrize("curve", CURVES4)
def test_srs_key_equals_setup(curve, qap, log_n):
    g = engine(curve, qap)
    m, _, _ = synthetic_r1cs(curve, log_n, seed=300 + log_n)
    srs = transcript(g, n_of(m))
    got = srs_key(g, m, srs, [D1])
    want = setup_key(g, m, D1)
    assert_same_key(g, *got[:1], *want[:1], got[1], want[1])
    if log_n == 4:   # no contribution: delta = 1; two contributions: their product; a contribution on a g16_setup key
        assert_same_key(g, *srs_key(g, m, srs)[:1], *setup_key(g, m, 1)[:1], srs_key(g, m, srs)[1], setup_key(g, m, 1)[1])
        a, ab = srs_key(g, m, srs, [D1, D2]), setup_key(g, m, D1 * D2 % g.curve.r)
        assert_same_key(g, a[0], ab[0], a[1], ab[1])
        setup_key(g, m, D1)
        k = g.contribute_delta(D2)
        assert_same_key(g, k, ab[0], g.export_proving_key_bytes(compress=False), ab[1])


@pytest.mark.parametrize("qap", ["libsnark", "circom"])
@pytest.mark.parametrize("curve", CURVES4)
def test_longer_transcript_same_key(curve, qap):
    g = engine(curve, qap)
    m, _, _ = synthetic_r1cs(curve, 6, seed=310)
    n = n_of(m)
    a = srs_key(g, m, transcript(g, n), [D1])
    b = srs_key(g, m, transcript(g, n, extra=3 * n), [D1])   # 2^(L+2)-sized members
    assert_same_key(g, a[0], b[0], a[1], b[1])


def _stress_matrices(curve):
    """num_inputs = 4; variable 5 used by every row of B and C; variable 9 used nowhere; row 0 of A has 1100 terms"""
    ni, nw, nc = 4, 1200, 40
    rng = np.random.default_rng(5)
    rows_a, rows_b, rows_c = [], [], []
    nv = ni + nw
    for i in range(nc):
        used = [v for v in range(nv) if v != 9]
        ra = [(int(rng.integers(1, 1 << 60)), int(v)) for v in rng.choice(used, 3, replace=False)]
        if i == 0:
            ra = [(int(rng.integers(1, 1 << 60)), v) for v in used[:1100]]
        rows_a.append(ra)
        rows_b.append([(1, 5), (int(rng.integers(1, 1 << 60)), int(rng.choice(used)))])
        rows_c.append([(int(rng.integers(2, 1 << 60)), 5), (1, 0)])
    return ConstraintMatrices.from_rows(curve, ni, nw, rows_a, rows_b, rows_c)


@pytest.mark.parametrize("qap", ["libsnark", "circom"])
@pytest.mark.parametrize("curve", CURVES4)
def test_sparse_sum_stress(curve, qap):
    g = engine(curve, qap)
    m = _stress_matrices(curve)
    got = srs_key(g, m, transcript(g, n_of(m)), [D1])
    want = setup_key(g, m, D1)
    assert_same_key(g, got[0], want[0], got[1], want[1])
    assert not got[0].a_query[9].any() and not got[0].b_g2_query[9].any()   # unused variable: the identity


@pytest.mark.parametrize("curve", ["bls12_381", "bn254"])
def test_2p20_equals_setup(curve):
    g = engine(curve, "libsnark")
    m, _, _ = synthetic_r1cs(curve, 20, seed=320)
    srs = transcript(g, n_of(m))
    got = srs_key(g, m, srs, [D1])
    want = setup_key(g, m, D1)
    assert_same_key(g, got[0], want[0], got[1], want[1])


@pytest.mark.parametrize("curve", ["bls12_381", "bn254", "bls12_377"])
def test_proofs_under_derived_key(curve):
    c = P.CURVES[curve]
    rng = P.Rng(11)
    a, b = rng.fr(c.r), rng.fr(c.r)
    cs = P.mimc_circuit(c, a, b, [rng.fr(c.r) for _ in range(4)]) if hasattr(P, "mimc_circuit") else P.silly_circuit(c, a, b)
    m = matrices_from_r1cs(cs)
    g = engine(curve, "libsnark")
    cd = g.codec
    z = np.ascontiguousarray(cd.fr.enc(cs.assignment))
    pk = srs_key(g, m, transcript(g, n_of(m)), [D1])[0]
    r_, s_ = rng.fr(c.r), rng.fr(c.r)

    def prove():
        return g.create_proof_with_reduction_and_matrices(None, r_, s_, None, cs.num_instance, cs.num_constraints, z)

    pf = prove()
    vk = P.VerifyingKey(cd.dec_g1(pk.vk.alpha_g1)[0], cd.dec_g2(pk.vk.beta_g2)[0], cd.dec_g2(pk.vk.gamma_g2)[0],
                        cd.dec_g2(pk.vk.delta_g2)[0], cd.dec_g1(pk.vk.gamma_abc_g1))
    pub = cd.fr.dec(z)[1:cs.num_instance]
    assert P.verify_proof(vk, c, proof_from_abi(curve, pf), pub)
    assert not P.verify_proof(vk, c, proof_from_abi(curve, pf), [(pub[0] + 1) % c.r] + pub[1:])
    # single, pipelined (both slots in flight) and batch proofs: bit-identical to those under the matching g16_setup key
    flat = lambda p: np.concatenate([p.a, p.b, p.c])
    rl, sl = np.ascontiguousarray(cd.fr.enc1(r_)), np.ascontiguousarray(cd.fr.enc1(s_))

    def pipelined():
        outs = [np.zeros_like(flat(pf)) for _ in range(2)]
        for slot in (0, 1):
            g.prove_submit_raw(slot, rl, sl, z.ctypes.data, 0)
        for slot in (0, 1):
            g.prove_wait_raw(slot, outs[slot])
        return outs

    def batch():
        return [flat(p) for p in g.create_proofs_batch([r_, r_], [s_, s_], np.ascontiguousarray(np.stack([z, z])))]

    under_srs = [flat(pf)] + pipelined() + batch()
    setup_key(g, m, D1)
    under_setup = [flat(prove())] + pipelined() + batch()
    assert len(under_srs) == len(under_setup) == 5
    for x, y in zip(under_srs, under_setup):
        assert np.array_equal(x, y)
        assert np.array_equal(x, flat(pf))


@pytest.mark.parametrize("curve", ["bls12_381", "bn254", "bls12_377"])
def test_srs_from_secrets_sampled(curve):
    g = engine(curve, "libsnark")
    cx = P.ctx(P.CURVES[curve])
    r = P.CURVES[curve].r
    g1, g2 = gens(curve)
    srs = g.srs_from_secrets(9, 5, TAU, ALPHA, BETA, g1, g2)
    cd = g.codec
    for i in (0, 1, 8):
        assert cd.dec_g1(srs.tau_g1[i])[0] == cx.G1.mul(g1, pow(TAU, i, r))
    for i in (0, 4):
        assert cd.dec_g2(srs.tau_g2[i])[0] == cx.G2.mul(g2, pow(TAU, i, r))
        assert cd.dec_g1(srs.alpha_tau_g1[i])[0] == cx.G1.mul(g1, ALPHA * pow(TAU, i, r) % r)
        assert cd.dec_g1(srs.beta_tau_g1[i])[0] == cx.G1.mul(g1, BETA * pow(TAU, i, r) % r)
    assert cd.dec_g2(srs.beta_g2)[0] == cx.G2.mul(g2, BETA)


def test_srs_from_secrets_bw6_sampled():
    import bw6_ref as B
    g = engine("bw6_761", "libsnark")
    r = g.curve.r
    g1, g2 = gens("bw6_761")
    srs = g.srs_from_secrets(5, 3, TAU, ALPHA, BETA, g1, g2)
    cd = g.codec
    assert cd.dec_g1(srs.tau_g1[4])[0] == B.mul(pow(TAU, 4, r), g1)
    assert cd.dec_g2(srs.tau_g2[2])[0] == B.mul(pow(TAU, 2, r), g2)
    assert cd.dec_g1(srs.alpha_tau_g1[1])[0] == B.mul(ALPHA * TAU % r, g1)


def _resident_proof(g, m, z):
    return g.create_proof_with_reduction_and_matrices(None, 5, 7, None, m.num_instance_variables, m.num_constraints, z)


@pytest.mark.parametrize("curve", ["bls12_381", "bw6_761"])
def test_rejections(curve):
    g = engine(curve, "libsnark")
    m, z, _ = synthetic_r1cs(curve, 5, seed=330)
    n = n_of(m)
    srs = transcript(g, n)
    setup_key(g, m, D1)
    before = _resident_proof(g, m, z)
    lib, ctx = g._lib, g._ctx

    def still_resident():
        p = _resident_proof(g, m, z)
        assert all(np.array_equal(getattr(p, k), getattr(before, k)) for k in "abc")

    short = dict(tau_g1=2 * n - 2, tau_g2=n - 1, alpha_tau_g1=n - 1, beta_tau_g1=n - 1)
    for member, ln in short.items():
        bad = type(srs)(**{k: (getattr(srs, k)[:ln] if k == member else getattr(srs, k)) for k in
                           ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1", "beta_g2")})
        with pytest.raises(ValueError, match=member):
            g.generate_parameters_from_srs(None, bad)
        still_resident()
    bad = type(srs)(srs.tau_g1, srs.tau_g2, srs.alpha_tau_g1, srs.beta_tau_g1, None)
    with pytest.raises(ValueError, match="null"):
        g.generate_parameters_from_srs(None, bad)
    d = _lib.SrsDesc()
    assert lib.g16_setup_from_srs(ctx, None, 0) == _lib.ERR_BAD_ARGUMENT
    assert lib.g16_setup_from_srs(ctx, C_byref(d), 4) == _lib.ERR_BAD_ARGUMENT
    still_resident()
    # a proof in flight
    r_ = np.ascontiguousarray(g.codec.fr.enc1(5)); s_ = np.ascontiguousarray(g.codec.fr.enc1(7))
    g.prove_submit_raw(0, r_, s_, z.ctypes.data, 0)
    with pytest.raises(ValueError, match="in flight"):
        g.generate_parameters_from_srs(None, srs)
    with pytest.raises(ValueError, match="in flight"):
        g.contribute_delta(D2)
    out = np.zeros_like(np.concatenate([before.a, before.b, before.c]))
    g.prove_wait_raw(0, out)
    still_resident()
    # contribute: delta = 0; a g16_pk_load key (world 1 and world 2: only g16_pk_load makes world > 1 keys, so both stop at
    # the same check, and the world test of g16_setup_contribute cannot be reached from the ABI today); no key
    with pytest.raises(ValueError, match="invertible"):
        g.contribute_delta(0)
    still_resident()
    pk = g.export_proving_key()
    g.load_proving_key(pk)
    with pytest.raises(ValueError, match="g16_setup"):
        g.contribute_delta(D2)
    g.load_proving_key(pk, rank=0, world=2)
    with pytest.raises(ValueError, match="g16_setup"):
        g.contribute_delta(D2)
    # off-curve points in each member: named, and no key afterwards
    for member, idx in (("tau_g1", 2 * n - 2), ("tau_g2", 3), ("alpha_tau_g1", 17), ("beta_tau_g1", 0), ("beta_g2", 0)):
        fields = {k: getattr(srs, k).copy() for k in ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1", "beta_g2")}
        arr = fields[member]
        (arr if arr.ndim == 1 else arr[idx])[-1] ^= 1   # y's top limb: off the curve, still below q
        with pytest.raises(DeserializeError, match=rf"{member}\[{idx}\]: point is not on the curve"):
            g.generate_parameters_from_srs(None, type(srs)(**fields))
        with pytest.raises(ValueError, match="no proving key|needs a resident key"):
            g.contribute_delta(D2)
    # no circuit
    g2 = Groth16(curve, 0)
    try:
        with pytest.raises(ValueError, match="circuit"):
            g2.generate_parameters_from_srs(None, srs)
        with pytest.raises(ValueError):
            g2.contribute_delta(D2)
    finally:
        g2.close()


def C_byref(x):
    import ctypes
    return ctypes.byref(x)


@pytest.mark.parametrize("curve", ["bls12_381", "bn254", "bls12_377"])
def test_torsion_point_needs_validate(curve):
    """a point of small order on the curve: refused with G16_SER_VALIDATE, accepted without it"""
    g = engine(curve, "libsnark")
    m, _, _ = synthetic_r1cs(curve, 4, seed=340)
    n = n_of(m)
    srs = transcript(g, n)
    c = P.CURVES[curve]
    cx = P.ctx(c)
    # a G2 point off the prime-order subgroup: any x with a curve point, without cofactor clearing
    Gp = cx.G2
    F = Gp.F
    x = F.from_int(1)
    while True:
        rhs = F.add(F.mul(F.mul(x, x), x), Gp.b)
        y = F.sqrt(rhs)
        if y is not None:
            break
        x = F.add(x, F.from_int(1))
    T = (x, y)
    assert Gp.mul(T, c.r) is not None
    tg2 = srs.tau_g2.copy()
    tg2[2] = g.codec.enc_g2([T])[0]
    bad = type(srs)(srs.tau_g1, tg2, srs.alpha_tau_g1, srs.beta_tau_g1, srs.beta_g2)
    with pytest.raises(DeserializeError, match=r"tau_g2\[2\]: point is not in the prime-order subgroup"):
        g.generate_parameters_from_srs(m, bad, validate=True)
    g.generate_parameters_from_srs(m, bad, validate=False)
