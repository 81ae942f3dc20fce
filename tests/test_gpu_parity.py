"""GPU parity tests (run on an H100 with `pytest -m gpu`): every C-ABI entry point against the CPU oracle.

Bar: bit-exact (integer arithmetic throughout).  Reference behaviour cited per test."""
import numpy as np
import pytest

import pyref as P
from groth16_b200 import CurveCodec, Groth16, PolynomialDegreeTooLarge, get_curve
from util import ALL_CURVES, matrices_from_r1cs, pk_from_abi, pk_to_abi, proof_from_abi, toxic

pytestmark = pytest.mark.gpu

_ENGINES = {}


def engine(name) -> Groth16:
    if name not in _ENGINES:
        _ENGINES[name] = Groth16(name, 0)
    return _ENGINES[name]


@pytest.mark.parametrize("curve", ALL_CURVES)
@pytest.mark.parametrize("log_n", [0, 1, 3, 6, 10, 11, 13])
def test_ntt_matches_oracle(curve, log_n):
    """ark-poly fft/ifft/coset (r1cs_to_qap.rs:201-207,232): natural order in/out, omega = two_adic_root^(2^(s-log n))."""
    c = P.CURVES[curve]
    g = engine(curve)
    cd = g.codec
    rng = P.Rng(100 + log_n)
    n = 1 << log_n
    vals = [rng.fr(c.r) for _ in range(n)]
    dom = P.Domain(c, n)
    enc = cd.fr.enc(vals)
    assert cd.fr.dec(g.ntt_log(log_n, enc)) == dom.fft(vals)
    assert cd.fr.dec(g.ntt_log(log_n, enc, inverse=True)) == dom.ifft(vals)
    assert cd.fr.dec(g.ntt_log(log_n, enc, coset=True)) == dom.fft(vals, offset=c.fr_gen)
    assert cd.fr.dec(g.ntt_log(log_n, enc, inverse=True, coset=True)) == dom.ifft(vals, offset=c.fr_gen)


def test_ntt_degree_too_large():
    """D::new(..) -> None -> PolynomialDegreeTooLarge (r1cs_to_qap.rs:178-179): BN254 two-adicity is 28."""
    g = engine("bn254")
    with pytest.raises(PolynomialDegreeTooLarge):
        g.ntt_log(29, np.zeros((1, 4), dtype=np.uint64))


@pytest.mark.parametrize("curve", ALL_CURVES)
@pytest.mark.parametrize("log_n", [3, 11])
def test_witness_map_evals(curve, log_n):
    """r1cs_to_qap.rs:201-234 on arbitrary evaluation vectors."""
    c = P.CURVES[curve]
    g = engine(curve)
    cd = g.codec
    rng = P.Rng(7 + log_n)
    n = 1 << log_n
    a, b, cc = ([rng.fr(c.r) for _ in range(n)] for _ in range(3))
    dom = P.Domain(c, n)
    want = P.witness_map_from_evals(dom, a, b, cc)
    got = cd.fr.dec(g.witness_map_from_evals(cd.fr.enc(a), cd.fr.enc(b), cd.fr.enc(cc)))
    assert got == want


def _edge_scalars(c, rng, n):
    sc = [rng.fr(c.r) for _ in range(n)]
    special = [0, 1, 2, c.r - 1, c.r - 2, (1 << 128), (1 << 16) - 1, 1 << 15, (1 << 15) + 1]
    for i, v in enumerate(special):
        if i < n:
            sc[i] = v % c.r
    return sc


@pytest.mark.parametrize("curve", ALL_CURVES)
@pytest.mark.parametrize("n", [0, 1, 2, 17, 300])
def test_msm_g1(curve, n):
    """VariableBaseMSM::msm_bigint (prover.rs:66,74,262) vs double-and-add; zero/one/r-1 scalars, identity bases,
    repeated bases (P+P) and inverse pairs (P-P)."""
    c = P.CURVES[curve]
    cx = P.ctx(c)
    g = engine(curve)
    cd = g.codec
    rng = P.Rng(31 + n)
    gen = cx.g1_gen()
    bases = [cx.G1.mul(gen, rng.fr(c.r)) for _ in range(n)]
    if n >= 17:
        bases[3] = None
        bases[5] = bases[4]
        bases[7] = cx.G1.neg(bases[6])
    sc = _edge_scalars(c, rng, n)
    if n >= 17:
        sc[5] = sc[4]
        sc[7] = sc[6]
    want = cx.G1.msm_naive(bases, sc)
    got = cd.dec_proj_g1(g.msm_g1(cd.enc_g1(bases) if n else np.zeros((0, 2 * g.nq), dtype=np.uint64),
                                  cd.fr.bigint(sc) if n else np.zeros((0, 4), dtype=np.uint64)))
    assert got == want


@pytest.mark.parametrize("curve", ALL_CURVES)
@pytest.mark.parametrize("n", [1, 40])
def test_msm_g2(curve, n):
    c = P.CURVES[curve]
    cx = P.ctx(c)
    g = engine(curve)
    cd = g.codec
    rng = P.Rng(77 + n)
    gen = cx.g2_gen()
    bases = [cx.G2.mul(gen, rng.fr(c.r)) for _ in range(n)]
    sc = _edge_scalars(c, rng, n)
    if n >= 17:
        bases[3] = None
        bases[5] = bases[4]
        sc[5] = sc[4]
    want = cx.G2.msm_naive(bases, sc)
    got = cd.dec_proj_g2(g.msm_g2(cd.enc_g2(bases), cd.fr.bigint(sc)))
    assert got == want


def test_msm_truncates_like_ark():
    """msm_bigint uses min(bases.len(), scalars.len()) (SURVEY.md section 2a; relied upon at prover.rs:66)."""
    c = P.CURVES["bn254"]
    cx = P.ctx(c)
    g = engine("bn254")
    cd = g.codec
    rng = P.Rng(5)
    bases = [cx.G1.mul(cx.g1_gen(), rng.fr(c.r)) for _ in range(7)]
    sc = [rng.fr(c.r) for _ in range(8)]
    assert cd.dec_proj_g1(g.msm_g1(cd.enc_g1(bases), cd.fr.bigint(sc))) == cx.G1.msm_naive(bases, sc[:7])


@pytest.mark.parametrize("curve", ALL_CURVES)
def test_setup_matches_oracle(curve):
    """generate_parameters_with_qap (generator.rs:47-208): every query of the GPU-built key equals the oracle's."""
    c = P.CURVES[curve]
    cx = P.ctx(c)
    g = engine(curve)
    rng = P.Rng(11)
    cs = P.silly_circuit(c, rng.fr(c.r), rng.fr(c.r))
    tw = toxic(c, 21)
    want = pk_to_abi(P.generate_parameters(cs, *tw))
    got = g.generate_parameters_with_qap(matrices_from_r1cs(cs), *tw, cx.g1_gen(), cx.g2_gen())
    for f in ("a_query", "b_g1_query", "b_g2_query", "h_query", "l_query", "beta_g1", "delta_g1"):
        assert np.array_equal(np.asarray(getattr(got, f)).ravel(), np.asarray(getattr(want, f)).ravel()), f
    for f in ("alpha_g1", "beta_g2", "gamma_g2", "delta_g2", "gamma_abc_g1"):
        assert np.array_equal(np.asarray(getattr(got.vk, f)).ravel(), np.asarray(getattr(want.vk, f)).ravel()), f


@pytest.mark.parametrize("curve", ALL_CURVES)
def test_prove_silly_circuit(curve):
    """src/test.rs:45-73 test_prove_and_verify: setup -> prove -> verify true for c = a*b, false for a wrong input;
    plus bit-exact equality with the oracle's prover on the same (pk, witness, r, s), r = 0 path included."""
    c = P.CURVES[curve]
    g = engine(curve)
    cd = g.codec
    rng = P.Rng(3)
    tw = toxic(c, 22)
    for it in range(3):
        a, b = rng.fr(c.r), rng.fr(c.r)
        cs = P.silly_circuit(c, a, b)
        opk = P.generate_parameters(cs, *tw)
        m = matrices_from_r1cs(cs)
        g.load_matrices(m)
        g.load_proving_key(pk_to_abi(opk))
        r_, s_ = (0, rng.fr(c.r)) if it == 2 else (rng.fr(c.r), rng.fr(c.r))
        pf = proof_from_abi(curve, g.create_proof_with_reduction_and_matrices(
            None, r_, s_, None, cs.num_instance, cs.num_constraints, cd.fr.enc(cs.assignment)))
        want = P.create_proof(opk, cs, r_, s_)
        assert (pf.a, pf.b, pf.c) == (want.a, want.b, want.c)
        if it == 0:
            assert P.verify_proof(opk.vk, c, pf, [a * b % c.r])
            assert not P.verify_proof(opk.vk, c, pf, [a])


@pytest.mark.parametrize("curve", ["bls12_377", "bls12_381"])
def test_prove_mimc(curve):
    """tests/mimc.rs:145-229 (BLS12-377 is the reference's curve for this test; BASELINE config 1 names BLS12-381):
    key built by the GPU setup, proof checked against the closed form in the exponent and by the pairing verifier."""
    c = P.CURVES[curve]
    cx = P.ctx(c)
    g = engine(curve)
    cd = g.codec
    rng = P.Rng(9)
    constants = [rng.fr(c.r) for _ in range(P.MIMC_ROUNDS)]
    xl, xr = rng.fr(c.r), rng.fr(c.r)
    cs = P.mimc_circuit(c, xl, xr, constants)
    assert cs.is_satisfied() and cs.num_constraints == 644 and cs.assignment[1] == P.mimc_hash(c, xl, xr, constants)
    tw = toxic(c, 23)
    m = matrices_from_r1cs(cs)
    pk_abi = g.generate_parameters_with_qap(m, *tw, cx.g1_gen(), cx.g2_gen())
    exps = P.generate_parameters(cs, *tw, scalars_only=True)
    opk = pk_from_abi(curve, pk_abi, toxic=dict(exps, g1=cx.g1_gen(), g2=cx.g2_gen()))
    r_, s_ = rng.fr(c.r), rng.fr(c.r)
    z = cd.fr.enc(cs.assignment)
    # witness map alone (r1cs_to_qap.rs:172-235)
    h = cd.fr.dec(g.witness_map_from_matrices(None, cs.num_instance, cs.num_constraints, z))
    assert h == P.witness_map(cs)
    pf = proof_from_abi(curve, g.create_proof_with_reduction_and_matrices(None, r_, s_, None, cs.num_instance,
                                                                          cs.num_constraints, z))
    want = P.proof_in_the_exponent(opk, cs, r_, s_, h=h)
    assert (pf.a, pf.b, pf.c) == (want.a, want.b, want.c)
    assert P.verify_proof(opk.vk, c, pf, [cs.assignment[1]])
    assert not P.verify_proof(opk.vk, c, pf, [xl])


def test_sharded_prove_equals_single():
    """SURVEY.md section 8e: dealing every query round-robin over `world` ranks and summing the partial points gives
    the same proof bit for bit (here: 3 ranks emulated sequentially on one GPU)."""
    curve = "bn254"
    c = P.CURVES[curve]
    cx = P.ctx(c)
    g = engine(curve)
    cd = g.codec
    cs = P.synthetic_circuit(c, 50, seed=4, num_inputs=2)
    assert cs.is_satisfied()
    tw = toxic(c, 24)
    m = matrices_from_r1cs(cs)
    pk_abi = g.generate_parameters_with_qap(m, *tw, cx.g1_gen(), cx.g2_gen())
    rng = P.Rng(12)
    r_, s_ = rng.fr(c.r), rng.fr(c.r)
    z = np.ascontiguousarray(cd.fr.enc(cs.assignment))
    single = g.create_proof_with_reduction_and_matrices(None, r_, s_, None, cs.num_instance, cs.num_constraints, z)
    world = 3
    parts = []
    rl = np.ascontiguousarray(cd.fr.enc1(r_))
    for rank in range(world):
        g.load_proving_key(pk_abi, rank, world)
        out = np.zeros(g.partial_limbs(), dtype=np.uint64)
        g.prove_partial_raw(rl, z.ctypes.data, 0, out)
        parts.append(out)
    sharded = g.prove_assemble(r_, s_, np.stack(parts))
    assert np.array_equal(single.a, sharded.a) and np.array_equal(single.b, sharded.b) and np.array_equal(single.c, sharded.c)
    exps = P.generate_parameters(cs, *tw, scalars_only=True)
    opk = pk_from_abi(curve, pk_abi, toxic=dict(exps, g1=cx.g1_gen(), g2=cx.g2_gen()))
    want = P.proof_in_the_exponent(opk, cs, r_, s_)
    pf = proof_from_abi(curve, sharded)
    assert (pf.a, pf.b, pf.c) == (want.a, want.b, want.c)


def _oracle_vs_gpu(curve, m, z, flags=0):
    """full prove through the C ABI vs the C++ CPU oracle on the same (pk, matrices, assignment, r, s)"""
    import orc
    from groth16_b200.params import GENERATORS
    c = P.CURVES[curve]
    g = engine(curve)
    cd = g.codec
    G = GENERATORS[curve]
    pk = g.generate_parameters_with_qap(m, 11, 22, 33, 44, 55, G["g1"], G["g2"])
    r, s = cd.fr.enc1(123456789), cd.fr.enc1(987654321)
    got = g.create_proof_with_reduction_and_matrices(None, r, s, None, m.num_instance_variables, m.num_constraints, z, flags=flags)
    want, _ = orc.prove(c.cid, cd.nq, pk, m, z, r, s, threads=8)
    nq = cd.nq
    assert np.array_equal(got.a, want[:2 * nq]) and np.array_equal(got.b, want[2 * nq:6 * nq]) and np.array_equal(got.c, want[6 * nq:])
    return pk, got


@pytest.mark.parametrize("curve", ALL_CURVES)
def test_prove_dummy_circuit_degenerate_distribution(curve):
    """benches/bench.rs:41-64 DummyCircuit: every witness scalar equal (each MSM window hits ONE bucket: maximal skew),
    a/b queries almost all identity.  2^12 - 100 constraints; proof bit-exact with the CPU oracle and pairing-verified."""
    from groth16_b200.workload import dummy_r1cs
    m, z, pub = dummy_r1cs(curve, (1 << 12) - 100, (1 << 12) - 100)
    pk_abi, got = _oracle_vs_gpu(curve, m, z)
    opk = pk_from_abi(curve, pk_abi)
    assert P.verify_proof(opk.vk, P.CURVES[curve], proof_from_abi(curve, got), pub)


@pytest.mark.parametrize("curve", ALL_CURVES)
def test_prove_synthetic_2p14(curve):
    """Non-degenerate synthetic R1CS at 2^14 (multi-pass NTT, precomputed-multiple MSM path) vs the CPU oracle, concurrent
    and serialised stream schedules; witness map alone vs the oracle as well."""
    import orc
    from groth16_b200 import _lib
    from groth16_b200.workload import synthetic_r1cs
    m, z, pub = synthetic_r1cs(curve, 14, seed=5)
    _oracle_vs_gpu(curve, m, z)
    _oracle_vs_gpu(curve, m, z, flags=_lib.SERIAL_MSMS)
    g = engine(curve)
    h = g.witness_map_from_matrices(None, m.num_instance_variables, m.num_constraints, z)
    assert np.array_equal(h, orc.witness_map(P.CURVES[curve].cid, m, z, threads=8))


def _skewed_msm_check():
    import orc
    curve = "bls12_381"
    c = P.CURVES[curve]
    g = engine(curve)
    cd = g.codec
    n = 1 << 15
    rs = np.random.RandomState(3)
    from groth16_b200.params import GENERATORS
    ks = rs.randint(0, 1 << 62, size=(n, 4), dtype=np.int64).astype(np.uint64)
    ks[:, 3] &= np.uint64((1 << 58) - 1)
    bases = orc.batch_mul_g1(c.cid, cd.nq, cd.enc_g1([GENERATORS[curve]["g1"]])[0], ks, threads=8)
    bases[5::97] = bases[4::97][:len(bases[5::97])]   # repeated bases: equal points meet inside a bucket
    sc = rs.randint(0, 1 << 62, size=(n, 4), dtype=np.int64).astype(np.uint64)
    sc[:, 3] &= np.uint64((1 << 58) - 1)
    kind = rs.randint(0, 4, size=n)
    sc[kind <= 1] = 0
    sc[kind <= 1, 0] = rs.randint(0, 2, size=int((kind <= 1).sum())).astype(np.uint64)
    sc[kind == 2, 1:] = 0
    sc[kind == 2, 0] &= np.uint64(0xFFFFFFFF)
    assert np.array_equal(g.msm_g1(bases, sc), orc.msm_g1(c.cid, cd.nq, bases, sc, threads=8))


def test_msm_skewed_scalars_large():
    """2^15-point G1 MSM whose scalars are 50 % in {0,1}, 25 % < 2^32, 25 % uniform (SURVEY.md section 8d 'realistic mix'),
    some bases repeated: giant buckets exercise every level of the segmented reduction.  Checked against the CPU oracle."""
    _skewed_msm_check()


LEAN_DEFAULT = (0, 0)   # Engine::Tune::ba_occ_g1 / ba_occ_g2


def _set_ba(rounds_g1, rounds_g2, min_entries=0, **kw):
    for name in ALL_CURVES:
        g = engine(name)
        g.set_option("msm_ba", rounds_g1)
        g.set_option("msm_ba_g2", rounds_g2)
        g.set_option("ba_min_entries_g1", min_entries if min_entries else 1 << 18)      # the test MSMs are small: force the rounds on
        g.set_option("ba_min_entries_g2", min_entries if min_entries else 1 << 18)
        g.set_option("ba_adaptive", 0)                                                    # exactly these many rounds
        for k, v in kw.items():
            g.set_option(k, v)


@pytest.mark.parametrize("rounds,m,G,gcd,lean", [(0, 16, 64, 1, 0), (1, 4, 7, 0, 0), (3, 32, 64, 1, 0), (6, 16, 16, 1, 0),
                                                 (4, 32, 16, 1, 1), (2, 5, 3, 0, 1), (3, 8, 16, 1, 2)])
def test_batched_affine_rounds(rounds, m, G, gcd, lean):
    """The batched-affine pre-reduction (csrc/msm_ba.cuh; default: 4 rounds on G1 MSMs; g16_set_option "msm_ba" /
    "msm_ba_g2") must not change a single bit whatever the number of rounds (0 = plain XYZZ accumulation), the additions
    per thread, the products per inversion, the inversion routine or the kernel build (lean = 1: the register-lean round
    kernels, "ba_occ_g1" / "ba_occ_g2"; lean = 2: capped grids pulling tiles from a counter, "ba_cap_*"): skewed G1 MSM with repeated bases, a 2^14-point G2
    MSM, and full proofs (synthetic 2^14, and the degenerate DummyCircuit where every scalar is equal) against the CPU
    oracle."""
    import orc
    from groth16_b200.params import GENERATORS
    from groth16_b200.workload import dummy_r1cs, synthetic_r1cs
    try:
        cap = 1 if lean == 2 else 0
        _set_ba(rounds, rounds, ba_m=m, ba_g=G, ba_inv_gcd=gcd, ba_occ_g1=int(lean == 1), ba_occ_g2=int(lean == 1),
                ba_cap_fwd_g1=cap, ba_cap_bwd_g1=cap, ba_cap_fwd_g2=cap, ba_cap_bwd_g2=cap)
        _ba_body(orc, GENERATORS, dummy_r1cs, synthetic_r1cs)
    finally:
        _set_ba(4, 5, ba_m=32, ba_g=16, ba_inv_gcd=1, ba_occ_g1=LEAN_DEFAULT[0], ba_occ_g2=LEAN_DEFAULT[1],
                ba_cap_fwd_g1=0, ba_cap_bwd_g1=0, ba_cap_fwd_g2=0, ba_cap_bwd_g2=0)   # the library defaults (Engine::Tune) ...
        for name in ALL_CURVES:
            engine(name).set_option("ba_min_entries_g1", 1 << 19)
            engine(name).set_option("ba_min_entries_g2", 1 << 19)
            engine(name).set_option("ba_adaptive", 1)


def _ba_body(orc, GENERATORS, dummy_r1cs, synthetic_r1cs):
    _skewed_msm_check()
    curve = "bn254"
    c = P.CURVES[curve]
    g = engine(curve)
    cd = g.codec
    n = 1 << 14
    rs = np.random.RandomState(11)
    ks = rs.randint(0, 1 << 62, size=(n, 4), dtype=np.int64).astype(np.uint64)
    ks[:, 3] &= np.uint64((1 << 58) - 1)
    bases = orc.batch_mul_g2(c.cid, cd.nq, cd.enc_g2([GENERATORS[curve]["g2"]])[0], ks, threads=8)
    sc = rs.randint(0, 1 << 62, size=(n, 4), dtype=np.int64).astype(np.uint64)
    sc[:, 3] &= np.uint64((1 << 58) - 1)
    assert np.array_equal(g.msm_g2(bases, sc), orc.msm_g2(c.cid, cd.nq, bases, sc, threads=8))
    m, z, _ = synthetic_r1cs("bls12_381", 14, seed=9)
    _oracle_vs_gpu("bls12_381", m, z)
    m, z, _ = dummy_r1cs("bls12_377", (1 << 14) - 100, (1 << 14) - 100)
    _oracle_vs_gpu("bls12_377", m, z)


@pytest.mark.parametrize("curve", ALL_CURVES)
def test_prepare_inputs(curve):
    """verifier.rs:25-39 as one G1 MSM on the GPU (see util.check_prepare_inputs)."""
    from util import check_prepare_inputs
    check_prepare_inputs(engine(curve), curve)


def test_api_error_paths():
    """Status codes instead of panics across the ABI (Cargo.toml:61 panic='abort' rationale): wrong order of calls, bad
    indices, sharded key used with the single-GPU entry point, domain larger than the field's two-adicity."""
    from groth16_b200 import ConstraintMatrices, PolynomialDegreeTooLarge
    g = Groth16("bn254", 0)
    c = P.CURVES["bn254"]
    cs = P.silly_circuit(c, 3, 5)
    m = matrices_from_r1cs(cs)
    z = g.codec.fr.enc(cs.assignment)
    with pytest.raises(ValueError):      # no circuit / key resident yet
        g.create_proof_with_reduction_and_matrices(None, 1, 2, None, 2, 6, z)
    opk = pk_to_abi(P.generate_parameters(cs, *toxic(c, 1)))
    with pytest.raises(ValueError):      # g16_pk_load before g16_circuit_load
        g.load_proving_key(opk)
    bad = ConstraintMatrices(m.num_instance_variables, m.num_witness_variables, m.num_constraints,
                             (m.a[0], m.a[1] + 100, m.a[2]), m.b, m.c)
    with pytest.raises(ValueError):      # column index out of range
        g.load_matrices(bad)
    g.load_matrices(m)
    g.load_proving_key(opk, 0, 2)        # sharded residency
    with pytest.raises(ValueError):
        g.create_proof_with_reduction_and_matrices(None, 1, 2, None, 2, 6, z)
    g.load_proving_key(opk)
    with pytest.raises(ValueError):      # wrong assignment length
        g.create_proof_with_reduction_and_matrices(None, 1, 2, None, 2, 6, z[:-1])
    pf = g.create_proof_with_reduction_and_matrices(None, 1, 2, None, 2, 6, z)
    want = P.create_proof(P.generate_parameters(cs, *toxic(c, 1)), cs, 1, 2)
    got = proof_from_abi("bn254", pf)
    assert (got.a, got.b, got.c) == (want.a, want.b, want.c)
    # a circuit whose domain would exceed 2^28 on BN254 -> PolynomialDegreeTooLarge (r1cs_to_qap.rs:178-179)
    rp = np.zeros(2, dtype=np.uint32)
    empty = (rp, np.zeros(0, dtype=np.uint32), np.zeros((0, 4), dtype=np.uint64))
    huge = ConstraintMatrices((1 << 28) + 1, 1, 1, empty, empty, empty)
    with pytest.raises(PolynomialDegreeTooLarge):
        g.load_matrices(huge)
    g.close()


def test_pipelined_proofs_equal_sequential():
    """g16_prove_submit / g16_prove_wait over the two proof slots: proofs produced while another proof is in flight are
    bit-identical to proofs produced one at a time (different (r, s) and different witnesses per proof)."""
    curve = "bls12_377"
    c = P.CURVES[curve]
    g = engine(curve)
    cd = g.codec
    from groth16_b200.params import GENERATORS
    from groth16_b200.workload import synthetic_r1cs
    m, z0, _ = synthetic_r1cs(curve, 13, seed=2)
    _, z1, _ = synthetic_r1cs(curve, 13, seed=2)   # same circuit (same seed => same matrices) ...
    G = GENERATORS[curve]
    g.generate_parameters_with_qap(m, 5, 6, 7, 8, 9, G["g1"], G["g2"], export=False)
    rng = P.Rng(8)
    jobs = []
    for i in range(5):
        r = np.ascontiguousarray(cd.fr.enc1(rng.fr(c.r)))
        s = np.ascontiguousarray(cd.fr.enc1(rng.fr(c.r)))
        jobs.append((r, s, z0 if i % 2 == 0 else z1))
    nq = g.nq
    seq = []
    for r, s, z in jobs:
        out = np.zeros(8 * nq, dtype=np.uint64)
        g.prove_raw(r, s, z.ctypes.data, 0, out)
        seq.append(out)
    outs = [np.zeros(8 * nq, dtype=np.uint64) for _ in jobs]
    g.prove_submit_raw(0, jobs[0][0], jobs[0][1], jobs[0][2].ctypes.data, 0)
    for i in range(1, len(jobs)):
        g.prove_submit_raw(i & 1, jobs[i][0], jobs[i][1], jobs[i][2].ctypes.data, 0)
        g.prove_wait_raw((i - 1) & 1, outs[i - 1])
    g.prove_wait_raw((len(jobs) - 1) & 1, outs[-1])
    for a_, b_ in zip(seq, outs):
        assert np.array_equal(a_, b_)
    with pytest.raises(ValueError):   # waiting on an idle slot is an error, not a hang
        g.prove_wait_raw(0, outs[0])


@pytest.mark.parametrize("curve", ["bn254", "bls12_381"])
def test_edge_circuits(curve):
    """Edge shapes around the witness map and the MSM entry counts, each against the big-int oracle:
    (a) no public inputs (instance = [One]); (b) num_constraints + num_instance exactly 2^k and 2^k + 1 (domain doubles);
    (c) an all-zero witness (every MSM over the witness sorts ZERO entries: empty partial lists, empty buckets);
    (d) a single constraint."""
    c = P.CURVES[curve]
    g = engine(curve)
    cd = g.codec
    rng = P.Rng(61)
    r = c.r

    def chain(n_constraints, n_inputs, zero=False):
        # x_{i+1} = (x_i + k_i) * x_i ; the last n_inputs products are public
        ninst = 1 + n_inputs
        vals = [0 if zero else rng.fr(r)]
        cols = [ninst]
        A, B, C, inst, wit = [], [], [], [], list(vals)
        for i in range(n_constraints):
            k = 0 if zero else rng.fr(r)
            v = (vals[-1] + k) * vals[-1] % r
            if i >= n_constraints - n_inputs:
                col = 1 + len(inst); inst.append(v)
            else:
                col = ninst + len(wit); wit.append(v)
            A.append([(1, cols[-1])] + ([(k, 0)] if k else [])); B.append([(1, cols[-1])]); C.append([(1, col)])
            cols.append(col); vals.append(v)
        return P.R1CS(c, ninst, len(wit), A, B, C, [1] + inst + wit)

    cases = [chain(5, 0), chain(6, 1), chain(7, 1), chain(1, 1), chain(9, 2, zero=True), chain(14, 1), chain(15, 1)]
    for cs in cases:
        assert cs.is_satisfied()
        tw = toxic(c, 70 + cs.num_constraints)
        opk = P.generate_parameters(cs, *tw)
        g.load_matrices(matrices_from_r1cs(cs))
        g.load_proving_key(pk_to_abi(opk))
        z = cd.fr.enc(cs.assignment)
        h = cd.fr.dec(g.witness_map_from_matrices(None, cs.num_instance, cs.num_constraints, z))
        assert h == P.witness_map(cs)
        r_, s_ = rng.fr(r), rng.fr(r)
        pf = proof_from_abi(curve, g.create_proof_with_reduction_and_matrices(None, r_, s_, None, cs.num_instance,
                                                                              cs.num_constraints, z))
        want = P.create_proof(opk, cs, r_, s_)
        assert (pf.a, pf.b, pf.c) == (want.a, want.b, want.c)
    assert P.verify_proof(opk.vk, c, pf, cs.assignment[1:cs.num_instance])
