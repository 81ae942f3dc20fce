"""GPU parity at the PRODUCTION kernel geometry (run on an H100 with `pytest -m gpu`).

test_gpu_parity.py stops at 2^15-pair MSMs / 2^13-point NTTs / 2^14-constraint proofs, where the MSM picks c = 11 and
the NTT plan has two passes.  What bench.py ships is different code paths: c = 16 with ONE bucket set and 16
precomputed multiples per base (from 2^16 pairs per query up), 64 sorted entries per accumulation thread, the batched-
affine rounds, and the three-pass NTT plan (log n >= 18).  These tests put exactly that under the oracle:

  * g16_ntt at log n = 18 / 20, all four modes, vs the C++ oracle's in-order radix-2 FFT (ark-poly semantics);
  * every MSM of the resident-key path at 2^17 and 2^20 pairs with uniform / 50-25-25 mix / all-equal scalars
    (prover.rs:66,74,262 call shapes) vs the oracle's Pippenger;
  * full proofs at 2^20 on BLS12-381, BN254, BLS12-377 and the reference's own DummyCircuit at 2^20 - 100
    (benches/bench.rs:17-20,41-64): bit-exact vs the oracle's prover under a key whose elements are sample-checked against
    the oracle's CPU setup (generator.rs:47-208), and pairing-verified (verifier.rs:44-65).
Bar: bit-exact."""
import numpy as np
import pytest

import orc
import pyref as P
from groth16_b200 import Groth16, _lib
from groth16_b200.params import GENERATORS
from groth16_b200.workload import dummy_r1cs, synthetic_r1cs
from util import ALL_CURVES, pk_from_abi, proof_from_abi

pytestmark = pytest.mark.gpu

TOXIC = (0x1111111111111111111111, 0x2222222222222222222223, 0x3333333333333333333335, 0x4444444444444444444447,
         0x5555555555555555555559)   # alpha, beta, gamma, delta, tau (bench.py uses the same)
THREADS = 16
_ENG = {}
_WORK = {}


def engine(name) -> Groth16:
    if name not in _ENG:
        _ENG[name] = Groth16(name, 0)
    return _ENG[name]


def workload(curve, kind, log_n):
    key = (curve, kind, log_n)
    if key not in _WORK:
        if kind == "dummy":
            k = (1 << log_n) - 100
            _WORK[key] = dummy_r1cs(curve, k, k)
        else:
            _WORK[key] = synthetic_r1cs(curve, log_n, seed=1)
    return _WORK[key]


def rand_fr_mont(rs, n):
    """n pseudo-random Fr elements as limbs (< 2^250, hence < r on all three curves; any value < r is a valid Montgomery
    image, so these are uniform-looking field elements)"""
    v = rs.randint(0, 1 << 62, size=(n, 4), dtype=np.int64).astype(np.uint64)
    v[:, 3] &= np.uint64((1 << 58) - 1)
    return np.ascontiguousarray(v)


# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve,log_n", [("bls12_381", 18), ("bls12_381", 20), ("bn254", 18), ("bls12_377", 18), ("bn254", 20)])
def test_ntt_three_pass_plan(curve, log_n):
    """ark-poly fft / ifft / coset fft / coset ifft (r1cs_to_qap.rs:201-207,220-221,232) on 2^18 and 2^20 points: the sizes
    whose plan has two strided passes + the bit-reversing pass, which no smaller test reaches."""
    g = engine(curve)
    cid = P.CURVES[curve].cid
    vals = rand_fr_mont(np.random.RandomState(1000 + log_n), 1 << log_n)
    for inverse in (False, True):
        for coset in (False, True):
            got = g.ntt_log(log_n, vals, inverse=inverse, coset=coset)
            want = orc.ntt(cid, log_n, vals, inverse=inverse, coset=coset, threads=THREADS)
            assert np.array_equal(got, want), (curve, log_n, inverse, coset)


@pytest.mark.parametrize("curve,log_n", [("bn254", 14), ("bls12_381", 15), ("bls12_377", 16), ("bn254", 17), ("bls12_381", 19),
                                         ("bn254", 21), ("bls12_381", 22)])
def test_ntt_plans(curve, log_n):
    """The plans around test_ntt_three_pass_plan's sizes: one strided pass + the bit-reversing pass (log n = 14 .. 17), two
    strided passes with uneven (19, 21) and even (22) splits; forward + coset-inverse, all four modes at 16 and 21."""
    g = engine(curve)
    cid = P.CURVES[curve].cid
    vals = rand_fr_mont(np.random.RandomState(2000 + log_n), 1 << log_n)
    modes = ((False, False), (True, True)) + (((False, True), (True, False)) if log_n in (16, 21) else ())
    for inverse, coset in modes:
        want = orc.ntt(cid, log_n, vals, inverse=inverse, coset=coset, threads=THREADS)
        assert np.array_equal(g.ntt_log(log_n, vals, inverse=inverse, coset=coset), want), (curve, log_n, inverse, coset)


def _setup(curve, m):
    g = engine(curve)
    G = GENERATORS[curve]
    pk = g.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=True)
    return g, pk


def _check_key_sample(curve, g, m, pk, samples=48):
    """The GPU-minted key against the oracle's CPU setup (generator.rs:47-208) on a random sample of every query (plus the
    first and last element): closes the loop that both provers could otherwise agree on a wrong-but-consistent key."""
    cd = g.codec
    cid, nq = cd.c.cid, cd.nq
    G = GENERATORS[curve]
    ex = orc.setup_scalars(cid, m, cd.fr.enc(list(TOXIC)), threads=THREADS)
    g1 = cd.enc_g1([G["g1"]])[0]
    g2 = cd.enc_g2([G["g2"]])[0]
    rs = np.random.RandomState(99)
    for name, exps, grp in (("a_query", ex["a"], 1), ("b_g1_query", ex["b"], 1), ("b_g2_query", ex["b"], 2),
                            ("h_query", ex["h"], 1), ("l_query", ex["l"], 1)):
        q = np.asarray(getattr(pk, name)).reshape(exps.shape[0], -1)
        idx = np.unique(np.concatenate([[0, exps.shape[0] - 1], rs.randint(0, exps.shape[0], size=samples)]))
        want = (orc.batch_mul_g1(cid, nq, g1, exps[idx], THREADS) if grp == 1 else orc.batch_mul_g2(cid, nq, g2, exps[idx], THREADS))
        assert np.array_equal(q[idx], want), name
    tx = cd.fr.enc(list(TOXIC))
    s1 = orc.batch_mul_g1(cid, nq, g1, tx[[0, 1, 3]], 1)
    s2 = orc.batch_mul_g2(cid, nq, g2, tx[[1, 2, 3]], 1)
    assert np.array_equal(pk.vk.alpha_g1, s1[0]) and np.array_equal(pk.beta_g1, s1[1]) and np.array_equal(pk.delta_g1, s1[2])
    assert np.array_equal(pk.vk.beta_g2, s2[0]) and np.array_equal(pk.vk.gamma_g2, s2[1]) and np.array_equal(pk.vk.delta_g2, s2[2])
    assert np.array_equal(np.asarray(pk.vk.gamma_abc_g1).reshape(-1), orc.batch_mul_g1(cid, nq, g1, ex["gamma_abc"], 1).reshape(-1))


def _scalar_sets(cd, nv, seed):
    """full assignments (Montgomery limbs) whose canonical values follow the three distributions of SURVEY.md section 8d"""
    r = cd.c.r
    rs = np.random.RandomState(seed)
    uniform = rand_fr_mont(rs, nv)                                   # uniform-looking canonical values (after from_mont)
    kind = rs.randint(0, 4, size=nv)
    small = rs.randint(0, 1 << 32, size=nv, dtype=np.int64)
    bits = rs.randint(0, 2, size=nv)
    big = rs.randint(0, 1 << 62, size=(nv, 4), dtype=np.int64)
    mix_ints = [int(bits[i]) if kind[i] <= 1 else (int(small[i]) if kind[i] == 2 else
                (int(big[i, 0]) | int(big[i, 1]) << 62 | int(big[i, 2]) << 124 | int(big[i, 3]) << 186) % r) for i in range(nv)]
    mix = np.ascontiguousarray(cd.fr.enc(mix_ints))
    equal = np.ascontiguousarray(np.tile(cd.fr.enc1(0x1234567890abcdef1234567890abcdef1234567890abcdef % r), (nv, 1)))
    return {"uniform": uniform, "mix_50_25_25": mix, "all_equal": equal}


def _from_mont_bigints(cd, z):
    """Montgomery limbs -> canonical BigInt limbs (into_bigint, prover.rs:64,71,82) by Python big-int arithmetic"""
    return cd.fr.bigint(cd.fr.dec(z))


@pytest.mark.parametrize("log_n", [17, 20])
def test_msm_resident_key_geometry(log_n):
    """All five MSMs of the resident-key path (c = 16, one bucket set, 16 precomputed multiples per base; G1 and G2) through
    g16_prove_partial with three scalar distributions, each against the oracle's msm_bigint on the exported key."""
    curve = "bls12_381"
    m, z_sat, _ = workload(curve, "synthetic", log_n)
    g, pk = _setup(curve, m)
    cd = g.codec
    cid, nq = cd.c.cid, cd.nq
    ni, nw = m.num_instance_variables, m.num_witness_variables
    nv = ni + nw
    r1 = cd.fr.enc1(5)
    a_q = np.asarray(pk.a_query).reshape(nv, -1)
    b1_q = np.asarray(pk.b_g1_query).reshape(nv, -1)
    b2_q = np.asarray(pk.b_g2_query).reshape(nv, -1)
    for name, z in _scalar_sets(cd, nv, 7 + log_n).items():
        out = np.zeros(g.partial_limbs(), dtype=np.uint64)
        g.prove_partial_raw(r1, z.ctypes.data, 0, out)
        tm = g.timings()
        assert tm["msm_pairs"]["h"] == (1 << log_n) - 1 and tm["msm_pairs"]["a"] == nv - 1
        zc = _from_mont_bigints(cd, z)
        h = orc.witness_map(cid, m, z, threads=THREADS)
        want = [orc.msm_g1(cid, nq, pk.h_query, _from_mont_bigints(cd, h), THREADS),        # prover.rs:66 (truncates to n - 1)
                orc.msm_g1(cid, nq, pk.l_query, zc[ni:], THREADS),                           # prover.rs:74
                orc.msm_g1(cid, nq, a_q[1:], zc[1:], THREADS),                               # prover.rs:262 (a_query[1..])
                orc.msm_g1(cid, nq, b1_q[1:], zc[1:], THREADS)]
        for k, w in enumerate(want):
            got = out[2 * nq * k:2 * nq * (k + 1)]
            if not w[2 * nq:].any():
                assert not got.any(), (name, k)
            else:
                assert np.array_equal(got, w[:2 * nq]), (name, k)
        w2 = orc.msm_g2(cid, nq, b2_q[1:], zc[1:], THREADS)
        got2 = out[8 * nq:]
        if not w2[4 * nq:].any():
            assert not got2.any(), name
        else:
            assert np.array_equal(got2, w2[:4 * nq]), name


def _prove_and_check(curve, kind, log_n):
    m, z, pub = workload(curve, kind, log_n)
    g, pk = _setup(curve, m)
    cd = g.codec
    nq = cd.nq
    _check_key_sample(curve, g, m, pk)
    r, s = cd.fr.enc1(123456789), cd.fr.enc1(987654321)
    got = g.create_proof_with_reduction_and_matrices(None, r, s, None, m.num_instance_variables, m.num_constraints, z)
    want, _ = orc.prove(cd.c.cid, nq, pk, m, z, r, s, threads=THREADS)
    assert np.array_equal(got.a, want[:2 * nq]) and np.array_equal(got.b, want[2 * nq:6 * nq]) and np.array_equal(got.c, want[6 * nq:])
    # prover.rs:98 branch at full size: r == 0 skips B in G1
    got0 = g.create_proof_with_reduction_and_matrices(None, 0, s, None, m.num_instance_variables, m.num_constraints, z)
    want0, _ = orc.prove(cd.c.cid, nq, pk, m, z, cd.fr.enc1(0), s, threads=THREADS)
    assert np.array_equal(np.concatenate([got0.a, got0.b, got0.c]), want0)
    # the pairing check of the reference's own tests (verifier.rs:44-65) on the big-int oracle
    vk_only = pk_from_abi(curve, type(pk)(pk.vk, pk.beta_g1, pk.delta_g1, pk.a_query[:1], pk.b_g1_query[:1], pk.b_g2_query[:1],
                                          pk.h_query[:1], pk.l_query[:1]))
    assert P.verify_proof(vk_only.vk, P.CURVES[curve], proof_from_abi(curve, got), pub)
    assert not P.verify_proof(vk_only.vk, P.CURVES[curve], proof_from_abi(curve, got), [(pub[0] + 1) % cd.c.r] + list(pub[1:]))


@pytest.mark.parametrize("curve", ALL_CURVES)
def test_prove_synthetic_2p20(curve):
    """BASELINE configs[1] (BN254) / configs[2] (BLS12-381) / the curve of configs[4] (BLS12-377) at 2^20 constraints."""
    _prove_and_check(curve, "synthetic", 20)


def test_prove_dummy_circuit_2p20_minus_100():
    """The reference's own benchmark workload at its own size: DummyCircuit with 2^20 - 100 variables and constraints
    (benches/bench.rs:17-20): every witness scalar equal (one bucket per window), a/b queries almost all identity."""
    _prove_and_check("bls12_381", "dummy", 20)


def test_ntt_of_another_size_between_load_and_prove():
    """ADVICE r1 (high): g16_ntt with log_n != the resident circuit's must not disturb the prover's domain."""
    curve = "bn254"
    m, z, pub = synthetic_r1cs(curve, 9, seed=2)
    g, pk = _setup(curve, m)
    cd = g.codec
    nq = cd.nq
    r, s = cd.fr.enc1(11), cd.fr.enc1(13)
    vals = rand_fr_mont(np.random.RandomState(5), 1 << 12)
    for other in (12, 5):
        got_ntt = g.ntt_log(other, vals[:1 << other], inverse=False, coset=True)
        assert np.array_equal(got_ntt, orc.ntt(cd.c.cid, other, vals[:1 << other], coset=True, threads=2))
        got = g.create_proof_with_reduction_and_matrices(None, r, s, None, m.num_instance_variables, m.num_constraints, z)
        want, _ = orc.prove(cd.c.cid, nq, pk, m, z, r, s, threads=4)
        assert np.array_equal(np.concatenate([got.a, got.b, got.c]), want)
        h = g.witness_map_from_matrices(None, m.num_instance_variables, m.num_constraints, z)
        assert np.array_equal(h, orc.witness_map(cd.c.cid, m, z, threads=2))


def test_prove_uses_the_pk_argument():
    """ADVICE r1 (medium): create_proof_with_reduction_and_matrices proves under the `pk` it is given, also when another
    key is resident (prover.rs:26 takes the key by reference per call)."""
    from util import oracle_setup
    curve = "bn254"
    m, z, pub = synthetic_r1cs(curve, 8, seed=4)
    g, pk_gpu = _setup(curve, m)
    cd = g.codec
    other_toxic = (7, 11, 13, 17, 19)
    pk_other, _ = oracle_setup(curve, m, other_toxic, threads=4)
    r, s = cd.fr.enc1(3), cd.fr.enc1(4)
    got = g.create_proof_with_reduction_and_matrices(pk_other, r, s, None, m.num_instance_variables, m.num_constraints, z)
    want, _ = orc.prove(cd.c.cid, cd.nq, pk_other, m, z, r, s, threads=4)
    assert np.array_equal(np.concatenate([got.a, got.b, got.c]), want)
    got2 = g.create_proof_with_reduction_and_matrices(pk_gpu, r, s, None, m.num_instance_variables, m.num_constraints, z)
    want2, _ = orc.prove(cd.c.cid, cd.nq, pk_gpu, m, z, r, s, threads=4)
    assert np.array_equal(np.concatenate([got2.a, got2.b, got2.c]), want2)
