"""GPU tier for BW6-761 (curve id 3): every prover path against tests/bw6_ref.py, a big-integer reference written from the
curve's definition.  BW6-761 has no pairing here, so a proof is checked by the closed form "proof in the exponent":
with the toxic waste known, A, B and C are fixed multiples of the generators (bw6_ref.expected_proof), independently of
any MSM."""
import os
import random

import numpy as np
import pytest

import bw6_arith
import bw6_ref as ref
from groth16_b200 import ConstraintMatrices, Groth16, _lib
from groth16_b200.params import GENERATORS
from groth16_b200.serialize import ArkCodec, DeserializeError
from groth16_b200.workload import synthetic_r1cs

pytestmark = pytest.mark.gpu

CURVE = "bw6_761"
G1, G2 = GENERATORS[CURVE]["g1"], GENERATORS[CURVE]["g2"]
_ENG = {}


def engine(qap="libsnark"):
    if qap not in _ENG:
        _ENG[qap] = Groth16(CURVE, 0, qap=qap)
    return _ENG[qap]


@pytest.fixture(scope="module", autouse=True)
def _release_engines():
    """the shared contexts hold a 2^20 key with its precomputed copies: free the device memory for the modules after this"""
    yield
    for g in _ENG.values():
        g.close()
    _ENG.clear()


def rng_fr(rng):
    return rng.randrange(ref.R)


def toxic(seed):
    rng = random.Random(seed)
    return [rng_fr(rng) for _ in range(5)]


def silly():
    """MySillyCircuit of the reference's tests: a * b = c, c public"""
    a, b = 0x1234567, ref.R - 99
    c = a * b % ref.R
    # variables: 0 = One, 1 = c (instance), 2 = a, 3 = b, 4 = a*b
    rows_a = [[(1, 2)], [(1, 4)]]
    rows_b = [[(1, 3)], [(1, 0)]]
    rows_c = [[(1, 4)], [(1, 1)]]
    m = ConstraintMatrices.from_rows(CURVE, 2, 3, rows_a, rows_b, rows_c)
    return m, [1, c, a, b, c]


def mimc(rounds=40, seed=3):
    """MiMC-style chain: x_{i+1} = (x_i + k_i)^3 as two constraints per round (t = x + k, t*t = s, s*t = x')"""
    rng = random.Random(seed)
    ks = [rng_fr(rng) for _ in range(rounds)]
    x0 = rng_fr(rng)
    z = [1, 0, x0]   # One, output (instance), x0
    ra, rb, rc = [], [], []
    cur = 2
    x = x0
    for k in ks:
        t = (x + k) % ref.R
        s = t * t % ref.R
        x = s * t % ref.R
        z += [s]
        si = len(z) - 1
        ra.append([(1, cur), (k, 0)])
        rb.append([(1, cur), (k, 0)])
        rc.append([(1, si)])
        z += [x]
        xi = len(z) - 1
        ra.append([(1, si)])
        rb.append([(1, cur), (k, 0)])
        rc.append([(1, xi)])
        cur = xi
    z[1] = x
    ra.append([(1, cur)])
    rb.append([(1, 0)])
    rc.append([(1, 1)])
    m = ConstraintMatrices.from_rows(CURVE, 2, len(z) - 2, ra, rb, rc)
    return m, z


def prove_and_check(g, m, z, tw, r_, s_, expect_valid=True):
    pk = g.generate_parameters_with_qap(m, *tw, G1, G2)
    zl = np.ascontiguousarray(g.codec.fr.enc(z))
    pf = g.create_proof_with_reduction_and_matrices(None, r_, s_, None, m.num_instance_variables, m.num_constraints, zl)
    cd = g.codec
    got = (cd.dec_g1(pf.a)[0], cd.dec_g2(pf.b)[0], cd.dec_g1(pf.c)[0])
    alpha, beta, _gamma, delta, tau = tw
    want = ref.expected_proof(ref.csr_rows(m), m.num_instance_variables, z, alpha, beta, delta, tau, r_, s_, G1, G2)
    if expect_valid:
        assert got == want
    else:
        assert got[0] == want[0] and got[1] == want[1] and got[2] != want[2]
    return pk, pf, zl


def test_device_arithmetic():
    """the device build of tests/arith_bw6 (PTX carry chains, out-of-line 24-limb product, safegcd) at the edge operands"""
    so = os.path.join(os.path.dirname(os.path.abspath(__file__)), "arith_bw6", "libg16bw6arith.so")
    bad = bw6_arith.check_all(bw6_arith.load(so))
    assert not bad, bad[:5]


def _witness_map_ref(a, b, c):
    """LibsnarkReduction's h from row evaluations: coset-ifft((A B - C) / Z) with X = coset-fft(ifft(x))"""
    n = len(a)
    ac, bc, cc = (ref.ntt(ref.ntt(x, inverse=True), coset=True) for x in (a, b, c))
    zi = pow((pow(ref.FR_GENERATOR, n, ref.R) - 1) % ref.R, -1, ref.R)
    return ref.ntt([(x * y - z) * zi % ref.R for x, y, z in zip(ac, bc, cc)], inverse=True, coset=True)


@pytest.mark.parametrize("log_n", [1, 3, 5])
def test_witness_map_evals(log_n):
    g = engine()
    rng = random.Random(log_n)
    n = 1 << log_n
    a, b, c = ([rng_fr(rng) for _ in range(n)] for _ in range(3))
    a[0] = ref.R - 1
    fr = g.codec.fr
    assert fr.dec(g.witness_map_from_evals(fr.enc(a), fr.enc(b), fr.enc(c))) == _witness_map_ref(a, b, c)


def test_witness_map_resident_circuit():
    g = engine()
    m, z = silly()
    g.load_matrices(m)
    h = g.codec.fr.dec(g.witness_map_from_matrices(m, m.num_instance_variables, m.num_constraints,
                                                   np.ascontiguousarray(g.codec.fr.enc(z))))
    rows = ref.csr_rows(m)
    nc, ni = m.num_constraints, m.num_instance_variables
    n = len(h)
    ev = [[sum(cf * z[v] for cf, v in row) % ref.R for row in mat] + [0] * (n - nc) for mat in rows]
    for i in range(ni):
        ev[0][nc + i] = z[i]
    assert h == _witness_map_ref(*ev)


def test_abi_sizes():
    g = engine()
    lib = g._lib
    assert lib.g16_fr_limbs(g._ctx) == 6 and lib.g16_fq_limbs(g._ctx) == 12 and lib.g16_g2_limbs(g._ctx) == 24
    assert g.partial_limbs() == 4 * 24 + 24
    assert g.nr == 6 and g.ng2 == 24


@pytest.mark.parametrize("log_n", list(range(1, 15)) + [18])
def test_ntt(log_n):
    g = engine()
    rng = random.Random(log_n)
    n = 1 << log_n
    x = [rng_fr(rng) for _ in range(n)]
    if log_n <= 4:
        x[0] = ref.R - 1
    xl = g.codec.fr.enc(x)
    outs = {(inv, cos): g.codec.fr.dec(g.ntt(xl, inverse=inv, coset=cos)) for inv in (False, True) for cos in (False, True)}
    if log_n <= 6:
        for (inv, cos), got in outs.items():
            assert got == ref.ntt(x, inverse=inv, coset=cos), (inv, cos)
    else:
        w = ref.domain_root(log_n)
        for k in (0, 1, n // 2 + 3, n - 1):   # y_k = sum_i x_i (g^i) w^(ik) at sampled k
            wk = pow(w, k, ref.R)
            for cos in (False, True):
                step = wk * (ref.FR_GENERATOR if cos else 1) % ref.R
                acc = 0
                for v in reversed(x):
                    acc = (acc * step + v) % ref.R
                assert outs[(False, cos)][k] == acc
        for cos in (False, True):   # inverse transforms: each undoes its forward transform
            back = g.codec.fr.dec(g.ntt(g.codec.fr.enc(outs[(False, cos)]), inverse=True, coset=cos))
            assert back == x


@pytest.mark.parametrize("grp", ["g1", "g2"])
def test_msm_edges(grp):
    g = engine()
    cd = g.codec
    b = ref.B1 if grp == "g1" else ref.B2
    gen = G1 if grp == "g1" else G2
    rng = random.Random(7)
    n = 40
    bases = [ref.mul(rng_fr(rng), gen) for _ in range(n)]
    bases[3] = None   # identity base
    bases[9] = None
    scal = [rng_fr(rng) for _ in range(n)]
    # (1 << 376) - 1: every window all ones, so every signed digit is negative and the carry runs up into the last window
    # (the one above bit 376) at any window size; (1 << 376) | 0xFFFF: the top bit alone above a full low block
    scal[:6] = [0, 1, ref.R - 1, (1 << 376) | 0xFFFF, ref.R - 2, (1 << 376) - 1]
    assert all(ref.on_curve(P, b) for P in bases)
    enc = cd.enc_g1 if grp == "g1" else cd.enc_g2
    fn = g.msm_g1 if grp == "g1" else g.msm_g2
    dec = cd.dec_proj_g1 if grp == "g1" else cd.dec_proj_g2
    out = fn(enc(bases), cd.fr.bigint(scal))
    assert dec(out) == ref.msm(bases, scal)
    assert dec(fn(enc(bases[:1]), cd.fr.bigint([0]))) is None


def test_setup_queries():
    g = engine()
    m, z = silly()
    tw = toxic(11)
    pk = g.generate_parameters_with_qap(m, *tw, G1, G2)
    cd = g.codec
    alpha, beta, gamma, delta, tau = tw
    assert cd.dec_g1(pk.vk.alpha_g1)[0] == ref.mul(alpha, G1)
    assert cd.dec_g2(pk.vk.beta_g2)[0] == ref.mul(beta, G2)
    assert cd.dec_g2(pk.vk.gamma_g2)[0] == ref.mul(gamma, G2)
    assert cd.dec_g2(pk.vk.delta_g2)[0] == ref.mul(delta, G2)
    assert cd.dec_g1(pk.delta_g1)[0] == ref.mul(delta, G1)
    # a_i(tau) of every variable, from the rows and the instance copies
    rows = ref.csr_rows(m)
    nc, ni = m.num_constraints, m.num_instance_variables
    L = (nc + ni - 1).bit_length()
    lag = ref.lagrange_at(tau, L)
    nv = len(z)
    qa, qb = [0] * nv, [0] * nv
    for j, row in enumerate(rows[0]):
        for cf, v in row:
            qa[v] += lag[j] * cf
    for j, row in enumerate(rows[1]):
        for cf, v in row:
            qb[v] += lag[j] * cf
    for i in range(ni):
        qa[i] += lag[nc + i]
    assert cd.dec_g1(pk.a_query) == [ref.mul(x % ref.R, G1) for x in qa]
    assert cd.dec_g2(pk.b_g2_query) == [ref.mul(x % ref.R, G2) for x in qb]
    n = 1 << L
    zt = (pow(tau, n, ref.R) - 1) % ref.R
    di = pow(delta, -1, ref.R)
    assert cd.dec_g1(pk.h_query) == [ref.mul(zt * di * pow(tau, i, ref.R) % ref.R, G1) for i in range(n - 1)]


def test_silly_and_mimc_proofs():
    g = engine()
    for k, (m, z) in enumerate((silly(), mimc())):
        tw = toxic(20 + k)
        rng = random.Random(k)
        prove_and_check(g, m, z, tw, rng_fr(rng), rng_fr(rng))
        prove_and_check(g, m, z, tw, 0, rng_fr(rng))          # r = 0
        bad = list(z)
        bad[2] = (bad[2] + 1) % ref.R                          # an assignment that does not satisfy the circuit
        prove_and_check(g, m, bad, tw, rng_fr(rng), rng_fr(rng), expect_valid=False)


@pytest.mark.parametrize("log_n", [6, 8, 10, 12])
def test_synthetic_proofs(log_n):
    g = engine()
    m, zl, _ = synthetic_r1cs(CURVE, log_n, seed=log_n)
    z = g.codec.fr.dec(zl)
    rng = random.Random(log_n)
    prove_and_check(g, m, z, toxic(log_n), rng_fr(rng), rng_fr(rng))


def test_synthetic_2p20_proof():
    g = engine()
    m, zl, _ = synthetic_r1cs(CURVE, 20, seed=5)
    z = g.codec.fr.dec(zl)
    rng = random.Random(20)
    prove_and_check(g, m, z, toxic(99), rng_fr(rng), rng_fr(rng))


def _rows(g, z, count, seed):
    """`count` proof inputs: (r, s) and a distinct assignment each (z itself first, then random values after One; a proof
    is a deterministic function of its inputs whether or not they satisfy the circuit), proof 1 with r = 0"""
    rng = random.Random(seed)
    out = []
    for k in range(count):
        zk = z if k == 0 else np.ascontiguousarray(g.codec.fr.enc([1] + [rng_fr(rng) for _ in range(z.shape[0] - 1)]))
        out.append((0 if k == 1 else rng_fr(rng), rng_fr(rng), zk))
    return out


def test_slots_batch_and_sharded():
    g = engine()
    m, zl, _ = synthetic_r1cs(CURVE, 10, seed=1)
    g.generate_parameters_with_qap(m, *toxic(5), G1, G2, export=False)
    pk = g.export_proving_key()
    rs = _rows(g, zl, 5, 3)
    cd = g.codec
    singles = [g.create_proof_with_reduction_and_matrices(None, r_, s_, None, m.num_instance_variables, m.num_constraints, zk)
               for r_, s_, zk in rs]
    flat = lambda p: np.concatenate([p.a, p.b, p.c])
    # both slots in flight
    outs = [np.zeros(4 * g.nq + g.ng2, dtype=np.uint64) for _ in rs]
    lim = [(np.ascontiguousarray(cd.fr.enc1(r_)), np.ascontiguousarray(cd.fr.enc1(s_))) for r_, s_, _ in rs]
    g.prove_submit_raw(0, lim[0][0], lim[0][1], rs[0][2].ctypes.data, 0)
    for i in range(1, len(rs)):
        g.prove_submit_raw(i & 1, lim[i][0], lim[i][1], rs[i][2].ctypes.data, 0)
        g.prove_wait_raw((i - 1) & 1, outs[i - 1])
    g.prove_wait_raw((len(rs) - 1) & 1, outs[-1])
    for o, p in zip(outs, singles):
        assert np.array_equal(o, flat(p))
    # batch proving in one group, in groups of 2 and of 1
    assert len({p.c.tobytes() for p in singles}) == len(rs)
    zs = np.ascontiguousarray(np.stack([zk for _, _, zk in rs]))
    for group in (0, 2, 1):
        got = g.create_proofs_batch([r_ for r_, _, _ in rs], [s_ for _, s_, _ in rs], zs, group=group)
        for p, q in zip(got, singles):
            assert np.array_equal(flat(p), flat(q)), group
    # partial / assemble: world 2 and 3, one context per rank
    r_, s_, _ = rs[0]
    rl = np.ascontiguousarray(cd.fr.enc1(r_))
    for world in (2, 3):
        parts = []
        ranks = [Groth16(CURVE, 0) for _ in range(world)]
        try:
            for rank, e in enumerate(ranks):
                e.load_matrices(m)
                e.load_proving_key(pk, rank, world)
                out = np.zeros(e.partial_limbs(), dtype=np.uint64)
                e.prove_partial_raw(rl, zl.ctypes.data, 0, out)
                parts.append(out)
            assert np.array_equal(flat(ranks[0].prove_assemble(r_, s_, np.stack(parts))), flat(singles[0]))
        finally:
            for e in ranks:
                e.close()


def test_circom_equals_libsnark():
    m, zl, _ = synthetic_r1cs(CURVE, 9, seed=2)
    tw = toxic(9)
    r_, s_ = 123456789, ref.R - 5
    proofs = []
    for qap in ("libsnark", "circom"):
        g = engine(qap)
        g.generate_parameters_with_qap(m, *tw, G1, G2, export=False)
        p = g.create_proof_with_reduction_and_matrices(None, r_, s_, None, m.num_instance_variables, m.num_constraints, zl)
        proofs.append(np.concatenate([p.a, p.b, p.c]))
    assert np.array_equal(proofs[0], proofs[1])


def test_serialized_key_round_trips():
    g = engine()
    m, zl, _ = synthetic_r1cs(CURVE, 7, seed=8)
    g.generate_parameters_with_qap(m, *toxic(4), G1, G2, export=False)
    r_, s_ = 77, 88
    want = g.create_proof_with_reduction_and_matrices(None, r_, s_, None, m.num_instance_variables, m.num_constraints, zl)
    codec = ArkCodec(CURVE, check_subgroup=True)
    pk = g.export_proving_key()
    for compress in (True, False):
        data = g.export_proving_key_bytes(compress=compress)
        vk = (g.codec.dec_g1(pk.vk.alpha_g1)[0], g.codec.dec_g2(pk.vk.beta_g2)[0], g.codec.dec_g2(pk.vk.gamma_g2)[0],
              g.codec.dec_g2(pk.vk.delta_g2)[0], g.codec.dec_g1(pk.vk.gamma_abc_g1))
        host = codec.proving_key(vk, g.codec.dec_g1(pk.beta_g1)[0], g.codec.dec_g1(pk.delta_g1)[0], g.codec.dec_g1(pk.a_query),
                                 g.codec.dec_g1(pk.b_g1_query), g.codec.dec_g2(pk.b_g2_query), g.codec.dec_g1(pk.h_query),
                                 g.codec.dec_g1(pk.l_query), compress=compress)
        assert data == host
        e = Groth16(CURVE, 0)
        try:
            e.load_matrices(m)
            e.load_proving_key_bytes(data, compress=compress, validate=True)
            got = e.create_proof_with_reduction_and_matrices(None, r_, s_, None, m.num_instance_variables, m.num_constraints, zl)
            assert np.array_equal(np.concatenate([got.a, got.b, got.c]), np.concatenate([want.a, want.b, want.c]))
            # off the curve: the last byte-pair of beta_g2's y (uncompressed) or a flipped x bit (compressed: no root or
            # another point; the two checks differ, so use an uncompressed stream for the off-curve case)
            nb = 96
            if not compress:
                bad = bytearray(data)
                bad[nb * 2 + 5] ^= 1          # vk.beta_g2.x: (x', y) is off the curve
                with pytest.raises(DeserializeError):
                    e.load_proving_key_bytes(bytes(bad), compress=False, validate=True)
            # not in the subgroup: a curve point without the cofactor cleared, in place of alpha_g1 (G1: y^2 = x^3 - 1) and
            # of vk.beta_g2 (G2 over Fq: y^2 = x^3 + 4), which follows alpha_g1 in the stream
            g1_size = len(codec.point(None, False, compress))
            for b, is_g2, off in ((ref.B1, False, 0), (ref.B2, True, g1_size)):
                rng = random.Random(1)
                while True:
                    x = rng.randrange(ref.Q)
                    y = ref.sqrt_fq((x ** 3 + b) % ref.Q)
                    if y is not None and ref.mul(ref.R, (x, y)) is not None:
                        break
                enc = codec.point((x, y), is_g2, compress)
                bad = bytearray(data)
                bad[off:off + len(enc)] = enc
                with pytest.raises(DeserializeError, match="subgroup"):
                    e.load_proving_key_bytes(bytes(bad), compress=compress, validate=True)
        finally:
            e.close()


@pytest.mark.parametrize("rounds", range(7))
def test_batched_affine_rounds(rounds):
    g = engine()
    m, zl, _ = synthetic_r1cs(CURVE, 14, seed=6)
    g.generate_parameters_with_qap(m, *toxic(14), G1, G2, export=False)
    r_, s_ = 5, 6
    base = g.create_proof_with_reduction_and_matrices(None, r_, s_, None, m.num_instance_variables, m.num_constraints, zl)
    keep = {k: g.get_option(k) for k in ("msm_ba", "msm_ba_g2", "ba_min_entries_g1", "ba_min_entries_g2", "ba_adaptive")}
    try:
        for k, v in (("msm_ba", rounds), ("msm_ba_g2", rounds), ("ba_min_entries_g1", 1 << 18), ("ba_min_entries_g2", 1 << 18),
                     ("ba_adaptive", 0)):
            g.set_option(k, v)
        assert g.config()["ba_rounds_g1"] == rounds and g.config()["ba_rounds_g2"] == rounds
        for gcd in (1, 0):   # safegcd and Fermat inversion
            g.set_option("ba_inv_gcd", gcd)
            p = g.create_proof_with_reduction_and_matrices(None, r_, s_, None, m.num_instance_variables, m.num_constraints, zl)
            assert np.array_equal(np.concatenate([p.a, p.b, p.c]), np.concatenate([base.a, base.b, base.c]))
    finally:
        g.set_option("ba_inv_gcd", 1)
        for k, v in keep.items():
            g.set_option(k, v)
