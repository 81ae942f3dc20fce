"""GPU tier of the witness check (g16_check_witness / Groth16.check_witness and the G16_CHECK_WITNESS prover flag; run on an
H100 with `pytest -m gpu`).

Every expected report comes from Python big-integer row evaluations (pyref.evaluate_constraint) and limb comparisons against
r, never from the library.  Covered: clean reports on all four curves under both reductions; reports after perturbations
(one, two or many witness elements, an instance element, a column only C reads, a row of 1100 terms); the first failing
row at 0, at nc - 1, above 2^16 and among the last rows of a 2^20 circuit; a fully random assignment; malformed elements on
all four curves; every prover path with the flag, for satisfied and unsatisfied assignments; a batch with a rejected and a
malformed proof; 65541 assignments in one call (grid-y limit and upload chunks); CircomReduction, whose witness map never
reads C; the argument checks; and (with two or more GPUs) a rejected sharded proof over the in-library NCCL exchange."""
import os
import random
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest

import orc
import pyref as P
from groth16_b200 import CHECK_WITNESS, ConstraintMatrices, Groth16, Unsatisfiable, WitnessReport, _lib
from groth16_b200.codec import ints_to_limbs, limbs_to_ints
from groth16_b200.params import GENERATORS, get_curve
from groth16_b200.workload import synthetic_r1cs

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CURVES = ["bls12_381", "bn254", "bls12_377", "bw6_761"]
TOXIC = (0x1111111111111111111111, 0x2222222222222222222223, 0x3333333333333333333335, 0x4444444444444444444447,
         0x5555555555555555555559)
_ENG = {}


def engine(curve, qap="libsnark") -> Groth16:
    if (curve, qap) not in _ENG:
        _ENG[(curve, qap)] = Groth16(curve, 0, qap=qap)
    return _ENG[(curve, qap)]


@pytest.fixture(scope="module", autouse=True)
def _engines():
    yield
    for g in _ENG.values():
        g.close()
    _ENG.clear()


# ---- the oracle: big-integer rows ----------------------------------------------------------------------------------------
def csr_rows(g, m):
    """(A, B, C) rows of `m` as lists of (coefficient, column) with canonical ints"""
    out = []
    for rp, col, val in (m.a, m.b, m.c):
        vals = g.codec.fr.dec(val) if len(col) else []
        cols = col.tolist()
        rp = rp.tolist()
        out.append([list(zip(vals[rp[i]:rp[i + 1]], cols[rp[i]:rp[i + 1]])) for i in range(m.num_constraints)])
    return out


def oracle(g, rows, z) -> WitnessReport:
    """the report of limbs `z` (nv, F): the first element >= r (element 0: not One) wins; else every constraint row"""
    fr = g.codec.fr
    r, mont_one = fr.p, fr.R % fr.p
    raw = limbs_to_ints(z, fr.nl)
    for j, v in enumerate(raw):
        if (j == 0 and v != mont_one) or v >= r:
            return WitnessReport(None, 0, j)
    zi = [v * fr.Rinv % r for v in raw]
    first, cnt = None, 0
    for i, (ra, rb, rc) in enumerate(zip(*rows)):
        if P.evaluate_constraint(ra, zi, r) * P.evaluate_constraint(rb, zi, r) % r != P.evaluate_constraint(rc, zi, r):
            cnt += 1
            first = i if first is None else first
    return WitnessReport(first, cnt, None)


def bumped(g, z, idx, by=1):
    """z with the canonical values at `idx` increased by `by`"""
    zi = g.codec.fr.dec(z)
    for j in idx:
        zi[j] = (zi[j] + by) % g.curve.r
    return np.ascontiguousarray(g.codec.fr.enc(zi))


def c_only_columns(m):
    used = set(m.a[1].tolist()) | set(m.b[1].tolist())
    return sorted(set(m.c[1].tolist()) - used)


# ---- circuits --------------------------------------------------------------------------------------------------------
def from_r1cs(curve, cs):
    m = ConstraintMatrices.from_rows(curve, cs.num_instance, cs.num_witness, cs.a, cs.b, cs.c)
    return m, np.ascontiguousarray(engine(curve).codec.fr.enc(cs.assignment))


def small_circuits(curve):
    """MySillyCircuit, MiMC, DummyCircuit and synthetic circuits with domains 2^1 and 2^2 (Python rows, satisfied)"""
    c = SimpleNamespace(r=get_curve(curve).r, name=curve)
    rng = random.Random(5)
    return {
        "silly": P.silly_circuit(c, rng.randrange(c.r), rng.randrange(c.r)),
        "mimc": P.mimc_circuit(c, 3, 4, [rng.randrange(c.r) for _ in range(P.MIMC_ROUNDS)]),
        "dummy": P.dummy_circuit(c, rng.randrange(c.r), rng.randrange(c.r), 10, 20),
        "log1": P.synthetic_circuit(c, 1, seed=3, num_inputs=0),
        "log2": P.synthetic_circuit(c, 2, seed=4, num_inputs=1),
    }


def wide_circuit(curve, seed=9):
    """row 0: A = sum of 1100 terms, B = One, C = w_out; rows 1-3 small (row 2: x = w_0 + w_1).  Columns w_p and w_sq appear
    only in C."""
    r = get_curve(curve).r
    rng = random.Random(seed)
    nw_in = 1100
    w = [rng.randrange(r) for _ in range(nw_in)]
    x = (w[0] + w[1]) % r
    k = [rng.randrange(1, r) for _ in range(nw_in)]
    out = sum(a * b for a, b in zip(k, w)) % r
    wp, wsq = w[0] * w[1] % r, out * out % r
    # columns: 0 One, 1 x, 2 .. 1101 w, 1102 w_out, 1103 w_p, 1104 w_sq
    A = [[(k[j], 2 + j) for j in range(nw_in)], [(1, 2)], [(1, 2), (1, 3)], [(1, 1102)]]
    B = [[(1, 0)], [(1, 3)], [(1, 0)], [(1, 1102)]]
    C = [[(1, 1102)], [(1, 1103)], [(1, 1)], [(1, 1104)]]
    m = ConstraintMatrices.from_rows(curve, 2, nw_in + 3, A, B, C)
    z = np.ascontiguousarray(engine(curve).codec.fr.enc([1, x] + w + [out, wp, wsq]))
    return m, z


def reports(g, z, **kw):
    return g.check_witness(z, **kw)


# ---- 1. clean reports ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("qap", ["libsnark", "circom"])
@pytest.mark.parametrize("curve", CURVES)
def test_clean_reports(curve, qap):
    g = engine(curve, qap)
    circuits = [from_r1cs(curve, cs) for cs in small_circuits(curve).values()]
    circuits += [synthetic_r1cs(curve, ln, seed=ln)[:2] for ln in range(3, 14)]
    circuits.append(wide_circuit(curve))
    for m, z in circuits:
        g.load_matrices(m)
        assert reports(g, z) == [WitnessReport(None, 0, None)]
        assert g.is_satisfied(z) and g.which_is_unsatisfied(z) is None


@pytest.mark.parametrize("qap", ["libsnark", "circom"])
@pytest.mark.parametrize("log_n", [16, 20])
def test_clean_reports_large(log_n, qap):
    g = engine("bls12_381", qap)
    m, z, _ = synthetic_r1cs("bls12_381", log_n, seed=log_n)
    g.load_matrices(m)
    assert reports(g, np.stack([z, z])) == [WitnessReport(None, 0, None)] * 2


# ---- 2. oracle reports after perturbations -----------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
def test_perturbed_reports(curve):
    g = engine(curve)
    rng = random.Random(17)
    for m, z in (synthetic_r1cs(curve, 10, seed=2)[:2], wide_circuit(curve)):
        g.load_matrices(m)
        rows = csr_rows(g, m)
        nv = z.shape[0]
        conly = c_only_columns(m)
        assert conly
        # columns from 4 on are constrained in both circuits (the synthetic circuit's seed witnesses 2 and 3 need not be)
        cases = [
            [rng.randrange(4, nv)],                               # one witness element
            rng.sample(range(4, nv), 2),                          # two
            rng.sample(range(4, nv), min(60, nv - 4)),            # many
            [1],                                                  # an instance element
            [conly[-1]],                                          # a column only C reads
            [4],                                                  # the wide row's third term
        ]
        zs = np.stack([bumped(g, z, idx, by=rng.randrange(1, 1 << 64)) for idx in cases])
        want = [oracle(g, rows, zk) for zk in zs]
        assert all(w.num_unsatisfied > 0 for w in want)
        assert reports(g, zs) == want
        for zk, w in zip(zs, want):
            assert not g.is_satisfied(zk) and g.which_is_unsatisfied(zk) == w.first_unsatisfied


# ---- 3. edge rows --------------------------------------------------------------------------------------------------------
def test_edge_rows_2p20():
    g = engine("bls12_381")
    m, z, _ = synthetic_r1cs("bls12_381", 20, seed=20)
    g.load_matrices(m)
    nc = m.num_constraints
    out_col = m.c[1]   # the column each synthetic row defines
    rows = csr_rows(g, m)
    zs = np.stack([bumped(g, z, [int(out_col[i])]) for i in (0, nc - 1, 70001, nc - 3)])
    want = [oracle(g, rows, zk) for zk in zs]
    assert [w.first_unsatisfied for w in want] == [0, nc - 1, 70001, nc - 3]
    assert reports(g, zs) == want


def test_fully_random_assignment_2p16():
    g = engine("bls12_381")
    m, z, _ = synthetic_r1cs("bls12_381", 16, seed=16)
    g.load_matrices(m)
    rng = random.Random(3)
    zr = np.ascontiguousarray(g.codec.fr.enc([1] + [rng.randrange(g.curve.r) for _ in range(z.shape[0] - 1)]))
    want = oracle(g, csr_rows(g, m), zr)
    assert want == WitnessReport(0, m.num_constraints, None)
    assert reports(g, zr) == [want]


# ---- 4. malformed elements ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
def test_malformed_elements(curve):
    g = engine(curve)
    m, z, _ = synthetic_r1cs(curve, 8, seed=8)
    g.load_matrices(m)
    fr = g.codec.fr
    nv = z.shape[0]
    r_limbs = ints_to_limbs([fr.p], fr.nl)[0]
    top = np.full(fr.nl, np.uint64(0xFFFFFFFFFFFFFFFF), dtype=np.uint64)
    rows = csr_rows(g, m)
    cases = []
    for j, v in ((5, r_limbs), (7, top), (nv - 1, r_limbs), (0, np.zeros(fr.nl, dtype=np.uint64)), (0, fr.enc1(2)),
                 (0, r_limbs)):
        zk = bumped(g, z, [3])                            # unsatisfied rows too: the element wins
        zk[j] = v
        if 0 < j < nv - 1:
            zk[j + 1] = r_limbs                           # a later malformed element does not hide the first
        cases.append((j, zk))
    zs = np.stack([zk for _, zk in cases])
    want = [WitnessReport(None, 0, j) for j, _ in cases]
    assert [oracle(g, rows, zk) for zk in zs] == want
    assert reports(g, zs) == want
    for zk in zs:
        assert not g.is_satisfied(zk)
        with pytest.raises(Unsatisfiable):
            g.which_is_unsatisfied(zk)


# ---- 5. / 6. the prover flag ------------------------------------------------------------------------------------------
class Prover:
    def __init__(self, curve, log_n=10):
        self.g = engine(curve)
        G = GENERATORS[curve]
        self.m, self.z, _ = synthetic_r1cs(curve, log_n, seed=40 + log_n)
        self.pk = self.g.generate_parameters_with_qap(self.m, *TOXIC, G["g1"], G["g2"], export=True)
        self.rows = csr_rows(self.g, self.m)
        self.nv = self.z.shape[0]
        self.plimbs = 4 * self.g.nq + self.g.ng2
        self.rng = random.Random(11)

    def fr(self, xs):
        return np.ascontiguousarray(self.g.codec.fr.enc(xs))

    def rs(self, k):
        r = self.g.curve.r
        return self.fr([self.rng.randrange(r) for _ in range(k)]), self.fr([self.rng.randrange(r) for _ in range(k)])

    def prove(self, r, s, z, flags=0, out=None):
        out = np.zeros(self.plimbs, dtype=np.uint64) if out is None else out
        self.g.prove_raw(np.ascontiguousarray(r), np.ascontiguousarray(s), np.ascontiguousarray(z).ctypes.data, flags, out)
        return out

    def launches(self):
        return self.g.timings()["launches"]

    def witness_map(self, z, flags, h):
        return self.g._lib.g16_witness_map(self.g._ctx, z.ctypes.data, flags, h.ctypes.data)


SENTINEL = np.uint64(0xA5A5A5A5A5A5A5A5)


@pytest.mark.parametrize("curve", ["bls12_381", "bw6_761"])
def test_flag_satisfied_paths_unchanged(curve):
    p = Prover(curve)
    g, z = p.g, p.z
    r, s = p.rs(3)
    base = p.prove(r[0], s[0], z)
    l0 = p.launches()
    assert np.array_equal(p.prove(r[0], s[0], z, CHECK_WITNESS), base)
    assert p.launches() == l0 + 1
    # submit / wait in both slots
    for slot in (0, 1):
        g.prove_submit_raw(slot, r[0], s[0], z.ctypes.data, CHECK_WITNESS)
    outs = [np.zeros(p.plimbs, dtype=np.uint64) for _ in range(2)]
    for slot in (0, 1):
        g.prove_wait_raw(slot, outs[slot])
        assert np.array_equal(outs[slot], base)
    # batch, group auto, 1 and 2
    zs = np.stack([z] * 3)
    plain = {}
    for group in (0, 1, 2):
        out = np.zeros((3, p.plimbs), dtype=np.uint64)
        g.prove_batch_raw(3, r, s, zs.ctypes.data, group, 0, out)
        plain[group] = (out, p.launches())
        out2 = np.zeros_like(out)
        g.prove_batch_raw(3, r, s, zs.ctypes.data, group, CHECK_WITNESS, out2)
        assert np.array_equal(out2, out)
        groups = {0: 1, 1: 3, 2: 2}[group]
        assert p.launches() == plain[group][1] + groups
    assert np.array_equal(plain[0][0][0], base)
    # partial + assemble
    part = np.zeros(g.partial_limbs(), dtype=np.uint64)
    g.prove_partial_raw(r[0], z.ctypes.data, 0, part)
    part2 = np.zeros_like(part)
    g.prove_partial_raw(r[0], z.ctypes.data, CHECK_WITNESS, part2)
    assert np.array_equal(part, part2)
    pf = g.prove_assemble(r[0], s[0], part2)
    assert np.array_equal(np.concatenate([pf.a, pf.b, pf.c]), base)
    # witness map
    n = 1 << g._lib.g16_domain_log(g._ctx)
    h0 = np.zeros((n, g.nr), dtype=np.uint64)
    h1 = np.zeros_like(h0)
    assert p.witness_map(z, 0, h0) == 0 and p.witness_map(z, CHECK_WITNESS, h1) == 0
    assert np.array_equal(h0, h1)
    # device-resident assignments
    import torch
    dz = torch.from_numpy(zs.view(np.int64).reshape(-1)).to("cuda:0")
    torch.cuda.synchronize()
    out = np.zeros(p.plimbs, dtype=np.uint64)
    g.prove_raw(r[0], s[0], dz.data_ptr(), _lib.ASSIGNMENT_ON_DEVICE | CHECK_WITNESS, out)
    assert np.array_equal(out, base)
    outb = np.zeros((3, p.plimbs), dtype=np.uint64)
    g.prove_batch_raw(3, r, s, dz.data_ptr(), 0, _lib.ASSIGNMENT_ON_DEVICE | CHECK_WITNESS, outb)
    assert np.array_equal(outb, plain[0][0])
    assert reports(g, dz.data_ptr(), count=3, flags=_lib.ASSIGNMENT_ON_DEVICE) == [WitnessReport(None, 0, None)] * 3


def test_flag_unsatisfied_paths_refuse():
    p = Prover("bls12_381")
    g, z, nq = p.g, p.z, p.g.nq
    out_col = p.m.c[1]
    bad = bumped(g, z, [int(out_col[7])])
    want = oracle(g, p.rows, bad)
    assert want.first_unsatisfied == 7
    msg = f"constraint 7 unsatisfied ({want.num_unsatisfied} in all)"
    r, s = p.rs(2)
    oracle_proof = lambda rr, ss, zz: orc.prove(g.curve.cid, nq, p.pk, p.m, zz, rr, ss, threads=8)[0]
    good = oracle_proof(r[1], s[1], z)

    def refused(call):
        with pytest.raises(Unsatisfiable, match=msg.replace("(", r"\(").replace(")", r"\)")):
            call()

    out = np.full(p.plimbs, SENTINEL, dtype=np.uint64)
    refused(lambda: p.prove(r[0], s[0], bad, CHECK_WITNESS, out))
    assert (out == SENTINEL).all()
    assert np.array_equal(p.prove(r[1], s[1], z, CHECK_WITNESS), good)   # slot 0 free again, next proof correct
    # submit / wait: bad in slot 0, good in slot 1
    g.prove_submit_raw(0, r[0], s[0], bad.ctypes.data, CHECK_WITNESS)
    g.prove_submit_raw(1, r[1], s[1], z.ctypes.data, CHECK_WITNESS)
    out0 = np.full(p.plimbs, SENTINEL, dtype=np.uint64)
    out1 = np.zeros(p.plimbs, dtype=np.uint64)
    refused(lambda: g.prove_wait_raw(0, out0))
    g.prove_wait_raw(1, out1)
    assert (out0 == SENTINEL).all() and np.array_equal(out1, good)
    # partial, partial submit / wait
    part = np.full(g.partial_limbs(), SENTINEL, dtype=np.uint64)
    refused(lambda: g.prove_partial_raw(r[0], bad.ctypes.data, CHECK_WITNESS, part))
    g.prove_partial_submit_raw(1, r[0], bad.ctypes.data, CHECK_WITNESS)
    refused(lambda: g.prove_partial_wait_raw(1, part))
    assert (part == SENTINEL).all()
    # witness map
    n = 1 << g._lib.g16_domain_log(g._ctx)
    h = np.full((n, g.nr), SENTINEL, dtype=np.uint64)
    assert p.witness_map(bad, CHECK_WITNESS, h) == _lib.ERR_UNSATISFIED
    assert _lib.last_error() == msg and (h == SENTINEL).all()
    with pytest.raises(Unsatisfiable):
        g.witness_map_from_matrices(None, p.m.num_instance_variables, p.m.num_constraints, bad, flags=CHECK_WITNESS)
    # batch of one, then both slots reusable
    ob = np.full((1, p.plimbs), SENTINEL, dtype=np.uint64)
    refused(lambda: g.prove_batch_raw(1, r[:1], s[:1], bad.ctypes.data, 0, CHECK_WITNESS, ob))
    assert (ob == 0).all()
    for slot in (0, 1):
        g.prove_submit_raw(slot, r[1], s[1], z.ctypes.data, CHECK_WITNESS)
    for slot in (0, 1):
        g.prove_wait_raw(slot, out1)
        assert np.array_equal(out1, good)
    # a malformed element names the element
    mal = z.copy()
    mal[5] = ints_to_limbs([g.curve.r], g.nr)[0]
    with pytest.raises(Unsatisfiable, match="assignment element 5 is not a canonical Fr"):
        p.prove(r[0], s[0], mal, CHECK_WITNESS)
    mal = z.copy()
    mal[0] = g.codec.fr.enc1(2)
    with pytest.raises(Unsatisfiable, match="assignment element 0 is not One"):
        p.prove(r[0], s[0], mal, CHECK_WITNESS)


# ---- 7. batch of 20 ----------------------------------------------------------------------------------------------------
def test_batch_of_20():
    p = Prover("bls12_381")
    g, z = p.g, p.z
    r, s = p.rs(20)
    zs = np.stack([bumped(g, z, [p.nv - 1 - k]) if k % 5 == 4 else z for k in range(20)])
    zs[3] = bumped(g, z, [int(p.m.c[1][11])])
    zs[17][9] = ints_to_limbs([g.curve.r], g.nr)[0]
    want = [oracle(g, p.rows, zk) for zk in zs]
    bad = [k for k, w in enumerate(want) if not w.ok]
    assert 3 in bad and 17 in bad and bad[0] == 3
    assert reports(g, zs) == want
    plain = np.zeros((20, p.plimbs), dtype=np.uint64)
    g.prove_batch_raw(20, r, s, zs.ctypes.data, 0, 0, plain)
    for group in (0, 7):
        out = np.full((20, p.plimbs), SENTINEL, dtype=np.uint64)
        with pytest.raises(Unsatisfiable, match=f"^proof 3: constraint {want[3].first_unsatisfied} unsatisfied"):
            g.prove_batch_raw(20, r, s, zs.ctypes.data, group, CHECK_WITNESS, out)
        for k in range(20):
            assert np.array_equal(out[k], np.zeros(p.plimbs, dtype=np.uint64) if k in bad else plain[k]), k
    assert np.array_equal(plain[0], orc.prove(g.curve.cid, g.nq, p.pk, p.m, zs[0], r[0], s[0], threads=8)[0])


# ---- 8. many proofs per call -------------------------------------------------------------------------------------------
def test_65541_assignments():
    g = engine("bn254")
    m, z, _ = synthetic_r1cs("bn254", 4, seed=4)
    g.load_matrices(m)
    rows = csr_rows(g, m)
    nv = z.shape[0]
    fr = g.codec.fr
    pattern = [z, bumped(g, z, [int(m.c[1][2])]), bumped(g, z, [nv - 1]), bumped(g, z, [2, 3, 4]), z.copy(), z.copy(), z]
    pattern[4][0] = np.zeros(fr.nl, dtype=np.uint64)
    pattern[5][nv - 1] = ints_to_limbs([fr.p], fr.nl)[0]
    want = [oracle(g, rows, zk) for zk in pattern]
    assert len({(w.first_unsatisfied, w.num_unsatisfied, w.first_malformed) for w in want}) == 6
    count = 65541
    zs = np.ascontiguousarray(np.stack(pattern)[np.arange(count) % 7])
    got = reports(g, zs)
    assert len(got) == count
    assert all(got[k] == want[k % 7] for k in range(count))
    import torch
    dz = torch.from_numpy(zs.view(np.int64).reshape(-1)).to("cuda:0")
    torch.cuda.synchronize()
    got = reports(g, dz.data_ptr(), count=count, flags=_lib.ASSIGNMENT_ON_DEVICE)
    assert all(got[k] == want[k % 7] for k in range(count))


# ---- 9. CircomReduction ------------------------------------------------------------------------------------------------
def test_circom_reduction_reads_c_only_with_the_flag():
    curve = "bls12_381"
    c = P.CURVES[curve]
    cs = P.synthetic_circuit(c, 60, seed=21, num_inputs=1)
    g = engine(curve, "circom")
    m = ConstraintMatrices.from_rows(curve, cs.num_instance, cs.num_witness, cs.a, cs.b, cs.c)
    G = GENERATORS[curve]
    pk = g.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=True)
    z = np.ascontiguousarray(g.codec.fr.enc(cs.assignment))
    col = [j for j in c_only_columns(m) if j >= cs.num_instance][-1]
    bad = bumped(g, z, [col])
    want = oracle(g, csr_rows(g, m), bad)
    assert want.num_unsatisfied == 1
    assert reports(g, bad) == [want]
    cd = g.codec
    vk = P.VerifyingKey(cd.dec_g1(pk.vk.alpha_g1)[0], cd.dec_g2(pk.vk.beta_g2)[0], cd.dec_g2(pk.vk.gamma_g2)[0],
                        cd.dec_g2(pk.vk.delta_g2)[0], cd.dec_g1(pk.vk.gamma_abc_g1))
    pub = cs.assignment[1:cs.num_instance]
    r, s = cd.fr.enc1(5), cd.fr.enc1(6)
    prove = lambda zz, flags: g.create_proof_with_reduction_and_matrices(None, r, s, None, m.num_instance_variables,
                                                                         m.num_constraints, zz, flags)
    assert P.verify_proof(vk, c, P.Proof(cd.dec_g1(prove(z, 0).a)[0], cd.dec_g2(prove(z, 0).b)[0],
                                         cd.dec_g1(prove(z, 0).c)[0]), pub)
    pf = prove(bad, 0)   # today's behaviour: proved without a word
    assert not P.verify_proof(vk, c, P.Proof(cd.dec_g1(pf.a)[0], cd.dec_g2(pf.b)[0], cd.dec_g1(pf.c)[0]), pub)
    with pytest.raises(Unsatisfiable, match=f"constraint {want.first_unsatisfied} unsatisfied"):
        prove(bad, CHECK_WITNESS)


# ---- 10. bad arguments -------------------------------------------------------------------------------------------------
def test_bad_arguments():
    lib = _lib.load()
    fresh = Groth16("bn254", 0)
    try:
        rep = (_lib.WitnessReport * 1)()
        z = np.zeros((4, 4), dtype=np.uint64)
        assert lib.g16_check_witness(fresh._ctx, 1, z.ctypes.data, 0, rep) == _lib.ERR_BAD_ARGUMENT   # no circuit
    finally:
        fresh.close()
    p = Prover("bn254")
    g, z = p.g, p.z
    rep = (_lib.WitnessReport * 2)()
    sentinel = _lib.WitnessReport(7, 7, 7)
    rep[0] = sentinel
    for flags in (_lib.SERIAL_MSMS, CHECK_WITNESS, 8, 1 << 31):
        assert lib.g16_check_witness(g._ctx, 1, z.ctypes.data, flags, rep) == _lib.ERR_BAD_ARGUMENT
    assert lib.g16_check_witness(g._ctx, 1, None, 0, rep) == _lib.ERR_BAD_ARGUMENT
    assert lib.g16_check_witness(g._ctx, 1, z.ctypes.data, 0, None) == _lib.ERR_BAD_ARGUMENT
    assert lib.g16_check_witness(None, 1, z.ctypes.data, 0, rep) == _lib.ERR_BAD_ARGUMENT
    assert lib.g16_check_witness(g._ctx, 0, None, 0, None) == _lib.G16_OK
    assert lib.g16_check_witness(g._ctx, 0, z.ctypes.data, 0, rep) == _lib.G16_OK
    assert (rep[0].first_unsatisfied, rep[0].num_unsatisfied, rep[0].first_malformed) == (7, 7, 7)
    r, s = p.rs(1)
    g.prove_submit_raw(0, r[0], s[0], z.ctypes.data, 0)
    assert lib.g16_check_witness(g._ctx, 1, z.ctypes.data, 0, rep) == _lib.ERR_BAD_ARGUMENT   # slot 0 in flight
    out = np.zeros(p.plimbs, dtype=np.uint64)
    g.prove_wait_raw(0, out)
    assert lib.g16_check_witness(g._ctx, 1, z.ctypes.data, 0, rep) == _lib.G16_OK
    assert rep[0].first_malformed == _lib.NONE and rep[0].num_unsatisfied == 0


# ---- 11. sharded proofs over NCCL ---------------------------------------------------------------------------------------
def _ngpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def test_sharded_refusal_keeps_collectives_matched():
    n = min(_ngpus(), 4)
    if n < 2:
        pytest.skip("needs at least 2 GPUs (the in-library exchange is NCCL between processes)")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(ROOT, "tools", "sharded_witness_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and f"SHARDED_CHECK_OK world={n}" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
