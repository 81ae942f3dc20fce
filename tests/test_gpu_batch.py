"""GPU tier of batch proving (g16_prove_batch / Groth16.create_proofs_batch; run on an H100 with `pytest -m gpu`).

Every proof of a batch must equal, bit for bit as raw limbs, g16_prove of the same (r, s, assignment): per curve on a 2^12
synthetic circuit (some proofs also against the CPU oracle, one pairing-verified), across group boundaries, slot counts and
G16_SERIAL_MSMS, with edge rows (r = 0, s = 0, r = s, an all-zero assignment, repeated rows, a constant witness), on the
c = 16 / batched-affine path of a 2^17 circuit, from a device buffer, and on every error path.  Against the CPU oracle, the
geometries only a batch reaches: rounds a group switches on, the three-pass NTT with several vectors per launch, a group
of 65535 proofs on grid y, device assignments over several groups, and residency plans changed between batch calls
(geometries the matrix of test_gpu_geometry.py runs in batches are there).  The assignments need not
satisfy the circuit: the library and the oracle compute the same deterministic function of them either way."""
import random

import numpy as np
import pytest

import orc
import pyref as P
from groth16_b200 import Groth16, _lib
from groth16_b200.params import GENERATORS
from groth16_b200.workload import synthetic_r1cs
from util import ALL_CURVES, pk_from_abi, proof_from_abi

pytestmark = pytest.mark.gpu

TOXIC = (0x1111111111111111111111, 0x2222222222222222222223, 0x3333333333333333333335, 0x4444444444444444444447,
         0x5555555555555555555559)
THREADS = 16


class Ctx:
    def __init__(self, curve, log_n, seed):
        self.curve = curve
        self.g = Groth16(curve, 0)
        self.cd = self.g.codec
        G = GENERATORS[curve]
        self.m, self.z, self.pub = synthetic_r1cs(curve, log_n, seed=seed)
        self.pk = self.g.generate_parameters_with_qap(self.m, *TOXIC, G["g1"], G["g2"], export=True)
        self.nv = self.m.num_instance_variables + self.m.num_witness_variables
        self.rng = random.Random(seed)

    def fr(self, xs):
        return np.ascontiguousarray(self.cd.fr.enc([x % self.g.curve.r for x in xs]), dtype=np.uint64).reshape(-1, 4)

    def rows(self, count):
        """(r, s, z) of `count` proofs: random scalars and random (unsatisfying) assignments with z[0] = 1"""
        r = self.fr([self.rng.randrange(self.g.curve.r) for _ in range(count)])
        s = self.fr([self.rng.randrange(self.g.curve.r) for _ in range(count)])
        z = np.empty((count, self.nv, 4), dtype=np.uint64)
        for k in range(count):
            z[k] = self.fr([1] + [self.rng.randrange(self.g.curve.r) for _ in range(self.nv - 1)])
        return r, s, z

    def single(self, r, s, z, flags=0):
        out = np.zeros(8 * self.g.nq, dtype=np.uint64)
        self.g.prove_raw(np.ascontiguousarray(r), np.ascontiguousarray(s), np.ascontiguousarray(z).ctypes.data, flags, out)
        return out

    def batch(self, r, s, z, group=0, flags=0):
        return np.stack([np.concatenate([p.a, p.b, p.c]) for p in self.g.create_proofs_batch(r, s, z, group=group, flags=flags)])

    def oracle(self, r, s, z):
        return orc.prove(self.g.curve.cid, self.g.nq, self.pk, self.m, z, r, s, threads=THREADS)[0]


_CTX = {}


def ctx(curve, log_n=12) -> Ctx:
    key = (curve, log_n)
    if key not in _CTX:
        _CTX[key] = Ctx(curve, log_n, seed=31 + log_n)
    return _CTX[key]


@pytest.fixture(scope="module", autouse=True)
def _contexts():
    yield
    for c in _CTX.values():
        c.g.close()
    _CTX.clear()


def assert_singles(c, r, s, z, got, flags=0):
    for k in range(len(r)):
        assert np.array_equal(got[k], c.single(r[k], s[k], z[k], flags)), (c.curve, k)


@pytest.mark.parametrize("curve", ALL_CURVES)
def test_batch_equals_single_and_oracle(curve):
    c = ctx(curve)
    for count in (1, 2, 7, 33):
        r, s, z = c.rows(count)
        if count == 7:
            z[3] = c.z   # the circuit's own satisfying assignment
        got = c.batch(r, s, z)
        assert got.shape == (count, 8 * c.g.nq)
        assert_singles(c, r, s, z, got)
        for k in sorted({0, count // 2, count - 1}):
            assert np.array_equal(got[k], c.oracle(r[k], s[k], z[k])), (curve, count, k)
        if count == 7:   # the satisfying row verifies under the pairing, and not for another public input
            vk = pk_from_abi(curve, c.pk).vk
            pf = proof_from_abi(curve, c.g.create_proofs_batch(r[3:4], s[3:4], z[3:4])[0])
            cur = P.CURVES[curve]
            assert P.verify_proof(vk, cur, pf, list(c.pub))
            assert not P.verify_proof(vk, cur, pf, [(c.pub[0] + 1) % cur.r])


def test_group_boundaries_slots_and_serial():
    c = ctx("bls12_381")
    r, s, z = c.rows(9)
    want = c.batch(r, s, z, group=1)
    assert_singles(c, r, s, z, want)
    for group in (2, 4, 9, 0):
        assert np.array_equal(c.batch(r, s, z, group=group), want), group
    slots = c.g.get_option("proof_slots")
    try:
        c.g.set_option("proof_slots", 1)
        for group in (2, 0):
            assert np.array_equal(c.batch(r, s, z, group=group), want), ("one slot", group)
    finally:
        c.g.set_option("proof_slots", slots)
    assert np.array_equal(c.batch(r, s, z, group=4, flags=_lib.SERIAL_MSMS), want)


@pytest.mark.parametrize("curve", ALL_CURVES)
def test_edge_rows(curve):
    c = ctx(curve)
    r, s, z = c.rows(8)
    fr = lambda x: c.fr([x])[0]
    r[0] = fr(0)                 # r = 0: B in G1 drops out (prover.rs:98)
    s[1] = fr(0)
    r[2] = s[2]
    r[3], s[3] = fr(0), fr(0)
    z[4] = 0                     # all-zero assignment: every MSM is the identity
    z[6] = z[5]                  # two identical rows
    r[6], s[6] = r[5], s[5]
    z[7] = c.fr([1] + [0x1234567] * (c.nv - 1))   # constant witness: one bucket per window
    got = c.batch(r, s, z)
    assert_singles(c, r, s, z, got)
    assert np.array_equal(got[5], got[6])
    assert np.array_equal(got[4], c.oracle(r[4], s[4], z[4]))


@pytest.mark.parametrize("curve", ["bls12_381", "bn254"])
def test_c16_batched_affine_path(curve):
    c = ctx(curve, 17)
    r, s, z = c.rows(4)
    want = [c.single(r[k], s[k], z[k]) for k in range(4)]
    ba, share = c.g.get_option("msm_ba"), c.g.get_option("share_b_sort")
    assert c.g.config()["c"] == 16
    try:
        for rounds in (0, ba):
            for sh in (0, 1):
                c.g.set_option("msm_ba", rounds)
                c.g.set_option("share_b_sort", sh)
                got = c.batch(r, s, z)
                for k in range(4):
                    assert np.array_equal(got[k], want[k]), (curve, rounds, sh, k)
    finally:
        c.g.set_option("msm_ba", ba)
        c.g.set_option("share_b_sort", share)


def test_assignments_on_device():
    import torch
    c = ctx("bn254")
    r, s, z = c.rows(5)
    want = c.batch(r, s, z)
    dz = torch.from_numpy(z.view(np.int64).reshape(-1)).to("cuda:0")
    torch.cuda.synchronize()
    out = np.zeros((5, 8 * c.g.nq), dtype=np.uint64)
    c.g.prove_batch_raw(5, r, s, dz.data_ptr(), 0, _lib.ASSIGNMENT_ON_DEVICE, out)
    assert np.array_equal(out, want)


def test_errors_and_state_after_a_batch():
    c = ctx("bls12_381")
    g = c.g
    r, s, z = c.rows(3)
    # single-proof paths before any batch on this key
    one = c.single(r[0], s[0], z[0])
    pair = np.zeros((2, 8 * g.nq), dtype=np.uint64)
    got = c.batch(r, s, z)
    t = g.timings()
    c.single(r[1], s[1], z[1])   # r != 0: every MSM runs
    assert t["msm_pairs"] == {k: 3 * v for k, v in g.timings()["msm_pairs"].items()}
    assert t["launches"] > 0 and t["total_ms"] > 0
    # count 0: OK, nothing touched
    sentinel = np.full((1, 8 * g.nq), 7, dtype=np.uint64)
    g.prove_batch_raw(0, r, s, z.ctypes.data, 0, 0, sentinel)
    assert (sentinel == 7).all()
    # null pointers
    for args in ((None, s, z), (r, None, z), (r, s, None)):
        rr, ss, zz = args
        rc = g._lib.g16_prove_batch(g._ctx, 3, None if rr is None else rr.ctypes.data, None if ss is None else ss.ctypes.data,
                                    None if zz is None else zz.ctypes.data, 0, 0, sentinel.ctypes.data)
        assert rc == _lib.ERR_BAD_ARGUMENT
    assert g._lib.g16_prove_batch(g._ctx, 1, r.ctypes.data, s.ctypes.data, z.ctypes.data, 0, 0, None) == _lib.ERR_BAD_ARGUMENT
    # a proof in flight: the batch is refused and the proof in flight comes out intact
    r0, s0, z0 = np.ascontiguousarray(r[0]), np.ascontiguousarray(s[0]), np.ascontiguousarray(z[0])
    g.prove_submit_raw(1, r0, s0, z0.ctypes.data, 0)
    with pytest.raises(ValueError):
        g.create_proofs_batch(r, s, z)
    out = np.zeros(8 * g.nq, dtype=np.uint64)
    g.prove_wait_raw(1, out)
    assert np.array_equal(out, one)
    # after a batch: g16_prove and a two-slot pipelined pair give their earlier bytes
    assert np.array_equal(c.single(r[0], s[0], z[0]), one)
    keep = [(np.ascontiguousarray(r[k]), np.ascontiguousarray(s[k]), np.ascontiguousarray(z[k])) for k in range(2)]
    for k in range(2):
        g.prove_submit_raw(k, keep[k][0], keep[k][1], keep[k][2].ctypes.data, 0)
    for k in range(2):
        g.prove_wait_raw(k, pair[k])
    assert np.array_equal(pair[0], got[0]) and np.array_equal(pair[1], got[1])
    # a sharded key is refused
    g.load_proving_key(c.pk, 0, 2)
    try:
        with pytest.raises(ValueError):
            g.create_proofs_batch(r, s, z)
    finally:
        g.load_proving_key(c.pk)
    assert np.array_equal(c.batch(r, s, z), got)   # the tail tables are rebuilt for the re-loaded key


# ---- geometries only a batch reaches -------------------------------------------------------------------------------------
def alone_entries(c, r, s, z):
    """rows' msm_entries summed over single proofs; a row with r = 0 is counted with r = 1 (a single proof skips B in G1,
    and with it the shared B sort, when r = 0; its entries do not depend on r)"""
    one = c.fr([1])[0]
    total = {}
    for k in range(len(r)):
        c.single(r[k] if r[k].any() else one, s[k], z[k])
        for n, v in c.g.timings()["msm_entries"].items():
            total[n] = total.get(n, 0) + v
    return total


def options(g, **opts):
    saved = {k: g.get_option(k) for k in opts}
    for k, v in opts.items():
        g.set_option(k, v)
    return saved


ROUNDS = [dict(ba_adaptive=1), dict(ba_adaptive=0)] + [dict(ba_adaptive=0, msm_ba=r, msm_ba_g2=r) for r in range(1, 7)]


@pytest.mark.parametrize("curve", ALL_CURVES)
@pytest.mark.parametrize("log_n,count", [(8, 20), (10, 8), (14, 3)])
def test_rounds_switched_on_by_the_group(curve, log_n, count):
    """at 2^8 and 2^10 one proof has fewer than 2^18 MSM entries and runs no batched-affine rounds; `count` of them in one
    group cross 2^18 (ba_min_entries 0) and do, with bucket padding per proof's bucket sets (at 2^14 one proof already runs
    them, and the group the same count).  Adaptive and forced 1 .. 6 rounds, one group and groups of 2: every proof against
    the oracle, and the sorted slots against the rows' single-proof sum"""
    c = ctx(curve, log_n)
    r, s, z = c.rows(count)
    r[1] = c.fr([0])[0]
    z[count // 2, 1:] = c.fr([0x9e3779b])[0]       # constant witness: one giant bucket per window
    want = np.stack([c.oracle(r[k], s[k], z[k]) for k in range(count)])
    for opts in ROUNDS:
        saved = options(c.g, ba_min_entries_g1=0, ba_min_entries_g2=0, **opts)
        try:
            alone = alone_entries(c, r, s, z)
            for group in (0, 2):
                out = np.zeros((count, 8 * c.g.nq), dtype=np.uint64)
                c.g.prove_batch_raw(count, r, s, z.ctypes.data, group, 0, out)
                for k in range(count):
                    assert np.array_equal(out[k], want[k]), (curve, log_n, opts, group, k)
                entries = c.g.timings()["msm_entries"]
                if log_n < 14 and group == 0:   # the group pads its buckets for rounds a single proof never runs
                    assert entries["h"] > alone["h"], (curve, log_n, opts, entries, alone)
                else:   # groups of 2 stay under 2^18 entries; at 2^14 one proof runs the group's rounds itself
                    assert entries == alone, (curve, log_n, opts, group, entries, alone)
        finally:
            options(c.g, **saved)


@pytest.mark.parametrize("curve", ["bls12_381", "bn254"])
def test_three_pass_ntt_with_vstride(curve):
    """a 2^18 domain takes the three-pass NTT plan; with 3 proofs per group every pass selects the proof's vector by
    blockIdx.y (NttPass::vstride).  One group of 3, and groups of 2 and 1"""
    c = ctx(curve, 18)
    r, s, z = c.rows(3)
    want = [c.oracle(r[k], s[k], z[k]) for k in range(3)]
    for group in (0, 2):
        got = c.batch(r, s, z, group=group)
        for k in range(3):
            assert np.array_equal(got[k], want[k]), (curve, group, k)


def test_grid_y_cap():
    """65541 proofs with group 100000: the library clamps the group to 65535 (grid y), so one group of 65535 and one of 6.
    Rows repeat with period 7 (coprime to 65535 and to powers of two): a proof index that wraps at 2^15, 2^16 or 65535
    lands on a row with other contents.  Proof k must equal proof k mod 7, and the 7 distinct proofs g16_prove's and the
    oracle's"""
    import resource
    import time
    c = ctx("bn254", 3)
    period, count = 7, 65541
    assert count % period == 0
    r7, s7, z7 = c.rows(period)
    r7[3] = c.fr([0])[0]
    t0 = time.perf_counter()
    reps = count // period
    r, s = np.ascontiguousarray(np.tile(r7, (reps, 1))), np.ascontiguousarray(np.tile(s7, (reps, 1)))
    z = np.ascontiguousarray(np.tile(z7, (reps, 1, 1)))
    out = np.zeros((count, 8 * c.g.nq), dtype=np.uint64)
    c.g.prove_batch_raw(count, r, s, z.ctypes.data, 100000, 0, out)
    wall = time.perf_counter() - t0
    pairs = c.g.timings()["msm_pairs"]
    assert (out.reshape(reps, period, -1) == out[None, :period]).all()
    for k in range(period):
        one = c.single(r7[k], s7[k], z7[k])
        if k == 0:   # every MSM of every proof ran (B in G1 too: a batch runs it whatever r is)
            assert pairs == {n: count * v for n, v in c.g.timings()["msm_pairs"].items()}
        assert np.array_equal(out[k], one), k
        assert np.array_equal(one, c.oracle(r7[k], s7[k], z7[k])), k
    print(f"grid-y cap: {count} proofs in {wall:.1f} s, peak host RSS {resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20:.2f} GiB")


def test_assignments_on_device_over_groups():
    import torch
    c = ctx("bls12_381")
    r, s, z = c.rows(7)
    want = c.batch(r, s, z)
    dz = torch.from_numpy(z.view(np.int64).reshape(-1)).to("cuda:0")
    torch.cuda.synchronize()
    for group in (3, 1):
        out = np.zeros((7, 8 * c.g.nq), dtype=np.uint64)
        c.g.prove_batch_raw(7, r, s, dz.data_ptr(), group, _lib.ASSIGNMENT_ON_DEVICE, out)
        assert np.array_equal(out, want), group


@pytest.mark.parametrize("curve", ["bn254", "bls12_377"])
def test_plan_change_between_batches(curve):
    """batch under msm_ne 1, re-load the key under msm_ne 8, then 0, and batch again on the same context: the slots keep
    their grown workspaces and tail buffers across the plans (other bucket-set counts per proof, other copies)"""
    c = ctx(curve)
    r, s, z = c.rows(5)
    want = np.stack([c.oracle(r[k], s[k], z[k]) for k in range(5)])
    ne0 = c.g.get_option("msm_ne")
    seen = []
    try:
        for ne in (1, 8, 0):
            c.g.set_option("msm_ne", ne)
            c.g.load_proving_key(c.pk)
            seen.append((c.g.config()["ne"], c.g.config()["copies"]))
            for group in (0, 2):
                assert np.array_equal(c.batch(r, s, z, group=group), want), (curve, ne, group)
    finally:
        c.g.set_option("msm_ne", ne0)
        c.g.load_proving_key(c.pk)
    assert len(set(seen)) == 3, seen
