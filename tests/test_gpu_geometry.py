"""GPU parity over every MSM geometry the prover can run (run on an H100 with `pytest -m gpu`).

The tuning knobs of include/g16b200.h change speed, never results.  test_gpu_production.py checks that for the default
single-GPU plan only (c = 16, one bucket set, 16 precomputed multiples, equal batched-affine rounds on G1 and G2).  Here one
2^17-constraint key per curve (every query >= 2^16 pairs, so c = 16 is chosen; one curve's engine open at a time) and ONE oracle proof per curve serve a matrix
of residency plans, uneven rounds, accumulation knobs, schedules and sharded keys: every configuration re-loads the key,
asserts through g16_get_config that the geometry it asked for was reached, proves, and must match the oracle bit for bit.
Each matrix test has a `_batch` twin that proves K = 3 rows per curve in one g16_prove_batch instead (one group, then
groups of 2 and 1), each against its own oracle proof, with the batch's sorted slots equal to the rows' single-proof sum.
Further: adversarial bases (duplicates, opposite pairs, identity runs) and signed-digit edge scalars at the resident
geometry, partial MSMs against the oracle's msm_bigint; the stand-alone g16_msm_g1 / g2 at c = 12 .. 16 and c = 17 / 20.

The three pairing curves are checked against the C++ oracle (orc).  BW6-761 has none: with the toxic waste known, every
point of its key is [d]G with d known (bw6_ref.query_exponents), so its proofs come from the closed form and every MSM over
key points, edited ones included, is one scalar multiple of the generator.  Its 377-bit scalars need W = 24 windows at
c = 16, above the 20-copy cap, so it is the curve whose default plan is raised to ne = 2."""
import contextlib
from dataclasses import dataclass

import numpy as np
import pytest

import bw6_ref as ref
import orc
import pyref as P
from groth16_b200 import Groth16, _lib
from groth16_b200.codec import limbs_to_ints
from groth16_b200.params import GENERATORS
from groth16_b200.workload import synthetic_r1cs
from util import ALL_CURVES

pytestmark = pytest.mark.gpu

LOG_N = 17
TOXIC = (0x1111111111111111111111, 0x2222222222222222222223, 0x3333333333333333333335, 0x4444444444444444444447,
         0x5555555555555555555559)
THREADS = 16
OPTIONS = ("msm_ne", "msm_c", "msm_maxcopies", "msm_ba", "msm_ba_g2", "ba_adaptive", "ba_min_entries_g1", "ba_min_entries_g2",
           "acc_k0_g1", "acc_k0_g2", "acc_block", "share_b_sort", "wm_first", "proof_slots")
M_H, M_L, M_A, M_B1, M_B2 = range(5)
MSMS = ("h", "l", "a", "b_g1", "b_g2")
BW6 = "bw6_761"
CURVES = ALL_CURVES + [BW6]


# ---- the launch geometry the library should pick (Engine::pick_geom / with_k0, msm_geom, msm_pick_k0) -----------------
def _pick_c(n):
    return min(max((n - 1).bit_length() - 4, 3), 16)


def _geom(n, bits, c, ne):
    c = c if c > 0 else _pick_c(n)
    w = (bits + c) // c
    ne = w if (ne <= 0 or ne > w) else ne
    return dict(c=c, W=w, ne=ne, copies=-(-w // ne), nkeys=ne << (c - 1), entries=n * w)


def _resident_geom(n, bits, o):
    if o["msm_ne"] <= 0:
        return _geom(n, bits, o["msm_c"], 0)
    c = o["msm_c"] if o["msm_c"] > 0 else (16 if n >= 1 << 16 else 0)
    ne = o["msm_ne"]
    g = _geom(n, bits, c, ne)
    while g["copies"] > o["msm_maxcopies"]:
        ne += 1
        g = _geom(n, bits, c, ne)
    return g


def _k0(g, sm_count, g2, o):
    k0, kmin = 64, (16 if g2 else 8)
    while k0 > kmin and g["entries"] // k0 < sm_count * 128 * (2 if g2 else 3) * 2:
        k0 >>= 1
    if g2 and k0 > 32:
        k0 = 32
    k = o["acc_k0_g2" if g2 else "acc_k0_g1"]
    return k if 4 <= k <= 1024 else k0


def _rounds(g, g2, o):
    r = o["msm_ba_g2" if g2 else "msm_ba"]
    fit, per = 0, g["entries"] // g["nkeys"]
    while (11 << fit) < per:
        fit += 1
    if not o["ba_adaptive"]:
        fit = r
    big = g["entries"] >= max(1 << 18, o["ba_min_entries_g2" if g2 else "ba_min_entries_g1"])
    return min(r, fit, 6) if r > 0 and big else 0


# ---- per-curve state: one engine, one key, one oracle proof ----------------------------------------------------------------
@dataclass
class Case:
    curve: str
    g: Groth16
    m: object
    z: np.ndarray
    pk: object
    r: np.ndarray
    s: np.ndarray
    want: np.ndarray
    defaults: dict
    config0: dict
    oracle: object = None    # CppOracle or Bw6Oracle of the module key
    rows: tuple = None       # (r, s, z) of the K batch rows, row 0 = (r, s, z) above
    wants: np.ndarray = None  # their oracle proofs

    @property
    def bits(self):
        return self.g.curve.r.bit_length()

    @property
    def pw(self):
        """u64 words of one proof: A (G1) || B (G2) || C (G1)"""
        return 4 * self.g.nq + self.g.ng2

    def pairs(self, rank=0, world=1):
        """(H, B2) pairs owned by `rank`: H has domain - 1 pairs, B-in-G2 one per variable but the constant One"""
        nv = self.m.num_instance_variables + self.m.num_witness_variables
        own = lambda n: (n - rank + world - 1) // world
        return own((1 << LOG_N) - 1), own(nv - 1)

    def expected(self, opts, rank=0, world=1):
        o = dict(self.defaults, **opts)
        nh, nb = self.pairs(rank, world)
        gh, gb = _resident_geom(nh, self.bits, o), _resident_geom(nb, self.bits, o)
        sm = self.config0["sm_count"]
        return dict(c=gh["c"], ne=gh["ne"], copies=gh["copies"], k0_g1=_k0(gh, sm, False, o), k0_g2=_k0(gb, sm, True, o),
                    ba_rounds_g1=_rounds(gh, False, o), ba_rounds_g2=_rounds(gb, True, o))


def _ints(cd, limbs):
    """Montgomery Fr limbs (one element or rows) -> ints"""
    return cd.fr.dec(np.asarray(limbs).reshape(-1, cd.fr.nl))


def _edited(d, edit):
    """copies of the key's discrete logs with `edit(array, neg)` applied to each query, as to the key's points"""
    out = {k: v.copy() for k, v in d.items()}
    for v in out.values():
        edit(v, lambda x: (-x) % ref.R)
    return out


class CppOracle:
    """The three pairing curves: the C++ oracle's prover and msm_bigint over the key's points"""

    def __init__(self, cs, pk):
        self.cs, self.pk = cs, pk
        cd = cs.g.codec
        self.cid, self.nq = cd.c.cid, cd.nq

    def for_key(self, pk, edit):
        return CppOracle(self.cs, pk)

    def proof(self, z, r, s):
        return orc.prove(self.cid, self.nq, self.pk, self.cs.m, z, r, s, threads=THREADS)[0]

    def partials(self, z):
        """the five MSMs of a partial proof (H, L, A, B in G1, B in G2) as affine words, the identity all zero"""
        cs, pk, cid, nq = self.cs, self.pk, self.cid, self.nq
        cd = cs.g.codec
        ni = cs.m.num_instance_variables
        nv = ni + cs.m.num_witness_variables
        zc = cd.fr.bigint(cd.fr.dec(z))
        h = orc.witness_map(cid, cs.m, z, threads=THREADS)
        ws = [orc.msm_g1(cid, nq, pk.h_query, cd.fr.bigint(cd.fr.dec(h)), THREADS),
              orc.msm_g1(cid, nq, pk.l_query, zc[ni:], THREADS),
              orc.msm_g1(cid, nq, pk.a_query.reshape(nv, -1)[1:], zc[1:], THREADS),
              orc.msm_g1(cid, nq, pk.b_g1_query.reshape(nv, -1)[1:], zc[1:], THREADS),
              orc.msm_g2(cid, nq, pk.b_g2_query.reshape(nv, -1)[1:], zc[1:], THREADS)]
        out = []
        for k, w in enumerate(ws):
            width = (4 if k == M_B2 else 2) * nq
            out.append(w[:width] if w[width:].any() else np.zeros(width, dtype=np.uint64))   # projective Z = 0: identity
        return out

    def check_msm(self, got, tile, sc, g2):
        """`tile(src, neg)` builds the bases from an array of the key's points (see _msm_inputs)"""
        bases = tile(*_msm_source(self.cs, g2))
        want = (orc.msm_g2 if g2 else orc.msm_g1)(self.cid, self.nq, bases, sc, THREADS)
        assert np.array_equal(got, want)


class Bw6Oracle:
    """BW6-761: the key's discrete logs d from the toxic waste (bw6_ref.query_exponents), edited like its points.  Proofs on
    the module key come from the O(n) closed form (bw6_ref.proof_exponents, any assignment); on an edited key from its five
    MSMs as d-dot-products, with h from bw6_ref's witness map.  An MSM over key points is [sum s_i d_i] G."""

    def __init__(self, cs, d=None, rows=None):
        self.cs = cs
        m = cs.m
        self.ni = m.num_instance_variables
        self.nv = self.ni + m.num_witness_variables
        self.rows = ref.csr_rows(m) if rows is None else rows
        self.edited = d is not None
        if d is None:
            alpha, beta, _gamma, delta, tau = TOXIC
            q = ref.query_exponents(self.rows, self.ni, self.nv, alpha, beta, delta, tau)
            d = {k: np.array(q[k], dtype=object) for k in ("a", "l", "h")}
            d["b_g1"], d["b_g2"] = np.array(q["b"], dtype=object), np.array(q["b"], dtype=object)
        self.d = d
        self.gen = GENERATORS[BW6]
        self._h = {}

    def for_key(self, pk, edit):
        return Bw6Oracle(self.cs, _edited(self.d, edit), self.rows)

    def _enc(self, pts):
        cd = self.cs.g.codec
        return [cd.enc_g2([p])[0] if g2 else cd.enc_g1([p])[0] for p, g2 in pts]

    def _msms(self, z):
        """the MSM exponents over this key for the assignment z (ints)"""
        key = tuple(z)
        if key not in self._h:
            self._h[key] = ref.witness_map(*ref.row_evals(self.rows, self.ni, z))
        return ref.msm_exponents(self.d, self._h[key], z, self.ni)

    def proof(self, z, r, s):
        cd = self.cs.g.codec
        z, (r,), (s,) = _ints(cd, z), _ints(cd, r), _ints(cd, s)
        alpha, beta, _gamma, delta, tau = TOXIC
        if self.edited:
            d0 = (self.d["a"][0], self.d["b_g1"][0], self.d["b_g2"][0])
            a_s, b_s, c_s = ref.proof_from_msms(self._msms(z), d0, alpha, beta, delta, r, s)
        else:
            a_s, b_s, c_s = ref.proof_exponents(self.rows, self.ni, z, alpha, beta, delta, tau, r, s)
        g1, g2 = self.gen["g1"], self.gen["g2"]
        return np.concatenate(self._enc([(ref.mul_proj(a_s, g1), False), (ref.mul_proj(b_s, g2), True),
                                         (ref.mul_proj(c_s, g1), False)]))

    def partials(self, z):
        e = self._msms(_ints(self.cs.g.codec, z))
        return self._enc([(ref.mul_proj(e[k], self.gen["g2" if k == "b_g2" else "g1"]), k == "b_g2") for k in MSMS])

    def check_msm(self, got, tile, sc, g2):
        cd = self.cs.g.codec
        d = tile(np.concatenate([self.d["h"], self.d["l"]]) if not g2 else self.d["b_g2"], lambda x: (-x) % ref.R)
        e = sum(k * x for k, x in zip(limbs_to_ints(sc, cd.fr.nl), d)) % ref.R
        want = ref.mul_proj(e, self.gen["g2" if g2 else "g1"])
        assert (cd.dec_proj_g2(got) if g2 else cd.dec_proj_g1(got)) == want


_CASES = {}


def _close_engines(keep=None):
    """close the engine of every curve but `keep`, after checking that every configuration restored its knobs; the host
    state (key, oracle, expected proofs) stays.  An engine keeps the high-water mark of its MSM and batch workspaces, up to
    ~20 GB for BW6-761 here: with all four curves' engines open, the free memory falls below what decide_ba_memory needs to
    grant the batched-affine rounds, and the geometry asked for is not the one reached.  So one engine is open at a time;
    the curve parameter is module-scoped, so that pytest runs each test's configurations curve by curve and an engine is
    re-opened about 70 times per module run instead of at nearly every test."""
    for cs in _CASES.values():
        if cs.curve != keep and cs.g is not None:
            try:
                assert {k: cs.g.get_option(k) for k in OPTIONS} == cs.defaults, cs.curve
            finally:
                cs.g.close()
                cs.g = None


def case(curve) -> Case:
    _close_engines(keep=curve)
    if curve in _CASES:
        cs = _CASES[curve]
        if cs.g is None:                   # re-open: a fresh context with the module's circuit and key resident
            cs.g = Groth16(curve, 0)
            cs.g.load_matrices(cs.m)
            cs.g.load_proving_key(cs.pk)
            assert {k: cs.g.get_option(k) for k in OPTIONS} == cs.defaults
        return cs
    g = Groth16(curve, 0)
    defaults = {k: g.get_option(k) for k in OPTIONS}
    cd = g.codec
    G = GENERATORS[curve]
    m, z, _ = synthetic_r1cs(curve, LOG_N, seed=21)
    g.set_option("msm_ne", 0)          # mint without precomputed multiples (bench.py's big-key flow), export, re-load
    try:
        pk = g.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=True)
    finally:
        g.set_option("msm_ne", defaults["msm_ne"])
    g.load_proving_key(pk)
    r, s = np.ascontiguousarray(cd.fr.enc1(0x1234567 + cd.c.cid)), np.ascontiguousarray(cd.fr.enc1(0x7654321))
    cs = Case(curve, g, m, z, pk, r, s, None, defaults, g.config())
    cs.oracle = Bw6Oracle(cs) if curve == BW6 else CppOracle(cs, pk)
    cs.want = cs.oracle.proof(z, r, s)
    cs.rows = batch_rows(cs)
    R, S, Z = cs.rows
    cs.wants = np.stack([cs.want] + [cs.oracle.proof(Z[k], R[k], S[k]) for k in range(1, K)])
    _CASES[curve] = cs
    return cs


K = 3   # batch rows per curve


def batch_rows(cs):
    """K rows that stress the bucket-set layout of a batch: row 0 is the module's (r, s, z); row 1 has a constant witness
    below 2^32 (one giant bucket per window, and with ne > 1 empty high bucket sets between its neighbours' sets); row 2 has
    r = 0 and runs of zero witness entries.  Rows 1 and 2 come from a fixed seed."""
    cd = cs.g.codec
    rr = np.random.RandomState(41)
    rnd = lambda: int.from_bytes(rr.bytes(32), "little") % cd.c.r
    z0 = cs.z
    nv = z0.shape[0]
    R = np.stack([cs.r, cd.fr.enc1(rnd()), cd.fr.enc1(0)]).astype(np.uint64)
    S = np.stack([cs.s, cd.fr.enc1(rnd()), cd.fr.enc1(rnd())]).astype(np.uint64)
    z1 = np.ascontiguousarray(np.broadcast_to(cd.fr.enc1(0x9e3779b), (nv, cs.g.nr)))
    z1[0] = cd.fr.enc1(1)
    z2 = np.ascontiguousarray(np.roll(z0, 17, axis=0))
    z2[0] = cd.fr.enc1(1)
    for lo in range(1000, nv - 4000, 9000):
        z2[lo:lo + 4000] = 0
    return np.ascontiguousarray(R), np.ascontiguousarray(S), np.ascontiguousarray(np.stack([z0, z1, z2]))


@pytest.fixture(scope="module", autouse=True)
def _engines():
    yield
    _close_engines()
    _CASES.clear()


@contextlib.contextmanager
def knobs(cs, **opts):
    """set options for one configuration; whatever happens, put back the values the context started with"""
    try:
        for k, v in opts.items():
            cs.g.set_option(k, v)
        yield
    finally:
        for k, v in cs.defaults.items():
            cs.g.set_option(k, v)


def load(cs, opts, rank=0, world=1, pk=None):
    """re-load the key under the current options and check that the intended geometry is what the library runs"""
    cs.g.load_proving_key(cs.pk if pk is None else pk, rank, world)
    cfg = cs.g.config()
    want = cs.expected(opts, rank, world)
    assert {k: cfg[k] for k in want} == want, (cs.curve, opts, rank, world)
    assert (cfg["rank"], cfg["world"]) == (rank, world)
    return cfg


def prove(cs, flags=0):
    m = cs.m
    pf = cs.g.create_proof_with_reduction_and_matrices(None, cs.r, cs.s, None, m.num_instance_variables, m.num_constraints,
                                                        cs.z, flags=flags)
    return np.concatenate([pf.a, pf.b, pf.c])




def single_entries(cs, R, S, Z, flags=0):
    """msm_entries (sorted slots, bucket padding included) of each row proved alone.  Entries do not depend on r, but with
    r = 0 a single proof skips B in G1 and with it the shared B sort: such a row is counted with r = 1."""
    one = cs.g.codec.fr.enc1(1)
    out = np.zeros(cs.pw, dtype=np.uint64)
    total = dict.fromkeys(MSMS, 0)
    for k in range(len(R)):
        r = R[k] if R[k].any() else one
        cs.g.prove_raw(np.ascontiguousarray(r), np.ascontiguousarray(S[k]), Z[k].ctypes.data, flags, out)
        for n, v in cs.g.timings()["msm_entries"].items():
            total[n] += v
    return total


def prove_batch(cs, rows, wants, flags=0, tag=()):
    """all rows in one g16_prove_batch, as one group and in groups of 2 (a group of 2 and a group of 1): every proof equals
    its oracle proof, and the batch's msm_entries equal the rows' single-proof sum, so each proof's bucket sets were sorted
    at the single proof's padding, disjoint from the other proofs' sets"""
    R, S, Z = rows
    alone = single_entries(cs, R, S, Z, flags)
    for group in (0, 2):
        out = np.zeros((len(R), cs.pw), dtype=np.uint64)
        cs.g.prove_batch_raw(len(R), R, S, Z.ctypes.data, group, flags, out)
        for k in range(len(R)):
            assert np.array_equal(out[k], wants[k]), (cs.curve, tag, group, k)
        assert cs.g.timings()["msm_entries"] == alone, (cs.curve, tag, group)


def run_config(curve, opts, check=None, flags=0, batch=False):
    cs = case(curve)
    with knobs(cs, **opts):
        cfg = load(cs, opts)
        if check:
            check(cfg)
        if batch:
            prove_batch(cs, cs.rows, cs.wants, flags, tag=tuple(opts.items()))
        else:
            assert np.array_equal(prove(cs, flags), cs.want), (curve, opts)


# ---- residency plans ------------------------------------------------------------------------------------------------------
RESIDENCY = ([dict(msm_ne=ne) for ne in (0, 1, 2, 3, 5, 8, 16)] +
             [dict(msm_ne=1, msm_maxcopies=mc) for mc in (1, 3)] +
             [dict(msm_ne=1, msm_c=c) for c in (12, 13, 14)])


def _residency_check(curve, opts):
    """literal cross-checks of _resident_geom: W = (bits + c) // c is 16 at c = 16 for the 256-bit scalars, 24 for BW6-761's
    377 bits (above the 20-copy cap, so msm_ne 1 runs ne 2 with 12 copies)"""
    wide = curve == BW6

    def check(cfg):
        if opts.get("msm_ne") == 0:
            assert cfg["copies"] == 1 and cfg["c"] == 13
        elif "msm_maxcopies" in opts:
            ne = ({1: 24, 3: 8} if wide else {1: 16, 3: 6})[opts["msm_maxcopies"]]
            assert cfg["copies"] <= opts["msm_maxcopies"] and cfg["ne"] == ne
        elif "msm_c" in opts:
            want = ({12: (12, 2, 16), 13: (13, 2, 15), 14: (14, 2, 14)} if wide else
                    {12: (12, 2, 11), 13: (13, 1, 20), 14: (14, 1, 19)})[opts["msm_c"]]
            assert (cfg["c"], cfg["ne"], cfg["copies"]) == want
        elif wide:
            assert (cfg["ne"], cfg["copies"]) == {1: (2, 12), 2: (2, 12), 3: (3, 8), 5: (5, 5), 8: (8, 3),
                                                  16: (16, 2)}[opts["msm_ne"]]
        else:
            assert cfg["ne"] == opts["msm_ne"] and cfg["copies"] == -(-16 // opts["msm_ne"])
    return check


@pytest.mark.parametrize("curve", CURVES, scope="module")
@pytest.mark.parametrize("opts", RESIDENCY, ids=lambda o: "-".join(f"{k}{v}" for k, v in o.items()))
def test_residency_plan(curve, opts):
    """msm_ne 0 (no copies, c from n), 1 .. 16 effective windows (3 and 5 leave a ragged last copy), a copies cap that forces
    ne up, and c = 12 / 13 / 14 (22 windows: above the 20-copy cap, so ne = 2; 20 windows: exactly on the cap; 19).  BW6-761
    has 24 windows at c = 16 (msm_ne 1 -> ne 2, 12 copies; 5 and 16 ragged) and 32 / 30 / 27 at c = 12 / 13 / 14."""
    run_config(curve, opts, _residency_check(curve, opts))


@pytest.mark.parametrize("curve", CURVES, scope="module")
@pytest.mark.parametrize("opts", RESIDENCY, ids=lambda o: "-".join(f"{k}{v}" for k, v in o.items()))
def test_residency_plan_batch(curve, opts):
    """the same plans with K rows per g16_prove_batch: ne > 1 gives every proof several bucket sets, ragged copies and
    c = 12 .. 14 other set sizes"""
    run_config(curve, opts, _residency_check(curve, opts), batch=True)


@pytest.mark.parametrize("curve", CURVES, scope="module")
def test_big_key_flow(curve):
    """bench.py's large-key flow verbatim: setup with msm_ne 0 and proof_slots 1, export, msm_ne 8, re-load, prove.  And the
    export must not depend on the residency plan: a setup run directly under msm_ne 2 exports the same key (and proves
    right from the setup-resident key)."""
    cs = case(curve)
    g, m = cs.g, cs.m
    G = GENERATORS[curve]
    fields = ("a_query", "b_g1_query", "b_g2_query", "h_query", "l_query", "beta_g1", "delta_g1")
    vk_fields = ("alpha_g1", "beta_g2", "gamma_g2", "delta_g2", "gamma_abc_g1")

    def same_key(a, b):
        for f in fields:
            assert np.array_equal(getattr(a, f), getattr(b, f)), f
        for f in vk_fields:
            assert np.array_equal(getattr(a.vk, f), getattr(b.vk, f)), f

    try:
        with knobs(cs, msm_ne=0, proof_slots=1):
            pk0 = g.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=True)
            same_key(pk0, cs.pk)
            g.set_option("msm_ne", 8)
            load(cs, dict(msm_ne=8, proof_slots=1), pk=pk0)
            assert np.array_equal(prove(cs), cs.want)
        with knobs(cs, msm_ne=2):
            pk2 = g.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=True)
            cfg = g.config()
            assert (cfg["ne"], cfg["copies"]) == (2, 12 if curve == BW6 else 8)
            assert np.array_equal(prove(cs), cs.want)
            same_key(pk2, cs.pk)
    finally:
        g.load_matrices(m)
        g.load_proving_key(cs.pk)


# ---- uneven batched-affine rounds (the shapes of the 2^24 memory guard) ---------------------------------------------------
UNEVEN = [dict(msm_ba=b1, msm_ba_g2=b2, ba_adaptive=0, share_b_sort=sh)
          for (b1, b2) in ((4, 0), (0, 4), (4, 2), (2, 4)) for sh in (1, 0)] + \
         [dict(msm_ba=4, msm_ba_g2=0, ba_adaptive=0, share_b_sort=1, msm_ne=8)]


def _uneven_check(opts):
    def check(cfg):
        assert (cfg["ba_rounds_g1"], cfg["ba_rounds_g2"]) == (opts["msm_ba"], opts["msm_ba_g2"])
        assert cfg["ba_rounds_g1"] != cfg["ba_rounds_g2"]
    return check


@pytest.mark.parametrize("curve", CURVES, scope="module")
@pytest.mark.parametrize("opts", UNEVEN, ids=lambda o: "-".join(f"{k}{v}" for k, v in o.items()))
def test_uneven_rounds(curve, opts):
    """B in G1 and B in G2 with different round counts: with share_b_sort 1 they still share one sorted list, padded for the
    larger count (ba_pad = max), so the MSM with fewer rounds (or none) walks a list longer than its own entries."""
    run_config(curve, opts, _uneven_check(opts))


@pytest.mark.parametrize("curve", CURVES, scope="module")
@pytest.mark.parametrize("opts", UNEVEN, ids=lambda o: "-".join(f"{k}{v}" for k, v in o.items()))
def test_uneven_rounds_batch(curve, opts):
    """the same uneven rounds under the batch's own padding (Engine::batch_geoms): one shared list for a whole group"""
    run_config(curve, opts, _uneven_check(opts), batch=True)


# ---- accumulation knobs ---------------------------------------------------------------------------------------------------
ACCUM = [("acc_k0_g1", v) for v in (4, 24, 128, 1024)] + [("acc_k0_g2", v) for v in (4, 48, 256)] + \
        [("acc_block", v) for v in (32, 64)]


def _accumulation_config(curve, rounds, knob, value, batch=False):
    opts = {knob: value} if rounds else {knob: value, "msm_ba": 0, "msm_ba_g2": 0}

    def check(cfg):
        assert cfg[{"acc_k0_g1": "k0_g1", "acc_k0_g2": "k0_g2", "acc_block": "acc_block"}[knob]] == value
        assert (cfg["ba_rounds_g1"] > 0 and cfg["ba_rounds_g2"] > 0) if rounds else (cfg["ba_rounds_g1"] == cfg["ba_rounds_g2"] == 0)
    run_config(curve, opts, check, batch=batch)


@pytest.mark.parametrize("curve", CURVES, scope="module")
@pytest.mark.parametrize("rounds", [1, 0], ids=["rounds", "no_rounds"])
@pytest.mark.parametrize("knob,value", ACCUM)
def test_accumulation_knobs(curve, rounds, knob, value):
    """sorted entries per level-0 thread (any value in 4 .. 1024, powers of two or not, above MSM_K0_MAX too; with rounds the
    last list runs k0 >> R) and the level-0 block size, with and without the batched-affine rounds"""
    _accumulation_config(curve, rounds, knob, value)


@pytest.mark.parametrize("curve", CURVES, scope="module")
@pytest.mark.parametrize("rounds", [1, 0], ids=["rounds", "no_rounds"])
@pytest.mark.parametrize("knob,value", ACCUM)
def test_accumulation_knobs_batch(curve, rounds, knob, value):
    """the same knobs over a group's sorted list (k0 1024 and 4 at the group's length)"""
    _accumulation_config(curve, rounds, knob, value, batch=True)


INT64_MAX = (1 << 63) - 1
# every option of g16_set_option and the values it accepts, as the union of closed ranges (include/g16b200.h)
ACCEPTED = {"msm_ne": [(0, 32)], "msm_c": [(0, 24)], "msm_maxcopies": [(1, 20)], "msm_ba": [(0, 6)], "msm_ba_g2": [(0, 6)],
            "ba_m": [(1, 256)], "ba_g": [(1, 4096)], "ba_min_entries_g1": [(0, INT64_MAX)],
            "ba_min_entries_g2": [(0, INT64_MAX)], "acc_k0_g1": [(0, 0), (4, 1024)], "acc_k0_g2": [(0, 0), (4, 1024)],
            "acc_block": [(32, 32), (64, 64), (128, 128)], "ba_inv_gcd": [(0, 1)], "ba_adaptive": [(0, 1)],
            "share_b_sort": [(0, 1)], "wm_split": [(0, 1)], "wm_first": [(-1, 1)], "proof_slots": [(1, 2)]}


def test_knobs_out_of_range_are_refused():
    """a value the kernels cannot honour is an error, not a silent replacement, and leaves the option unchanged: for every
    option the values just outside its set (below, above, and in each gap of a discrete set); every endpoint of the set
    is accepted and reads back unchanged"""
    cs = case("bn254")
    saved = {k: cs.g.get_option(k) for k in ACCEPTED}
    try:
        for k, ranges in ACCEPTED.items():
            bad = {ranges[0][0] - 1, ranges[-1][1] + 1} | {v for (_, hi), (lo, _) in zip(ranges, ranges[1:]) for v in (hi + 1, lo - 1)}
            for v in sorted(b for b in bad if b <= INT64_MAX):
                before = cs.g.get_option(k)
                with pytest.raises(ValueError):
                    cs.g.set_option(k, v)
                assert cs.g.get_option(k) == before, (k, v)
            for v in sorted({e for r in ranges for e in r}):
                cs.g.set_option(k, v)
                assert cs.g.get_option(k) == v, (k, v)
            cs.g.set_option(k, saved[k])
    finally:
        for k, v in saved.items():
            cs.g.set_option(k, v)
    with pytest.raises(ValueError):
        cs.g.get_option("no_such_option")


def test_options_from_environment():
    """g16_ctx_create reads G16_<OPTION> for every option; a value outside the option's set makes it fail, naming the
    variable"""
    import os
    keep = {k: os.environ.get(k) for k in ("G16_ACC_BLOCK", "G16_WM_SPLIT")}
    try:
        os.environ.update(G16_ACC_BLOCK="64", G16_WM_SPLIT="0")
        g = Groth16("bn254", 0)
        try:
            assert (g.get_option("acc_block"), g.get_option("wm_split")) == (64, 0)
        finally:
            g.close()
        os.environ["G16_ACC_BLOCK"] = "100"
        with pytest.raises(ValueError, match="G16_ACC_BLOCK"):
            Groth16("bn254", 0)
    finally:
        for k, v in keep.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# ---- schedules ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES, scope="module")
def test_schedules(curve):
    """witness map first, one proof slot (memory guard recomputed), serialised MSMs and two pipelined proofs under ne = 8"""
    run_config(curve, dict(wm_first=1))
    run_config(curve, dict(proof_slots=1))
    run_config(curve, dict(msm_ne=8), flags=_lib.SERIAL_MSMS)
    cs = case(curve)
    with knobs(cs, msm_ne=8):
        load(cs, dict(msm_ne=8))
        outs = [np.zeros(cs.pw, dtype=np.uint64) for _ in range(2)]
        for slot in (0, 1):
            cs.g.prove_submit_raw(slot, cs.r, cs.s, cs.z.ctypes.data, 0)
        for slot in (0, 1):
            cs.g.prove_wait_raw(slot, outs[slot])
        for o in outs:
            assert np.array_equal(o, cs.want)


@pytest.mark.parametrize("curve", CURVES, scope="module")
def test_schedules_batch(curve):
    """witness map first, one proof slot (the groups then share slot 0) and serialised MSMs under ne = 8, in batches"""
    run_config(curve, dict(wm_first=1), batch=True)
    run_config(curve, dict(proof_slots=1), batch=True)
    run_config(curve, dict(msm_ne=8), flags=_lib.SERIAL_MSMS, batch=True)


# ---- sharded keys ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES, scope="module")
@pytest.mark.parametrize("world,opts", [(2, {}), (3, {}), (8, {}), (2, dict(msm_ne=4))], ids=["w2", "w3", "w8", "w2-ne4"])
def test_sharded_key(curve, world, opts):
    """every rank's round-robin share at its own geometry (2 ranks: rank 0's H shard has 2^16 pairs and runs c = 16, rank 1's
    has 2^16 - 1 and falls back to the size rule, c = 12), partial sums assembled into the oracle's proof"""
    cs = case(curve)
    g = cs.g
    parts = []
    try:
        with knobs(cs, **opts):
            for rank in range(world):
                cfg = load(cs, opts, rank, world)
                if world == 2 and not opts:
                    assert cfg["c"] == (16 if rank == 0 else 12)
                out = np.zeros(g.partial_limbs(), dtype=np.uint64)
                g.prove_partial_raw(cs.r, cs.z.ctypes.data, 0, out)
                parts.append(out)
        pf = g.prove_assemble(cs.r, cs.s, np.stack(parts))
        assert np.array_equal(np.concatenate([pf.a, pf.b, pf.c]), cs.want)
    finally:
        g.load_proving_key(cs.pk)


# ---- adversarial bases and signed-digit edge scalars at the resident geometry ----------------------------------------------
def edge_scalars(r, c):
    """canonical scalars at the signed-digit boundaries of c-bit windows"""
    bits = r.bit_length()
    B = 1 << (c - 1)
    out = {0, 1, r - 1, r - 2, (r - 1) // 2, 1 << (bits - 1)}
    for digit in (B, B + 1, B - 1, (1 << c) - 1):
        v = 0
        for k in range(bits // c + 2):
            v += digit << (c * k)
            out.add(v % r)
            if v < r:
                out.add(v)
    for k in range(1, bits // c + 2):
        out.add(((1 << (c * k)) - 1) % r)
        out.add((1 << (c * k)) % r)
    return sorted(out)


def _neg_points(cd, curve, arr, g2):
    pts = cd.dec_g2(arr) if g2 else cd.dec_g1(arr)
    if curve == BW6:
        neg = ref.neg
    else:
        cx = P.ctx(curve)
        neg = (cx.G2 if g2 else cx.G1).neg
    return cd.enc_g2([neg(p) for p in pts]) if g2 else cd.enc_g1([neg(p) for p in pts])


_ADV = {}
DUP = np.arange(1000, 1600, 2)
OPP = np.arange(2000, 2600, 2)


def _adversarial_edit(Q, neg):
    """base pairs (i, i + 1): duplicates from 1000, opposites from 2000; identity runs longer than a batched-affine tile.
    The same positions in every query, so that b_g1 and b_g2 keep one identity pattern (shared sorted list)."""
    Q[DUP + 1] = Q[DUP]
    Q[OPP + 1] = neg(Q[OPP])
    Q[3000:3000 + 700] = 0
    Q[5000:5000 + 3] = 0


def adversarial(curve):
    """key with duplicate / opposite base pairs (equal scalars: the pair meets in one bucket in every window) and identity
    runs longer than a batched-affine tile in all five queries, an assignment of edge scalars for c = 13 and c = 16, the
    oracle of that key and its five MSMs over the assignment"""
    if curve in _ADV:
        return _ADV[curve]
    cs = case(curve)
    cd = cs.g.codec
    ni = cs.m.num_instance_variables
    z = cs.z.copy()
    edges = edge_scalars(cd.c.r, 16) + edge_scalars(cd.c.r, 13)
    z[4000:4000 + len(edges)] = cd.fr.enc(edges)
    rs = np.random.RandomState(5)
    q = {f: np.array(getattr(cs.pk, f), copy=True) for f in ("a_query", "b_g1_query", "b_g2_query", "h_query", "l_query")}

    # scalars: a / b base k <-> z[k], l base k <-> z[ni + k]; the h scalars come from the witness map
    for name, Q in q.items():
        _adversarial_edit(Q, lambda a: _neg_points(cd, curve, a, name == "b_g2_query"))
    for first in (1000, 2000):
        for k in range(first, first + 600, 2):
            for off in (0, ni):
                v = edges[(k // 2) % len(edges)] if k % 4 == 0 else int(rs.randint(1, 1 << 62))
                z[k + off] = z[k + 1 + off] = cd.fr.enc1(v % cd.c.r)
    pk = type(cs.pk)(cs.pk.vk, cs.pk.beta_g1, cs.pk.delta_g1, q["a_query"], q["b_g1_query"], q["b_g2_query"], q["h_query"],
                     q["l_query"])
    oracle = cs.oracle.for_key(pk, _adversarial_edit)
    _ADV[curve] = (pk, np.ascontiguousarray(z), oracle.partials(z), oracle)
    return _ADV[curve]


_ADV_ROWS = {}


def adversarial_rows(curve):
    """batch rows on the adversarial key: its edge-scalar assignment, the same negated (every scalar but the constant One
    becomes r - z_i, so every signed digit and carry flips) and a random row; with their oracle proofs"""
    if curve not in _ADV_ROWS:
        cs = case(curve)
        cd = cs.g.codec
        pk, z, _, oracle = adversarial(curve)
        vals = cd.fr.dec(z)
        zn = cd.fr.enc([vals[0]] + [(-v) % cd.c.r for v in vals[1:]]).reshape(z.shape)
        rr = np.random.RandomState(43)
        R, S = (np.ascontiguousarray(cd.fr.enc([int.from_bytes(rr.bytes(32), "little") % cd.c.r for _ in range(K)]))
                for _ in range(2))
        rows = (R, S, np.ascontiguousarray(np.stack([z, zn, np.roll(cs.z, 5, axis=0)])))
        wants = np.stack([oracle.proof(rows[2][k], rows[0][k], rows[1][k]) for k in range(K)])
        _ADV_ROWS[curve] = (rows, wants)
    return _ADV_ROWS[curve]


def _adversarial_opts(ne, rounds):
    return dict(msm_ne=ne, ba_adaptive=0, msm_ba=4 if rounds else 0, msm_ba_g2=4 if rounds else 0)


@pytest.mark.parametrize("curve", CURVES, scope="module")
@pytest.mark.parametrize("ne", [0, 1, 8])
@pytest.mark.parametrize("rounds", [1, 0], ids=["rounds", "no_rounds"])
def test_adversarial_batch(curve, ne, rounds):
    """the adversarial key in batches: there is no batch partial API, so full proofs of the edge-scalar row, its negation
    and a random row, against the oracle's proofs on that key"""
    cs = case(curve)
    pk = adversarial(curve)[0]
    rows, wants = adversarial_rows(curve)
    opts = _adversarial_opts(ne, rounds)
    try:
        with knobs(cs, **opts):
            assert load(cs, opts, pk=pk)["c"] == (13 if ne == 0 else 16)
            prove_batch(cs, rows, wants, tag=("adversarial", ne, rounds))
    finally:
        cs.g.load_proving_key(cs.pk)


@pytest.mark.parametrize("curve", CURVES, scope="module")
@pytest.mark.parametrize("ne", [0, 1, 8])
@pytest.mark.parametrize("rounds", [1, 0], ids=["rounds", "no_rounds"])
def test_adversarial_partials(curve, ne, rounds):
    """tangent (P + P) and cancellation (P - P) cases inside one bucket of the device rounds, G1 and G2, identity runs, and
    the carry chains of edge scalars at c = 13 (ne 0) and c = 16: every partial MSM against the oracle's.  For BW6-761 the
    signed digits of c = 13 run to W = 30 windows, the carry of c = 16 into the 24th."""
    cs = case(curve)
    pk, z, want, _ = adversarial(curve)
    nq = cs.g.nq
    opts = _adversarial_opts(ne, rounds)
    try:
        with knobs(cs, **opts):
            cfg = load(cs, opts, pk=pk)
            assert cfg["c"] == (13 if ne == 0 else 16)
            out = np.zeros(cs.g.partial_limbs(), dtype=np.uint64)
            cs.g.prove_partial_raw(cs.r, z.ctypes.data, 0, out)
    finally:
        cs.g.load_proving_key(cs.pk)
    for k, w in enumerate(want):
        got = out[2 * nq * k:2 * nq * k + w.shape[0]]
        assert np.array_equal(got, w), (curve, ne, rounds, MSMS[k])


# ---- stand-alone g16_msm_g1 / g2 above 2^15 pairs ---------------------------------------------------------------------------
def _msm_source(cs, g2):
    """the key points the stand-alone bases are tiled from, and their negation"""
    cd = cs.g.codec
    src = np.asarray(cs.pk.b_g2_query) if g2 else np.concatenate([np.asarray(cs.pk.h_query), np.asarray(cs.pk.l_query)])
    return src, lambda a: _neg_points(cd, cs.curve, a, g2)


def _msm_tile(n):
    """n entries tiled from a source array, with duplicates, opposites and identities: the same edit of key points and of
    their discrete logs"""
    def tile(src, neg):
        out = np.resize(src, (n,) + src.shape[1:]).copy()
        out[101:401:2] = out[100:400:2]
        out[501:801:2] = neg(out[500:800:2])
        out[900:1200] = 0
        return out
    return tile


def _msm_inputs(curve, n, c, g2=False):
    """n bases taken from the module key (tiled when n exceeds it), with duplicates, opposites and identities; edge scalars
    for c-bit windows, equal scalars on the duplicate / opposite pairs, uniform-looking canonical scalars elsewhere"""
    cs = case(curve)
    cd = cs.g.codec
    tile = _msm_tile(n)
    bases = np.ascontiguousarray(tile(*_msm_source(cs, g2)))
    rs = np.random.RandomState(n + c)
    nr = cs.g.nr
    sc = rs.randint(0, 1 << 62, size=(n, nr), dtype=np.int64).astype(np.uint64)
    sc[:, nr - 1] &= np.uint64((1 << (58 if nr == 4 else 56)) - 1)    # below 2^250 / 2^376: below r
    edges = edge_scalars(cd.c.r, c)
    sc[2000:2000 + len(edges)] = cd.fr.bigint(edges)
    sc[101:401:2] = sc[100:400:2]
    sc[501:801:2] = sc[500:800:2]
    sc[3000:3100] = 0
    return bases, np.ascontiguousarray(sc), tile


def _check_msm(curve, n, c_expect, g2=False, msm_c=0):
    cs = case(curve)
    bases, sc, tile = _msm_inputs(curve, n, c_expect, g2)
    assert msm_c or _pick_c(n) == c_expect
    with knobs(cs, msm_c=msm_c):
        got = cs.g.msm_g2(bases, sc) if g2 else cs.g.msm_g1(bases, sc)
    cs.oracle.check_msm(got, tile, sc, g2)


@pytest.mark.parametrize("curve", CURVES, scope="module")
@pytest.mark.parametrize("n,c", [((1 << 16) - 1, 12), ((1 << 16) + 1, 13), ((1 << 17) + 3, 14)])
def test_standalone_msm_g1(curve, n, c):
    """no precomputation: W bucket sets of 2^(c-1) buckets each, scans over many blocks"""
    _check_msm(curve, n, c)


def test_standalone_msm_g1_c16():
    """2^20 pairs: c = 16, 16 bucket sets of 2^15 buckets, batched-affine rounds on a caller-supplied base array"""
    _check_msm("bls12_381", 1 << 20, 16)


def test_standalone_msm_g2():
    _check_msm("bls12_377", (1 << 16) + 1, 13, g2=True)


@pytest.mark.parametrize("msm_c", [17, 20])
def test_standalone_msm_wide_windows(msm_c):
    """msm_c above 16 (the header allows 24): at c = 20 there are 13 x 2^19 keys, 1664 scan blocks, and msm_scan_tops loops
    over its 1024-wide block scan twice"""
    _check_msm("bn254", 1 << 16, msm_c, msm_c=msm_c)


@pytest.mark.parametrize("curve", [BW6])
@pytest.mark.parametrize("g2,n,c,msm_c", [(False, 1 << 20, 16, 0), (True, (1 << 16) + 1, 13, 0), (False, 1 << 16, 17, 17),
                                          (False, 1 << 16, 20, 20)], ids=["g1-2p20-c16", "g2-c13", "g1-c17", "g1-c20"])
def test_standalone_msm_wide_scalars(curve, g2, n, c, msm_c):
    """377-bit scalars: 2^20 pairs at c = 16 (W = 24, the batched-affine rounds on the wide instance), G2 at c = 13 (W = 30),
    and c = 17 / 20 (W = 23 / 19)"""
    _check_msm(curve, n, c, g2=g2, msm_c=msm_c)
