"""Element-level checks of the product arithmetic against Python big integers: every Fp operation of the eight fields (Fr
and Fq of BLS12-381, BN254, BLS12-377 and BW6-761), the three Fq2 towers and the XYZZ point operations of G1 and G2 of
all four curves, one operation per vector, compared bit for bit.

tests/arith/arith_ops.cu runs the templates of fp.cuh, ec.cuh, fp_inv.cuh and msm_ba.cuh themselves, built three ways:
the plain 64-bit host back-end and the device algorithm under emulated PTX carries (CPU tests, built here with g++), and
the sm_90a device build libg16arith.so (GPU tests; made by __graft_entry__.build()).  Only the device build runs the
inline-asm carry primitives, the out-of-line base-field product mont_mul_call and the __ldg loads of ba_ld.

Operands and results are raw Montgomery limbs, which is what the carry chains see: mul(x, y) must give x*y*R^-1 mod p.
They are chosen where this kind of arithmetic breaks -- 0, p - 1, (p +- 1)/2, R, R^2, R^-1, every 2^k, 2^k - 1 and
p - 2^k, limb patterns, pairs whose top-limb partial product is 0xffffffff -- plus random values.  Point results are
normalised here (x = X/ZZ, y = Y/ZZZ, identity <=> ZZ == 0, and ZZ^3 == ZZZ^2 for every finite result); the accumulators
carry ZZ != 1 so that the doubling and inverse branches of the additions are reached from general projective inputs.
Vectors are generated once per process from fixed seeds, and every (field, op) asserts a minimum vector count.

BW6-761 (12-limb Fr, 24-limb Fq, G1 and G2 both over Fq) has no pyref curve: its points are checked in value space over
tests/bw6_ref.py, and its Fp cases run the same operand sets at 24 limbs."""
import ctypes as C
import functools
import glob
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

import bw6_ref as ref
import pyref as P
from groth16_b200.params import GENERATORS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARITH = os.path.join(ROOT, "tests", "arith")
SRC = os.path.join(ARITH, "arith_ops.cu")
DEVICE_LIB = os.path.join(ARITH, "libg16arith.so")
CSRC = os.path.join(ROOT, "groth16_b200", "csrc")

CURVES = ("bls12_381", "bn254", "bls12_377")   # the pairing curves (pyref)
BW6 = "bw6_761"
POINT_CURVES = CURVES + (BW6,)
# op ids of arith_ops.cu
ADD, SUB, NEG, DBL, MUL, SQR, MUL_SMALL, FROM_MONT, TO_MONT, POW_U64, INV, INV_GCD, MUL_NR, BA_INV = range(14)
MADD, MADD_NEG, MADD_LAZY, MADD_LAZY_NEG, PADD, PDBL, PDBL_AFFINE, PMUL_U32, TO_AFFINE = range(20, 29)
FP_OPS = {"add": ADD, "sub": SUB, "neg": NEG, "dbl": DBL, "mul": MUL, "sqr": SQR, "mul_small": MUL_SMALL,
          "from_mont": FROM_MONT, "to_mont": TO_MONT, "pow_u64": POW_U64, "inv": INV, "inv_safegcd": INV_GCD,
          "ba_inv": BA_INV}
BASE_ONLY = {"ba_inv"}   # Fp ops that run on the base fields only (the batched-affine inversion of a G1 / BW6 G2 combine)
FQ2_OPS = {"add": ADD, "sub": SUB, "neg": NEG, "dbl": DBL, "mul": MUL, "sqr": SQR, "mul_nr": MUL_NR, "inv": INV,
           "ba_inv": BA_INV}
POINT_OPS = {"madd": MADD, "madd_neg": MADD_NEG, "madd_lazy": MADD_LAZY, "madd_lazy_neg": MADD_LAZY_NEG, "add": PADD,
             "dbl_inplace": PDBL, "dbl_affine": PDBL_AFFINE, "mul_u32": PMUL_U32, "to_affine": TO_AFFINE}
# minimum vectors per case: a change to the generator must not quietly shrink the coverage
MIN_FP = {"add": 100_000, "sub": 100_000, "mul": 100_000, "neg": 1 << 16, "dbl": 1 << 16, "sqr": 1 << 16,
          "from_mont": 1 << 16, "to_mont": 1 << 16, "mul_small": 10_000, "pow_u64": 5_000, "inv": 2_500,
          "inv_safegcd": 2_500, "ba_inv": 5_000}
MIN_FQ2 = {"add": 30_000, "sub": 30_000, "mul": 30_000, "neg": 10_000, "dbl": 10_000, "sqr": 10_000, "mul_nr": 8_000,
           "inv": 3_000, "ba_inv": 6_000}
MIN_POINT = {"madd": 150, "madd_neg": 150, "madd_lazy": 150, "madd_lazy_neg": 150, "add": 200, "dbl_inplace": 20,
             "dbl_affine": 20, "mul_u32": 50, "to_affine": 80}
M32 = 0xFFFFFFFF


def _field_ids():
    fp, fq2 = {}, {}
    for i, name in enumerate(CURVES):
        c = P.CURVES[name]
        fp[f"{name}_fr"] = (2 * i, c.r)
        fp[f"{name}_fq"] = (2 * i + 1, c.q)
        fq2[f"{name}_fq2"] = (6 + i, c.q, -c.beta)   # Fq2 = Fq[u]/(u^2 + NR), NR = -beta
    fp[f"{BW6}_fr"] = (9, ref.R)
    fp[f"{BW6}_fq"] = (10, ref.Q)
    return fp, fq2


FP_FIELDS, FQ2_FIELDS = _field_ids()
CASES = ([f"fp-{f}-{o}" for f in FP_FIELDS for o in FP_OPS if f.endswith("_fq") or o not in BASE_ONLY]
         + [f"fq2-{f}-{o}" for f in FQ2_FIELDS for o in FQ2_OPS]
         + [f"pt-{c}_{g}-{o}" for c in POINT_CURVES for g in ("g1", "g2") for o in POINT_OPS])


# ------------------------------------------------------------------------------------------------------------------
# limbs
# ------------------------------------------------------------------------------------------------------------------
def _nw(p):
    nb = p.bit_length()
    return 8 if nb <= 256 else 12 if nb <= 384 else 24


def _pack(vals, nw):
    """ints -> (n, nw) little-endian u32 limbs"""
    b = b"".join(v.to_bytes(4 * nw, "little") for v in vals)
    return np.frombuffer(b, dtype="<u4").reshape(len(vals), nw).astype(np.uint32)


def _unpack(arr):
    """(n, w) u32 limbs -> ints"""
    b = np.ascontiguousarray(arr, dtype="<u4").tobytes()
    w = 4 * arr.shape[1]
    return [int.from_bytes(b[i:i + w], "little") for i in range(0, len(b), w)]


def _hex(v, nw):
    return f"{v:0{8 * nw}x}"


def _dedupe(xs):
    return list(dict.fromkeys(xs))


# ------------------------------------------------------------------------------------------------------------------
# operands
# ------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(None)
def _edges(p):
    """(core, full) edge operands of Fp, as raw limbs below p.  full: the named values, every 2^k, 2^k - 1, p - 2^k below
    the bit length, and the limb patterns; core (~110-150 values): the named values, the patterns and the powers of two
    at the limb boundaries."""
    nw, nb, R = _nw(p), p.bit_length(), 1 << (32 * _nw(p))
    named = [0, 1, 2, 3, p - 1, p - 2, p - 3, (p - 1) // 2, (p + 1) // 2, R % p, R * R % p, pow(R, -1, p), (-R) % p]
    top_shift = 32 * (nw - 1)
    top = p >> top_shift

    def below_p(v):   # a limb pattern as it is, or with its top bits cleared, or with p's top limb - 1 on top
        if v < p:
            return [v]
        return [v & ((1 << (nb - 1)) - 1), (v & ((1 << top_shift) - 1)) | ((top - 1) << top_shift)]

    pats = [sum(M32 << (32 * i) for i in range(nw)), sum(0x80000000 << (32 * i) for i in range(nw)),
            sum(M32 << (32 * i) for i in range(0, nw, 2)), sum(M32 << (32 * i) for i in range(1, nw, 2))]
    pats += [M32 << (32 * i) for i in range(nw)]
    patterns = [x for v in pats for x in below_p(v)]

    def pow2(ks):
        return [x for k in ks for x in (1 << k, (1 << k) - 1, p - (1 << k))]

    core_ks = sorted({k for i in range(1, nw) for k in (32 * i - 1, 32 * i, 32 * i + 1)} | {0, 1, nb - 2, nb - 1})
    core = _dedupe(named + patterns + pow2(core_ks))
    full = _dedupe(core + pow2(range(nb)))
    assert all(0 <= x < p for x in full)
    return core, full


def _carry_pairs(p, rng):
    """pairs (a, b) and (b, a) where a's top limb t times one lower limb of b is 0xffffffff mod 2^32: the low word of that
    32x32 partial product is all ones, so a carry into it runs on through the madc chain"""
    nw = _nw(p)
    sh = 32 * (nw - 1)
    top = p >> sh
    ts = [top - 1 if (top - 1) & 1 else top - 2] + [rng.randrange(1, top) | 1 for _ in range(7)]
    out = []
    for t in ts:
        bj = M32 * pow(t, -1, 1 << 32) % (1 << 32)
        for j in range(nw - 1):
            a = rng.randrange(1 << sh) | (t << sh)
            b = (rng.randrange(p) & ~(M32 << (32 * j))) | (bj << (32 * j))
            if a < p and b < p:
                out += [(a, b), (b, a)]
    return out


@functools.lru_cache(None)
def _fp_pairs(p, seed):
    rng = random.Random(seed)
    core, full = _edges(p)
    pairs = [(a, b) for a in core for b in full] + [(a, a) for a in full] + [(a, (p - a) % p) for a in full]
    pairs += _carry_pairs(p, rng)
    pairs += [(rng.randrange(p), rng.randrange(p)) for _ in range(1 << 16)]
    return pairs


@functools.lru_cache(None)
def _fp_singles(p, seed, n_random):
    rng = random.Random(seed)
    return _edges(p)[1] + [rng.randrange(p) for _ in range(n_random)]


def _fq2_edge_elems(q, rng, n):
    """Fq2 elements whose components are Fq edges: (e, 0), (0, e), (e, e) for the core, and n sampled edge x edge pairs"""
    core, full = _edges(q)
    els = [(e, 0) for e in core] + [(0, e) for e in core] + [(e, e) for e in core]
    els += [(rng.choice(full), rng.choice(full)) for _ in range(n)]
    return _dedupe(els)


# ------------------------------------------------------------------------------------------------------------------
# cases: inputs plus a checker
# ------------------------------------------------------------------------------------------------------------------
class Case:
    def __init__(self, name, fid, op, inp, check, describe):
        self.name, self.fid, self.op, self.inp = name, fid, op, np.ascontiguousarray(inp, dtype=np.uint32)
        self.check = check           # out -> indices of failing vectors
        self.describe = describe     # (i, out) -> text

    def __len__(self):
        return self.inp.shape[0]


def _exact_case(name, fid, op, ins, want, nw_in, nw_out):
    """ins: list of operand columns (lists of ints, or (n, k) u32 arrays of extra words), want: list of ints"""
    cols = [c if isinstance(c, np.ndarray) else _pack(c, w) for c, w in zip(ins, nw_in)]
    inp = np.hstack(cols)
    exp = _pack(want, nw_out)

    def check(out):
        return np.nonzero((out != exp).any(axis=1))[0]

    def describe(i, out):
        ops = " ".join(f"{_unpack(c[i:i + 1])[0]:x}" for c in cols)
        return f"#{i}: in {ops}  got {_hex(_unpack(out[i:i + 1])[0], nw_out)}  want {_hex(want[i], nw_out)}"
    return Case(name, fid, op, inp, check, describe)


def _fp_case(name, field, opname):
    fid, p = FP_FIELDS[field]
    nw = _nw(p)
    R = 1 << (32 * nw)
    Ri = pow(R, -1, p)
    seed = f"{field}:{opname}"
    if opname in ("add", "sub", "mul"):
        pairs = _fp_pairs(p, field)
        a, b = [x for x, _ in pairs], [y for _, y in pairs]
        f = {"add": lambda x, y: (x + y) % p, "sub": lambda x, y: (x - y) % p, "mul": lambda x, y: x * y * Ri % p}[opname]
        return _exact_case(name, fid, FP_OPS[opname], [a, b], [f(x, y) for x, y in pairs], [nw, nw], nw)
    if opname in ("neg", "dbl", "sqr", "from_mont", "to_mont"):
        a = _fp_singles(p, field, 1 << 16)
        f = {"neg": lambda x: (-x) % p, "dbl": lambda x: 2 * x % p, "sqr": lambda x: x * x * Ri % p,
             "from_mont": lambda x: x * Ri % p, "to_mont": lambda x: x * R % p}[opname]
        return _exact_case(name, fid, FP_OPS[opname], [a], [f(x) for x in a], [nw], nw)
    if opname == "mul_small":
        a0 = _fp_singles(p, field, 4096)
        a = [x for x in a0 for _ in (3, 4, 5)]
        k = [k for _ in a0 for k in (3, 4, 5)]
        return _exact_case(name, fid, MUL_SMALL, [a, np.array(k, dtype=np.uint32)[:, None]],
                           [x * k % p for x, k in zip(a, k)], [nw, 1], nw)
    if opname == "pow_u64":
        rng = random.Random(seed)
        es = [0, 1, 2, 3, M32, 1 << 32, (1 << 64) - 1]
        full = _edges(p)[1]
        a = [x for x in full for _ in es] + [rng.randrange(p) for _ in range(2048)]
        e = [e for _ in full for e in es] + [rng.randrange(1 << 64) for _ in range(2048)]
        # value x R^-1 to the power e, back in Montgomery form: x^e R^(1-e)
        want = [pow(x, ee, p) * pow(Ri, ee - 1, p) % p if ee else R % p for x, ee in zip(a, e)]
        return _exact_case(name, fid, POW_U64, [a, e], want, [nw, 2], nw)
    if opname in ("inv", "inv_safegcd"):
        a = _fp_singles(p, field, 2048)
        # value x R^-1 -> R x^-1, in Montgomery form R^2 x^-1; the inverse of zero is zero
        return _exact_case(name, fid, FP_OPS[opname], [a], [R * R * pow(x, -1, p) % p if x else 0 for x in a], [nw], nw)
    if opname == "ba_inv":
        a = _fp_singles(p, f"{field}:ba_inv", 2048)
        gcd = np.array([g for _ in a for g in (0, 1)], dtype=np.uint32)[:, None]   # Fermat and safegcd
        a2 = [x for x in a for _ in (0, 1)]
        return _exact_case(name, fid, BA_INV, [a2, gcd], [R * R * pow(x, -1, p) % p if x else 0 for x in a2], [nw, 1], nw)
    raise KeyError(opname)


def _fq2_case(name, field, opname):
    fid, q, nr = FQ2_FIELDS[field]
    nw = _nw(q)
    R = 1 << (32 * nw)
    Ri = pow(R, -1, q)
    rng = random.Random(f"{field}:{opname}")
    enc = lambda z: z[0] | (z[1] << (32 * nw))
    rnd = lambda: (rng.randrange(q), rng.randrange(q))

    def mul(x, y):   # raw Montgomery limbs: (x0 + x1 u)(y0 + y1 u) with u^2 = -NR, each product times R^-1
        return ((x[0] * y[0] - nr * x[1] * y[1]) * Ri % q, (x[0] * y[1] + x[1] * y[0]) * Ri % q)

    def inv(x):      # value x/R -> R/x: raw R^2 conj(x) / norm(x); the inverse of zero is zero
        n = (x[0] * x[0] + nr * x[1] * x[1]) % q
        if n == 0:
            return (0, 0)
        s = R * R * pow(n, -1, q) % q
        return (x[0] * s % q, (-x[1]) * s % q)

    if opname in ("add", "sub", "mul"):
        els = _fq2_edge_elems(q, rng, 4096)
        pairs = [(rng.choice(els), rng.choice(els)) for _ in range(1 << 14)] + [(x, x) for x in els]
        pairs += [(x, ((-x[0]) % q, (-x[1]) % q)) for x in els[:1024]] + [(rnd(), rnd()) for _ in range(1 << 14)]
        f = {"add": lambda x, y: ((x[0] + y[0]) % q, (x[1] + y[1]) % q),
             "sub": lambda x, y: ((x[0] - y[0]) % q, (x[1] - y[1]) % q), "mul": mul}[opname]
        return _exact_case(name, fid, FQ2_OPS[opname], [[enc(x) for x, _ in pairs], [enc(y) for _, y in pairs]],
                           [enc(f(x, y)) for x, y in pairs], [2 * nw, 2 * nw], 2 * nw)
    if opname in ("neg", "dbl", "sqr"):
        a = _fq2_edge_elems(q, rng, 4096) + [rnd() for _ in range(1 << 13)]
        f = {"neg": lambda x: ((-x[0]) % q, (-x[1]) % q), "dbl": lambda x: (2 * x[0] % q, 2 * x[1] % q),
             "sqr": lambda x: mul(x, x)}[opname]
        return _exact_case(name, fid, FQ2_OPS[opname], [[enc(x) for x in a]], [enc(f(x)) for x in a], [2 * nw], 2 * nw)
    if opname == "mul_nr":
        a = _fp_singles(q, f"{field}:mul_nr", 1 << 13)
        return _exact_case(name, fid, MUL_NR, [a], [nr * x % q for x in a], [nw], nw)
    if opname in ("inv", "ba_inv"):
        a = _fq2_edge_elems(q, rng, 2048) + [rnd() for _ in range(1024)]
        if opname == "inv":
            return _exact_case(name, fid, INV, [[enc(x) for x in a]], [enc(inv(x)) for x in a], [2 * nw], 2 * nw)
        gcd = np.array([g for _ in a for g in (0, 1)], dtype=np.uint32)[:, None]   # Fermat and safegcd
        a2 = [x for x in a for _ in (0, 1)]
        return _exact_case(name, fid, BA_INV, [[enc(x) for x in a2], gcd], [enc(inv(x)) for x in a2], [2 * nw, 1], 2 * nw)
    raise KeyError(opname)


class _Bw6Group:
    """BW6-761's G1 (b = -1) or G2 (b = 4), both over Fq, with the methods of pyref.Group, over tests/bw6_ref.py"""

    def __init__(self, b):
        self.b = b

    def add(self, p, q):
        return ref.add(p, q)

    def dbl(self, p):
        return ref.add(p, p)     # (x, 0): 2 y = 0, the identity

    def neg(self, p):
        return ref.neg(p)

    def mul(self, p, k):
        return ref.mul_proj(k, p)


class _Group:
    """G1 or G2 of a curve in value space (pyref, or bw6_ref for BW6-761), with the raw Montgomery encoding of its
    coordinates"""

    def __init__(self, curve, g2):
        if curve == BW6:
            self.q, self.r = ref.Q, ref.R
            self.F, self.G = P.FqOps(ref.Q), _Bw6Group(ref.B2 if g2 else ref.B1)
            self.gen = GENERATORS[BW6]["g2" if g2 else "g1"]
            self.fq2 = False                        # G2 over Fq
            self.fid = FP_FIELDS[f"{BW6}_fq"][0]
            self.sw = 12                            # Fr::N: 377-bit scalars in 12 words
        else:
            c = P.CURVES[curve]
            cx = P.ctx(c)
            self.q, self.r = c.q, c.r
            self.F, self.G = (cx.Fq2, cx.G2) if g2 else (cx.Fq, cx.G1)
            self.gen = cx.g2_gen() if g2 else cx.g1_gen()
            self.fq2 = g2
            self.fid = FQ2_FIELDS[f"{curve}_fq2"][0] if g2 else FP_FIELDS[f"{curve}_fq"][0]
            self.sw = 8
        self.nw = _nw(self.q)
        self.R = 1 << (32 * self.nw)
        self.Ri = pow(self.R, -1, self.q)
        self.ew = 2 * self.nw if self.fq2 else self.nw      # words per coordinate

    @functools.lru_cache(None)
    def pool(self, seed):
        """128 pseudo-random subgroup points: S, S + D, S + 2D, ... for random multiples S, D of the generator (one affine
        addition per point instead of one scalar multiplication)"""
        rng = random.Random(seed)
        s, d = (self.G.mul(self.gen, rng.randrange(1, self.r)) for _ in range(2))
        out = [s]
        for _ in range(127):
            out.append(self.G.add(out[-1], d))
        return out

    def rand(self, rng):
        return rng.randrange(1, self.q) if not self.fq2 else (rng.randrange(self.q), rng.randrange(1, self.q))

    def raw(self, v):
        if not self.fq2:
            return v * self.R % self.q
        return (v[0] * self.R % self.q) | ((v[1] * self.R % self.q) << (32 * self.nw))

    def val(self, w):
        """raw limbs -> value, None if a component is not below q"""
        if not self.fq2:
            return w * self.Ri % self.q if w < self.q else None
        lo, hi = w & ((1 << (32 * self.nw)) - 1), w >> (32 * self.nw)
        return (lo * self.Ri % self.q, hi * self.Ri % self.q) if lo < self.q and hi < self.q else None

    def xyzz(self, pt, lam):
        """affine value point -> XYZZ raw words (x lam^2, y lam^3, lam^2, lam^3); None -> all zero"""
        if pt is None:
            return [0, 0, 0, 0]
        F = self.F
        l2 = F.mul(lam, lam)
        l3 = F.mul(l2, lam)
        return [self.raw(v) for v in (F.mul(pt[0], l2), F.mul(pt[1], l3), l2, l3)]

    def affine(self, pt):
        return [0, 0] if pt is None else [self.raw(pt[0]), self.raw(pt[1])]

    def check_xyzz(self, words, want):
        """XYZZ raw words against an affine value point: identity <=> ZZ == 0, else ZZ^3 == ZZZ^2, X/ZZ, Y/ZZZ"""
        F = self.F
        v = [self.val(w) for w in words]
        if any(x is None for x in v):
            return False
        X, Y, ZZ, ZZZ = v
        if want is None:
            return F.is_zero(ZZ)
        if F.is_zero(ZZ) or F.mul(F.mul(ZZ, ZZ), ZZ) != F.mul(ZZZ, ZZZ):
            return False
        return (F.mul(X, F.inv(ZZ)), F.mul(Y, F.inv(ZZZ))) == tuple(want)


@functools.lru_cache(None)
def _group(curve, g2):
    return _Group(curve, g2)


def _pt_case(name, curve, grp, opname):
    g = _group(curve, grp == "g2")
    F, G = g.F, g.G
    rng = random.Random(f"{curve}:{grp}:{opname}")
    pool = g.pool(f"{curve}:{grp}")
    rpt = lambda: rng.choice(pool)
    Pp, Q = rng.sample(pool, 2)
    P2, Pn = G.dbl(Pp), G.neg(Pp)
    lams = [F.one, F.neg(F.one), F.add(F.one, F.one), g.rand(rng)]
    # (0, sqrt(b)) where it exists: x == 0 on a finite point (not on BW6-761's G1: b = -1 is a non-residue, q = 3 mod 4;
    # (0, 2) on its G2, b = 4); (x, 0): a point whose doubling is the identity (off the curve, but the doubling and
    # addition formulas never read b)
    y0 = F.sqrt(G.b)
    specials = [(F.zero, y0)] if y0 is not None else []
    T = (g.rand(rng), F.zero)
    accs = [(None, F.one)] + [(pt, lam) for pt in [Pp, Q, P2, Pn] + specials for lam in lams]
    addends = [None, Pp, Pn, Q, P2] + specials
    ew = g.ew
    vecs, want = [], []   # vecs: list of input word lists (coordinate-sized ints, scalars as raw 8-word ints)

    if opname in ("madd", "madd_neg", "madd_lazy", "madd_lazy_neg"):
        neg = opname.endswith("_neg")
        pairs = [(a, b) for a in accs for b in addends] + [((T, lam), T) for lam in lams]
        for _ in range(64):
            a = rpt()
            b = a if rng.random() < 0.125 else rpt()
            pairs.append(((a, g.rand(rng)), G.neg(b) if neg and rng.random() < 0.125 else b))
        for (a, lam), b in pairs:
            vecs.append(g.xyzz(a, lam) + g.affine(b))
            want.append(G.add(a, G.neg(b) if neg else b))
        sizes = [ew] * 6
    elif opname == "add":
        mus = [F.one, g.rand(rng)]
        pairs = [(a, (b, mu)) for a in accs for b in addends for mu in mus]
        pairs += [((T, lam), (T, mu)) for lam in lams for mu in mus]
        for _ in range(64):
            a = rpt()
            b = a if rng.random() < 0.125 else rpt()
            pairs.append(((a, g.rand(rng)), (b, g.rand(rng))))
        for (a, lam), (b, mu) in pairs:
            vecs.append(g.xyzz(a, lam) + g.xyzz(b, mu))
            want.append(G.add(a, b))
        sizes = [ew] * 8
    elif opname == "dbl_inplace":
        for a, lam in accs + [(T, lam) for lam in lams] + [(rpt(), g.rand(rng)) for _ in range(16)]:
            vecs.append(g.xyzz(a, lam))
            want.append(G.dbl(a))
        sizes = [ew] * 4
    elif opname == "dbl_affine":
        for a in addends + [T] + [rpt() for _ in range(16)]:
            vecs.append(g.affine(a))
            want.append(G.dbl(a))
        sizes = [ew] * 2
    elif opname == "mul_u32":
        # scalars of Fr::N words, as the engine's proof tail passes them: all ones below the top bit of r, all ones in
        # every word, r and its neighbours, random values over the whole width
        r, sb = g.r, 32 * g.sw
        top = (1 << 255) - 1 if g.sw == 8 else (1 << (r.bit_length() - 1)) - 1
        ks = [0, 1, 2, r - 1, r, r + 1, top, (1 << sb) - 1] + [rng.randrange(1 << sb) for _ in range(6)]
        for a, lam in [(None, F.one), (Pp, F.one), (Pp, g.rand(rng)), (Q, F.neg(F.one))]:
            for k in ks:
                vecs.append(g.xyzz(a, lam) + [k])
                want.append(G.mul(a, k))
        sizes = [ew] * 4 + [g.sw]
    elif opname == "to_affine":
        pts = accs + [(rpt(), g.rand(rng)) for _ in range(64)]
        for a, lam in pts:
            vecs.append(g.xyzz(a, lam))
            want.append(a)
        return _exact_case(name, g.fid, TO_AFFINE, [[v[i] for v in vecs] for i in range(4)],
                           [x | (y << (32 * ew)) for x, y in (g.affine(a) for a in want)], [ew] * 4, 2 * ew)
    else:
        raise KeyError(opname)

    inp = np.hstack([_pack([v[i] for v in vecs], w) for i, w in enumerate(sizes)])

    def check(out):
        words = [_unpack(out[:, i * ew:(i + 1) * ew]) for i in range(4)]
        return np.array([i for i in range(len(want)) if not g.check_xyzz([w[i] for w in words], want[i])], dtype=np.int64)

    def describe(i, out):
        ins = " ".join(f"{x:x}" for x in vecs[i])
        got = " ".join(f"{x:x}" for x in _unpack(out[i:i + 1, :].reshape(4, ew)))
        return f"#{i}: in {ins}  got XYZZ {got}  want affine value {want[i]}"
    return Case(name, g.fid, POINT_OPS[opname], inp, check, describe)


@functools.lru_cache(None)
def _case(name):
    kind, field, opname = name.split("-")
    if kind == "fp":
        case, floor = _fp_case(name, field, opname), MIN_FP[opname]
    elif kind == "fq2":
        case, floor = _fq2_case(name, field, opname), MIN_FQ2[opname]
    else:
        curve, grp = field.rsplit("_", 1)
        case, floor = _pt_case(name, curve, grp, opname), MIN_POINT[opname]
    assert len(case) >= floor, f"{name}: {len(case)} vectors, fewer than the {floor} this test promises"
    return case


# ------------------------------------------------------------------------------------------------------------------
# the three builds
# ------------------------------------------------------------------------------------------------------------------
class ArithLib:
    BACKENDS = {0: "host_u64", 1: "emulated_ptx", 2: "device"}

    def __init__(self, path, backend):
        self.lib = C.CDLL(path)
        self.lib.g16t_backend.restype = C.c_int
        self.lib.g16t_shape.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        self.lib.g16t_run.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int64]
        self.lib.g16t_run.restype = C.c_int
        got = self.BACKENDS.get(self.lib.g16t_backend())
        assert got == backend, f"{path} is the {got} build, expected {backend}"

    def run(self, case):
        """validates the whole input here, so that nothing the library reads or writes can fall outside the arrays"""
        iw, ow = C.c_int(), C.c_int()
        assert self.lib.g16t_shape(case.fid, case.op, C.byref(iw), C.byref(ow)) == 0, case.name
        inp = case.inp
        n = inp.shape[0]
        assert inp.dtype == np.uint32 and inp.flags.c_contiguous and inp.shape == (n, iw.value), (case.name, inp.shape, iw)
        if case.op == MUL_SMALL:
            assert (inp[:, -1] < 64).all()          # Fp::mul_small loops over the bits of a non-negative int
        if case.op == BA_INV:
            assert (inp[:, -1] <= 1).all()
        out = np.zeros((n, ow.value), dtype=np.uint32)
        rc = self.lib.g16t_run(case.fid, case.op, inp.ctypes.data, out.ctypes.data, n)
        assert rc == 0, f"{case.name}: g16t_run returned {rc}"
        return out


HOST_BUILDS = {"host_u64": [], "emulated_ptx": ["-DG16_EMULATE_PTX"]}


@pytest.fixture(scope="module")
def host_libs(tmp_path_factory):
    d = tmp_path_factory.mktemp("arith")
    procs = {}
    for name, flags in HOST_BUILDS.items():
        so = str(d / f"libg16arith_{name}.so")
        cmd = ["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", SRC, "-o", so] + flags
        procs[name] = (so, subprocess.Popen(cmd, stderr=subprocess.PIPE, text=True))
    libs = {}
    for name, (so, pr) in procs.items():
        _, err = pr.communicate()
        assert pr.returncode == 0, err
        libs[name] = ArithLib(so, name)
    return libs


@pytest.fixture(scope="module")
def device_lib():
    deps = [SRC, os.path.join(ARITH, "Makefile")] + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h"))
    newest = max(os.path.getmtime(p) for p in deps)
    if not os.path.exists(DEVICE_LIB) or os.path.getmtime(DEVICE_LIB) < newest:
        if shutil.which("nvcc") is None:
            pytest.fail(f"{DEVICE_LIB} is missing or older than its sources, and nvcc is not available to rebuild it: "
                        "run __graft_entry__.build()")
        subprocess.check_call(["make", "-s", "-C", ARITH])
    return ArithLib(DEVICE_LIB, "device")


def _verify(lib, name):
    case = _case(name)
    out = lib.run(case)
    bad = case.check(out)
    if len(bad):
        lines = "\n".join(case.describe(int(i), out) for i in bad[:4])
        pytest.fail(f"{name}: {len(bad)} of {len(case)} vectors differ from the big-integer result; first ones:\n{lines}")


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("backend", list(HOST_BUILDS))
def test_arith_host(host_libs, backend, name):
    """the plain host back-end and the device algorithm under emulated PTX carries, every vector"""
    _verify(host_libs[backend], name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_arith_device(device_lib, name):
    """the sm_90a build: inline-asm carry chains, mont_mul_call for the base fields, ba_ld's __ldg loads"""
    _verify(device_lib, name)


def test_vector_counts():
    """every case meets its floor (asserted in _case); the counts are printed for the record"""
    counts = {name: len(_case(name)) for name in CASES}
    for name, n in counts.items():
        print(f"{name:40s} {n:8d}")
    print(f"total {sum(counts.values())} vectors in {len(counts)} cases")
