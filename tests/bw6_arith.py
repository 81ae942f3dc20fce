"""Driver of tests/arith_bw6/bw6_arith.cu: BW6-761's Fr (12 limbs) and Fq (24 limbs), the safegcd inversion and the XYZZ
point operations, at carry-chain edge operands, against Python big integers.  `check_all(lib)` runs every case on one build
of the harness (host CIOS, emulated PTX, or the device) and returns the list of mismatches."""
import ctypes as C
import random

import numpy as np

import bw6_ref as ref

FR, FQ = 0, 1
ADD, SUB, NEG, DBL, MUL, SQR, FROM_MONT, TO_MONT, INV, INV_GCD = range(10)
MADD, MADD_LAZY, PADD, PDBL = 20, 21, 22, 23
MOD = {FR: ref.R, FQ: ref.Q}
NLIMBS = {FR: 12, FQ: 24}


def load(path):
    lib = C.CDLL(path)
    lib.bw6t_shape.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.bw6t_run.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int64]
    return lib


def edges(p, n):
    """raw limb values below p that stress the carry chains: limb boundaries, p - small, halves, Montgomery constants"""
    R = 1 << (32 * n)
    out = {0, 1, 2, 3, p - 1, p - 2, p - 3, (p - 1) // 2, (p + 1) // 2, R % p, (R - 1) % p, R * R % p, pow(R, -1, p),
           (p - 1) // 2 + 1}
    for k in range(31, 32 * n, 32):
        for v in (1 << k, (1 << k) - 1, (1 << (k + 1)) - 1, p - (1 << k)):
            if 0 <= v < p:
                out.add(v)
    rng = random.Random(p & 0xFFFF)
    out |= {rng.randrange(p) for _ in range(8)}
    return sorted(out)


def run(lib, field, op, vecs, in_words, out_words):
    a = np.ascontiguousarray(np.array(vecs, dtype=np.uint32).reshape(-1, in_words))
    out = np.zeros((a.shape[0], out_words), dtype=np.uint32)
    assert lib.bw6t_run(field, op, a.ctypes.data, out.ctypes.data, a.shape[0]) == 0
    return out


def limbs(v, n):
    return [(v >> (32 * i)) & 0xFFFFFFFF for i in range(n)]


def value(ws):
    return sum(int(w) << (32 * i) for i, w in enumerate(ws))


def check_fields(lib):
    bad = []
    for field in (FR, FQ):
        p, n = MOD[field], NLIMBS[field]
        R = 1 << (32 * n)
        Ri = pow(R, -1, p)
        ev = edges(p, n)
        pairs = [(a, b) for a in ev for b in ev]
        vec = [limbs(a, n) + limbs(b, n) for a, b in pairs]
        want = {
            ADD: lambda a, b: (a + b) % p, SUB: lambda a, b: (a - b) % p, NEG: lambda a, b: (-a) % p,
            DBL: lambda a, b: 2 * a % p, MUL: lambda a, b: a * b * Ri % p, SQR: lambda a, b: a * a * Ri % p,
            FROM_MONT: lambda a, b: a * Ri % p, TO_MONT: lambda a, b: a * R % p,
            INV: lambda a, b: 0 if a == 0 else R * R * pow(a, -1, p) % p,
            INV_GCD: lambda a, b: 0 if a == 0 else R * R * pow(a, -1, p) % p,
        }
        for op, fn in want.items():
            unary = op in (NEG, DBL, SQR, FROM_MONT, TO_MONT, INV, INV_GCD)
            ps = [(a, 0) for a in ev] if unary else pairs
            vs = [limbs(a, n) + limbs(b, n) for a, b in ps] if unary else vec
            got = run(lib, field, op, vs, 2 * n, n)
            for (a, b), g in zip(ps, got):
                if value(g) != fn(a, b):
                    bad.append((field, op, a, b))
    return bad


def _mont(v):
    return v * (1 << 768) % ref.Q


def _xyzz(P, lam):
    """XYZZ of affine P with the scale lam (identity: all zero)"""
    if P is None:
        return [0, 0, 0, 0]
    q = ref.Q
    return [P[0] * lam * lam % q, P[1] * pow(lam, 3, q) % q, lam * lam % q, pow(lam, 3, q)]


def _affine_of(ws):
    q = ref.Q
    Ri = pow(1 << 768, -1, q)
    X, Y, ZZ, ZZZ = (value(ws[24 * k:24 * k + 24]) * Ri % q for k in range(4))
    if ZZ == 0:
        return None
    return X * pow(ZZ, -1, q) % q, Y * pow(ZZZ, -1, q) % q


def check_points(lib):
    """madd (inlined and lazily loaded), add and dbl in XYZZ over BW6's Fq, with the exceptional cases: P = Q, P = -Q,
    either operand the identity, and points of both groups (the formulas never read b)"""
    from groth16_b200.params import GENERATORS
    bad = []
    rng = random.Random(5)
    enc = lambda vals: sum((limbs(_mont(v), 24) for v in vals), [])
    for gname in ("g1", "g2"):
        G = GENERATORS["bw6_761"][gname]
        pts = [None, G, ref.neg(G), ref.mul(2, G), ref.mul(ref.R - 1, G)] + [ref.mul(rng.randrange(ref.R), G) for _ in range(4)]
        cases = [(P, Q) for P in pts for Q in pts]
        lam = lambda: rng.randrange(1, ref.Q)
        for op in (MADD, MADD_LAZY, PADD):
            vecs = []
            for P, Q in cases:
                second = (_xyzz(Q, lam()) if op == PADD else ([0, 0] if Q is None else [Q[0], Q[1]]) + [0, 0])
                vecs.append(enc(_xyzz(P, lam())) + enc(second))
            got = run(lib, FQ, op, vecs, 192, 96)
            for (P, Q), g in zip(cases, got):
                if _affine_of(g) != ref.add(P, Q):
                    bad.append((gname, op, P, Q))
        vecs = [enc(_xyzz(P, lam())) + [0] * 96 for P in pts]
        got = run(lib, FQ, PDBL, vecs, 192, 96)
        for P, g in zip(pts, got):
            if _affine_of(g) != ref.add(P, P):
                bad.append((gname, PDBL, P))
    return bad


def check_all(lib):
    return check_fields(lib) + check_points(lib)
