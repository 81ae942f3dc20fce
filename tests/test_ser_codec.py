"""Point by point checks of the proving-key point codec (csrc/ser.cuh: ser_decode, ser_encode, ser_sqrt) on all four curves,
against groth16_b200.serialize.ArkCodec, _sqrt_fq and _Fq2, byte for byte and result code for result code.

tests/arith/arith_ops.cu runs the templates of ser.cuh themselves in the three builds of tests/test_arith_ops.py: the plain
host back-end and the emulated-PTX build (CPU tests) and the sm_90a device build libg16arith.so (GPU tests), which alone runs
the inline-PTX carry chains under the codec's square roots, its pow and its subgroup double-and-add.  Decoding runs on G1 of
fields 1, 3, 5, 10 and on G2 of fields 6, 7, 8, 10 (BW6-761's G2 is over Fq), every case in all four flag combinations
(compressed or not, subgroup check or not).  The cases:
  * random subgroup points, the identity, -G, x = 0 and y = 0 points, cofactor torsion [r]T0 and Q + T, each encoded and
    decoded, and every single malformation of a good encoding (every flag error, x >= q, the spare bits under BW6-761's
    and BLS12-377's SWFlags, an off-curve point, an x with no curve point);
  * Fq2 square roots of elements with c1 = 0, which random points never reach: G2 points whose x^3 + b' lies in Fq, with a
    root in Fq (y = (t, 0): the sign falls through to c0) and without one (y = t u);
  * BLS12-377's Tonelli-Shanks at every order 2^k of a^t, k = 0 .. 46, directly and through the Fq2 root;
  * the sign boundary: y = (q -+ 1) / 2 through the encoder, and the curve points of G1 closest to it from each side through
    the decoder (x from a cube root: y^2 - b must be a cube);
  * the general Fq2 root with both of its branches, (a0 + alpha) / 2 and the (a0 - alpha) / 2 fallback.
Each curve has floors, in the style of test_arith_ops.py's MIN_FP: every result code the curve can produce, every
square-root branch and a minimum number of vectors, so that a change to the generator cannot quietly shrink coverage."""
import collections
import functools
import io
import random

import numpy as np
import pytest

import bw6_ref as ref
import pyref as P
from groth16_b200.params import GENERATORS
from groth16_b200.serialize import ArkCodec, DeserializeError, _sqrt_fq
from test_arith_ops import HOST_BUILDS, Case, _pack, _unpack, device_lib, host_libs  # noqa: F401 (fixtures)

CURVES = ("bls12_381", "bn254", "bls12_377", "bw6_761")
BW6 = "bw6_761"
# arith_ops.cu: the field ids of each curve's G1 and G2 coordinates, and the codec's op ids
FIELDS = {"bls12_381": (1, 6), "bn254": (3, 7), "bls12_377": (5, 8), "bw6_761": (10, 10)}
SER_DECODE_G1, SER_DECODE_G2, SER_ENCODE_G1, SER_ENCODE_G2, SQRT = range(30, 35)
COMPRESSED, VALIDATE = 1, 2   # G16_SER_*
REASONS = {1: "compression flag mismatch", 2: "both SWFlags set", 3: "non-zero bytes in the encoding of the point at infinity",
           4: "sort flag set on an uncompressed point", 5: "non-canonical field element (>= q)",
           6: "x is not the abscissa of a curve point", 7: "point is not on the curve",
           8: "point is not in the prime-order subgroup"}
CODE = {v: k for k, v in REASONS.items()}
TS_S = 46   # 2-adicity of BLS12-377's q - 1

# floors per curve: result codes (4 only in the zcash format of BLS12-381, 1 too; 2 only in the generic SWFlags format),
# square-root branches (sqrt: direct SQRT vectors, decode: the root of x^3 + b of a compressed decode), sign-boundary
# vectors and the number of vectors over all of the curve's cases
_FP_BRANCHES = {"fp-root", "fp-none"}
_FQ2_BRANCHES = {"fq2-c1zero-real", "fq2-c1zero-tu", "fq2-plus", "fq2-minus", "fq2-none"}
_SIGN = {"sign:enc-below", "sign:enc-above", "sign:dec-below", "sign:dec-above"}
_SIGN_FQ2 = {"sign:enc-c1-below", "sign:enc-c1-above", "sign:enc-c0-below", "sign:enc-c0-above"}


def _floor_labels(curve):
    codes = {0, 1, 3, 4, 5, 6, 7, 8} if curve == "bls12_381" else {0, 2, 3, 5, 6, 7, 8}
    want = {f"code:{c}" for c in codes} | _SIGN
    branches = set(_FP_BRANCHES) | (_FQ2_BRANCHES if curve != BW6 else set())
    want |= {f"{w}:{b}" for w in ("sqrt", "decode") for b in branches}
    if curve != BW6:
        want |= _SIGN_FQ2
    if curve == "bls12_377":
        want |= {f"sqrt:ts-order-{k}" for k in range(TS_S + 1)}
    return want


MIN_VECTORS = {"bls12_381": 600, "bn254": 540, "bls12_377": 950, "bw6_761": 500}


# ------------------------------------------------------------------------------------------------------------------
# field helpers
# ------------------------------------------------------------------------------------------------------------------
def _cbrt(a, p):
    """a cube root of a in Fp (p = 1 mod 3), or None: Adleman-Manders-Miller with a base-3 discrete log in the 3-Sylow
    subgroup"""
    a %= p
    if a == 0:
        return 0
    if pow(a, (p - 1) // 3, p) != 1:
        return None
    s, t = 0, p - 1
    while t % 3 == 0:
        s, t = s + 1, t // 3
    z = 2
    while pow(z, (p - 1) // 3, p) == 1:
        z += 1
    g = pow(z, t, p)                      # order 3^s
    w = pow(g, 3 ** (s - 1), p)           # a primitive cube root of unity
    x = pow(a, pow(3, -1, t), p)          # x^3 = a b with b in the 3-Sylow subgroup, a cube there: b = g^j, 3 | j
    b = pow(x, 3, p) * pow(a, -1, p) % p
    gi, j = pow(g, -1, p), 0
    for i in range(s):
        c = pow(b * pow(gi, j, p) % p, 3 ** (s - 1 - i), p)
        j += (0 if c == 1 else 1 if c == w else 2) * 3 ** i
    x = x * pow(gi, j // 3, p) % p
    assert pow(x, 3, p) == a
    return x


def _ts_order(a, q):
    """k such that a^t has order exactly 2^k (t the odd part of q - 1)"""
    b, k = pow(a, (q - 1) >> TS_S, q), 0
    while b != 1:
        b, k = b * b % q, k + 1
    return k


def _branch(k: ArkCodec, a, fq2):
    """the square-root branch ser_sqrt (and _sqrt_fq / _Fq2.sqrt) takes for a"""
    q = k.q
    if not fq2:
        return "fp-root" if _sqrt_fq(a, q) is not None else "fp-none"
    a0, a1 = a[0] % q, a[1] % q
    if a1 == 0:
        return "fq2-c1zero-real" if _sqrt_fq(a0, q) is not None else "fq2-c1zero-tu"
    alpha = _sqrt_fq((a0 * a0 + k.fq2.nr * a1 * a1) % q, q)
    if alpha is None:
        return "fq2-none"
    return "fq2-plus" if _sqrt_fq((a0 + alpha) * pow(2, -1, q) % q, q) is not None else "fq2-minus"


# ------------------------------------------------------------------------------------------------------------------
# groups in value space: pyref for the pairing curves, bw6_ref for BW6-761
# ------------------------------------------------------------------------------------------------------------------
class Grp:
    """G1 or G2 of a curve: points are (x, y) (Fq2 coordinates as (c0, c1) pairs), None for the identity"""

    def __init__(self, curve, g2):
        self.curve, self.g2 = curve, g2
        self.k = ArkCodec(curve)
        self.q = self.k.q
        self.fq2 = g2 and self.k.g2_fq2            # coordinates are Fq2 pairs
        self.b = self.k.b2 if g2 else self.k.b1
        if curve == BW6:
            self.r = ref.R
            self.gen = GENERATORS[BW6]["g2" if g2 else "g1"]
            self.add, self.neg = ref.add, ref.neg
            self.mul = lambda pt, n: ref.mul_proj(n, pt)
        else:
            c = P.CURVES[curve]
            cx = P.ctx(c)
            G = cx.G2 if g2 else cx.G1
            self.r = c.r
            self.gen = cx.g2_gen() if g2 else cx.g1_gen()
            self.add, self.neg, self.mul = G.add, G.neg, G.mul

    def rhs(self, x):
        """x^3 + b"""
        q = self.q
        if not self.fq2:
            return (x * x * x + self.b) % q
        f = self.k.fq2
        x3 = f.mul(f.mul(x, x), x)
        return ((x3[0] + self.b[0]) % q, (x3[1] + self.b[1]) % q)

    def solve_y(self, x):
        try:
            return self.k._solve_y(x, self.g2)
        except DeserializeError:
            return None


@functools.lru_cache(None)
def _grp(curve, g2):
    return Grp(curve, g2)


def _torsion_points(curve, g2):
    """(T0, -T0, T, Q + T): a full-group point outside the r-torsion, its cofactor part T = [r]T0, and a subgroup point plus
    it; empty when the group has cofactor 1 (BN254 G1)"""
    G = _grp(curve, g2)
    for x0 in range(1, 200):
        x = (x0, 1) if G.fq2 else x0
        y = G.solve_y(x)
        if y is None:
            continue
        T0 = (x, y)
        T = G.mul(T0, G.r)
        if T is None:
            continue                   # in the subgroup already (always so for BN254 G1)
        return [T0, G.neg(T0), T, G.add(G.mul(G.gen, 12345), T)]
    return []


def _special_points(curve, g2):
    """x = 0 points (order 3) and y = 0 points (order 2: x^3 = -b, every cube root) of the full curve group where they
    exist, in coordinates over Fq: BLS12-377's (-1, 0), BW6-761's (1, 0) on G1 and (0, +-2) on G2"""
    G = _grp(curve, g2)
    q = G.q
    zero = (0, 0) if G.fq2 else 0
    out = []
    y = G.solve_y(zero)
    if y is not None:
        out += [(zero, y), G.neg((zero, y))]
    if not G.fq2:
        x = _cbrt(-G.b, q)
        if x is not None:
            w = _cbrt_unity(q)
            out += [(x * w ** i % q, 0) for i in range(3)]
    return out


def _cbrt_unity(q):
    z = 2
    while pow(z, (q - 1) // 3, q) == 1:
        z += 1
    return pow(z, (q - 1) // 3, q)


def _c1_zero_points(curve, each=3):
    """G2 points over Fq2 whose x^3 + b' lies in Fq, `each` with a root in Fq (y = (t, 0)) and `each` without (y = t u).
    With u^2 = -NR and x = x0 + x1 u, the c1 of x^3 + b' is 3 x0^2 x1 - NR x1^3 + b'_1: zero for x0^2 = (NR x1^3 - b'_1) /
    (3 x1), one square root in Fq per x1 = 1, 2, ..."""
    G = _grp(curve, True)
    q, nr, b1 = G.q, G.k.fq2.nr, G.b[1]
    out = {"fq2-c1zero-real": [], "fq2-c1zero-tu": []}
    for x1 in range(1, 400):
        if min(len(v) for v in out.values()) >= each:
            break
        x0 = _sqrt_fq((nr * x1 ** 3 - b1) * pow(3 * x1, -1, q) % q, q)
        if x0 is None:
            continue
        for x0s in (x0, (-x0) % q):
            x = (x0s, x1)
            rhs = G.rhs(x)
            assert rhs[1] == 0
            kind = _branch(G.k, rhs, True)
            if len(out[kind]) < each:
                out[kind].append((x, G.solve_y(x)))
    assert min(len(v) for v in out.values()) >= each, out
    return out


def _sign_boundary_points(curve):
    """the G1 points with y closest to (q - 1) / 2 from below (y <= (q - 1) / 2: y < -y) and from above: y stepped outward
    until y^2 - b is a cube, x its cube root"""
    G = _grp(curve, False)
    q = G.q
    h = (q - 1) // 2
    out = {}
    for side, y0, step in (("below", h, -1), ("above", h + 1, 1)):
        y = y0
        while True:
            x = _cbrt(y * y - G.b, q)
            if x is not None:
                break
            y += step
        out[side] = (x, y)
    return out


# ------------------------------------------------------------------------------------------------------------------
# vectors
# ------------------------------------------------------------------------------------------------------------------
Vec = collections.namedtuple("Vec", "curve g2 op flags arg want labels")
# op "D": arg = encoding bytes, want = (code, point or None);  "E": arg = point or None, want = bytes;
# "S": arg = field element (g2: the curve's G2 coordinate field), want = root or None


def _decode_want(G: Grp, raw: bytes, flags):
    k = ArkCodec(G.curve, check_subgroup=bool(flags & VALIDATE))
    try:
        return 0, k.read_point(io.BytesIO(raw), G.g2, bool(flags & COMPRESSED))
    except DeserializeError as e:
        return CODE[str(e)], None


def _decode_vec(G: Grp, raw, flags, labels=()):
    code, pt = _decode_want(G, bytes(raw), flags)
    labels = {f"code:{code}", *labels}
    if flags & COMPRESSED and code in (0, 6, 8) and not (raw[0 if G.k.zcash else -1] & 0x40):
        x = pt[0] if pt is not None else _read_x(G, raw)
        labels.add("decode:" + _branch(G.k, G.rhs(x), G.fq2))
    return Vec(G.curve, G.g2, "D", flags, bytes(raw), (code, pt), labels)


def _read_x(G: Grp, raw):
    """x of a compressed encoding whose flags and canonical checks passed"""
    nb = G.k.fq_bytes
    b = bytearray(raw)
    if G.k.zcash:
        b[0] &= 0x1F
        vals = [int.from_bytes(b[i:i + nb], "big") for i in range(0, len(b), nb)]
        return (vals[1], vals[0]) if G.fq2 else vals[0]
    b[-1] &= 0x3F
    vals = [int.from_bytes(b[i:i + nb], "little") for i in range(0, len(b), nb)]
    return (vals[0], vals[1]) if G.fq2 else vals[0]


def _encode_vec(G: Grp, pt, flags, labels=()):
    return Vec(G.curve, G.g2, "E", flags, pt, G.k.point(pt, G.g2, bool(flags & COMPRESSED)), set(labels))


def _sqrt_vec(G: Grp, a, labels=()):
    root = G.k.fq2.sqrt(a) if G.fq2 else _sqrt_fq(a, G.q)
    return Vec(G.curve, G.g2, "S", 0, a, root, {"sqrt:" + _branch(G.k, a, G.fq2), *labels})


def _malformations(G: Grp, good: bytes, compress):
    """each single malformation of a good encoding"""
    k, q, nb = G.k, G.q, G.k.fq_bytes
    inf_enc = k.point(None, G.g2, compress)
    bad = []
    if k.zcash:
        b = bytearray(good); b[0] ^= 0x80; bad.append(b)                       # compression flag
        b = bytearray(good); b[0] |= 0x40; bad.append(b)                       # infinity flag on a real point
        b = bytearray(inf_enc); b[0] |= 0x20; bad.append(b)                    # infinity + sort flag
        b = bytearray(inf_enc); b[-1] = 1; bad.append(b)                       # infinity + payload
        if not compress:
            b = bytearray(good); b[0] |= 0x20; bad.append(b)                   # sort flag uncompressed
        # x >= q in the first wire value (x.c1 for G2): q itself and the largest 381-bit value
        for v in (q, (1 << 381) - 1):
            b = bytearray(good); fl = b[0] & 0xE0
            b[0:nb] = v.to_bytes(nb, "big"); b[0] = (b[0] & 0x1F) | fl; bad.append(b)
    else:
        b = bytearray(good); b[-1] |= 0xC0; bad.append(b)                      # both SWFlags
        b = bytearray(good); b[-1] = (b[-1] & 0x3F) | 0x40; bad.append(b)      # infinity flag on a real point
        b = bytearray(inf_enc); b[0] = 1; bad.append(b)                        # infinity + payload
        for v in (q, q + 5):
            b = bytearray(good); b[0:nb] = v.to_bytes(nb, "little"); bad.append(b)
        # the spare bits under the flags (bits 377..381 of BLS12-377's last value, 761..765 of BW6-761's), each alone
        top = q.bit_length() % 8
        if 0 < top < 6:
            b = bytearray(good); b[-1] |= 0x3F & ~((1 << top) - 1); bad.append(b)
            for bit in range(top, 6):
                b = bytearray(good); b[-1] |= 1 << bit; bad.append(b)
    if compress:
        for x0 in range(2, 60):        # an x with no curve point
            x = (x0, 0) if G.fq2 else x0
            if G.solve_y(x) is None:
                b = bytearray(k.point((x, (0, 0) if G.fq2 else 0), G.g2, True))
                if k.zcash:
                    b[0] &= ~0x20 & 0xFF
                else:
                    b[-1] &= 0x3F
                bad.append(b)
                break
    return bad


@functools.lru_cache(None)
def _vectors(curve):
    """every vector of one curve"""
    rng = random.Random(f"ser-codec:{curve}")
    out = []
    for g2 in (False, True):
        G = _grp(curve, g2)
        q = G.q
        pts = [G.mul(G.gen, rng.randrange(1, G.r)) for _ in range(3)] + [None, G.mul(G.gen, G.r - 1)]
        pts += _special_points(curve, g2) + _torsion_points(curve, g2)
        c1z = _c1_zero_points(curve) if G.fq2 else {}
        for kind, ps in c1z.items():
            pts += [p for pt in ps for p in (pt, G.neg(pt))]
        sign = {} if g2 else _sign_boundary_points(curve)
        for flags in (0, 1, 2, 3):
            compress = bool(flags & COMPRESSED)
            encs = []
            for pt in pts:
                out.append(_encode_vec(G, pt, flags))
                encs.append(G.k.point(pt, g2, compress))
            for side, pt in sign.items():
                for p in (pt, G.neg(pt)):
                    out.append(_encode_vec(G, p, flags))
                    out.append(_decode_vec(G, G.k.point(p, g2, compress), flags, {f"sign:dec-{side}"}))
            good = G.k.point(pts[0], g2, compress)
            if not compress:                                                   # y + 1: off the curve
                y = pts[0][1]
                y1 = ((y[0] + 1) % q, y[1]) if G.fq2 else (y + 1) % q
                encs.append(G.k.point((pts[0][0], y1), g2, False))
            for raw in encs + [bytes(b) for b in _malformations(G, good, compress)]:
                out.append(_decode_vec(G, raw, flags))
            # the sign boundary through the encoder, on coordinates off the curve (it does not check the curve)
            h = (q - 1) // 2
            for side, v in (("below", h), ("above", h + 1)):
                if not G.fq2:
                    for x in (1, 5):
                        out.append(_encode_vec(G, (x, v), flags, {f"sign:enc-{side}"}))
                else:
                    for x in ((1, 0), (3, 7)):
                        for y in ((0, v), (5, v), (h, v)):
                            out.append(_encode_vec(G, (x, y), flags, {f"sign:enc-c1-{side}"}))
                        out.append(_encode_vec(G, (x, (v, 0)), flags, {f"sign:enc-c0-{side}"}))
        # square roots: edges, random elements and squares, the x^3 + b of every point above and of the c1 = 0 points
        if not G.fq2:
            els = [0, 1, 2, 3, 4, q - 1, q - 2, q - 4, (q - 1) // 2, (q + 1) // 2] + [rng.randrange(q) for _ in range(48)]
            els += [pow(rng.randrange(q), 2, q) for _ in range(16)]
            els += [G.rhs(p[0]) for p in pts if p is not None]
        else:
            f = G.k.fq2
            els = [(0, 0), (1, 0), (0, 1), (q - 1, 0), (0, q - 1), (4, 0), (0, 4), (1, 1), ((q - 1) // 2, (q + 1) // 2)]
            els += [(rng.randrange(q), rng.randrange(q)) for _ in range(48)] + [(rng.randrange(q), 0) for _ in range(16)]
            els += [f.mul(e, e) for e in ((rng.randrange(q), rng.randrange(q)) for _ in range(16))]
            els += [G.rhs(p[0]) for p in pts if p is not None]
        out += [_sqrt_vec(G, a) for a in els]
    if curve == "bls12_377":
        # Tonelli-Shanks at every order of a^t: with c = z^t (z = 5, a non-residue) of order 2^46 and s = v^(2^46) of odd
        # order, a_k = c^(2^(46 - k)) s makes a^t of order exactly 2^k; k = 46 is a non-residue
        G, G2 = _grp(curve, False), _grp(curve, True)
        q = G.q
        t = (q - 1) >> TS_S
        c = pow(5, t, q)
        for rep in range(2):
            s = pow(rng.randrange(1, q), 1 << TS_S, q)
            for kk in range(TS_S + 1):
                a = pow(c, 1 << (TS_S - kk), q) * s % q
                assert _ts_order(a, q) == kk
                out.append(_sqrt_vec(G, a, {f"sqrt:ts-order-{kk}"}))
                # through the Fq2 root: a u^2 = (-NR a, 0), and (a, 0)
                out.append(_sqrt_vec(G2, ((-G2.k.fq2.nr * a) % q, 0)))
                out.append(_sqrt_vec(G2, (a, 0)))
        out += [_sqrt_vec(G, a) for a in (0, 1, q - 1, 4)]
    return out


# ------------------------------------------------------------------------------------------------------------------
# vectors -> harness cases
# ------------------------------------------------------------------------------------------------------------------
def _words(G: Grp):
    """u32 words of one coordinate"""
    return G.k.fq_bytes // 4 * (2 if G.fq2 else 1)


def _coords(G: Grp, pt):
    """canonical x || y as ints of C words each (Fq2: c0 low, c1 high); the identity is zero"""
    if pt is None:
        return [0, 0]
    if not G.fq2:
        return [pt[0] % G.q, pt[1] % G.q]
    sh = 8 * G.k.fq_bytes
    return [v[0] % G.q | (v[1] % G.q) << sh for v in pt]


def _field_int(G: Grp, a):
    return a % G.q if not G.fq2 else a[0] % G.q | (a[1] % G.q) << (8 * G.k.fq_bytes)


def _pad(raw: bytes, nbytes):
    return int.from_bytes(bytes(raw) + bytes(nbytes - len(raw)), "little")


CASE_NAMES = [f"{c}-{g}-{op}" for c in CURVES for g in ("g1", "g2") for op in ("decode", "encode", "sqrt")]


@functools.lru_cache(None)
def _case(name):
    curve, grp, opname = name.split("-")
    g2 = grp == "g2"
    G = _grp(curve, g2)
    C = _words(G)
    kind = {"decode": "D", "encode": "E", "sqrt": "S"}[opname]
    vecs = [v for v in _vectors(curve) if v.g2 == g2 and v.op == kind]
    fid = FIELDS[curve][g2]
    flags = np.array([[v.flags if kind != "S" else 0] for v in vecs], dtype=np.uint32)
    if kind == "D":
        op = SER_DECODE_G2 if g2 else SER_DECODE_G1
        inp = np.hstack([flags, _pack([_pad(v.arg, 8 * C) for v in vecs], 2 * C)])
        want = np.hstack([np.array([[v.want[0]] for v in vecs], dtype=np.uint32),
                          _pack([c for v in vecs for c in _coords(G, v.want[1])], C).reshape(len(vecs), 2 * C)])
    elif kind == "E":
        op = SER_ENCODE_G2 if g2 else SER_ENCODE_G1
        inp = np.hstack([flags, _pack([c for v in vecs for c in _coords(G, v.arg)], C).reshape(len(vecs), 2 * C)])
        want = _pack([_pad(v.want, 8 * C) for v in vecs], 2 * C)
    else:
        op = SQRT
        inp = _pack([_field_int(G, v.arg) for v in vecs], C)
        want = np.hstack([np.array([[v.want is not None] for v in vecs], dtype=np.uint32),
                          _pack([0 if v.want is None else _field_int(G, v.want) for v in vecs], C)])
    inp = np.ascontiguousarray(inp, dtype=np.uint32)

    def check(out):
        return np.nonzero((out != want).any(axis=1))[0]

    def describe(i, out):
        v = vecs[i]
        return (f"#{i} flags {v.flags} {sorted(v.labels)}: in {_unpack(inp[i:i + 1])[0]:x}\n"
                f"    got  {_unpack(out[i:i + 1])[0]:x}\n    want {_unpack(want[i:i + 1])[0]:x}")
    return Case(name, fid, op, inp, check, describe)


def _verify(lib, name):
    case = _case(name)
    out = lib.run(case)
    bad = case.check(out)
    if len(bad):
        lines = "\n".join(case.describe(int(i), out) for i in bad[:4])
        pytest.fail(f"{name}: {len(bad)} of {len(case)} vectors differ from ArkCodec; first ones:\n{lines}")


# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
def test_codec_coverage_floors(curve):
    """every result code the curve can produce, every square-root branch, both sides of the sign boundary, a minimum
    vector count"""
    vecs = _vectors(curve)
    seen = collections.Counter(lab for v in vecs for lab in v.labels)
    missing = _floor_labels(curve) - set(seen)
    assert not missing, f"{curve}: no vector reaches {sorted(missing)}"
    assert len(vecs) >= MIN_VECTORS[curve], f"{curve}: {len(vecs)} vectors, fewer than the {MIN_VECTORS[curve]} promised"
    print(f"{curve}: {len(vecs)} vectors; " + ", ".join(f"{k} {n}" for k, n in sorted(seen.items())))


@pytest.mark.parametrize("name", CASE_NAMES)
@pytest.mark.parametrize("backend", list(HOST_BUILDS))
def test_codec_host(host_libs, backend, name):
    """the plain host back-end and the device algorithm under emulated PTX carries, every vector"""
    _verify(host_libs[backend], name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_NAMES)
def test_codec_device(device_lib, name):
    """the sm_90a build of the codec: every vector, identical answers"""
    _verify(device_lib, name)
