"""ark-serialize `CanonicalSerialize` / `CanonicalDeserialize` wire formats for the Groth16 structures
(/root/reference/src/data_structures.rs:8,31,87,125 derive them): Proof, VerifyingKey, ProvingKey.   SURVEY.md section 8f-4.

Two point encodings exist in the arkworks ecosystem:
  * generic short-Weierstrass (ark-ec `Affine<P>`, used by ark-bn254 and ark-bls12-377): field elements little-endian,
    SWFlags in the two top bits of the LAST byte (bit 7: y is "negative" i.e. y > -y, bit 6: point at infinity);
    compressed = x with flags, uncompressed = x || y with flags; Fq2 = c0 || c1 with the flags on c1.
  * ark-bls12-381 overrides it with the zcash / IETF format: big-endian, three flag bits in the FIRST byte (bit 7:
    compressed, bit 6: infinity, bit 5: y lexicographically largest), Fq2 as c1 || c0.
`Vec<T>` is a u64 little-endian length followed by the items; structs are their fields in declaration order.

Status: the BLS12-381 encoder is pinned by the IETF generator encodings (tests/test_serialize.py).  The generic format
is restated from ark-serialize 0.5 semantics and has NOT been checked against an arkworks build (no Rust toolchain here);
oracle/ark_fixture/ is the Rust program whose output settles it (tests/test_ark_fixture.py loads whatever it wrote).
Points are (x, y) Python-int tuples (G2: ((x0, x1), (y0, y1))), identity = None -- the same convention as codec.py.

Validation (ark's `Validate::Yes`): every read checks for truncated input, canonical field elements (< q), that an
uncompressed point satisfies the curve equation and that the unused flag bits are clear; `check_subgroup=True` adds the
r-torsion check ([r]P = O), which costs a scalar multiplication per point in Python and is therefore opt-in.
"""
from __future__ import annotations

import io
from typing import List, Optional

from .params import CurveParams, get_curve

# Fq2 non-residues (u^2 = -NR) and curve coefficients needed to decompress
_FQ2_NR = {"bls12_381": 1, "bn254": 1, "bls12_377": 5}
_G1_B = {"bls12_381": 4, "bn254": 3, "bls12_377": 1, "bw6_761": -1}


def _g2_b(c: CurveParams):
    """G2's coefficient b: an Fq2 pair, or one Fq element when G2 is over Fq (BW6-761: y^2 = x^3 + 4)"""
    q = c.q
    if c.g2_over_fq:
        return 4
    if c.name == "bls12_381":
        return (4, 4)
    if c.name == "bn254":  # 3 / (9 + u)
        n = pow(82, -1, q)
        return (27 * n % q, (-3 * n) % q)
    return (0, 155198655607781456406391640216936120121836107652948796323930557600032281009004493664981332883744016074664192874906)


# ------------------------------------------------------------------------------------------------------------------
# field helpers
# ------------------------------------------------------------------------------------------------------------------
def _sqrt_fq(a: int, p: int) -> Optional[int]:
    a %= p
    if a == 0:
        return 0
    if pow(a, (p - 1) // 2, p) != 1:
        return None
    if p % 4 == 3:
        return pow(a, (p + 1) // 4, p)
    s, t = 0, p - 1
    while t % 2 == 0:
        s, t = s + 1, t // 2
    z = 2
    while pow(z, (p - 1) // 2, p) != p - 1:
        z += 1
    m, c, tt, r = s, pow(z, t, p), pow(a, t, p), pow(a, (t + 1) // 2, p)
    while tt != 1:
        i, t2 = 0, tt
        while t2 != 1:
            t2, i = t2 * t2 % p, i + 1
        b = pow(c, 1 << (m - i - 1), p)
        m, c = i, b * b % p
        tt, r = tt * c % p, r * b % p
    return r


class _Fq2:
    def __init__(self, p, nr):
        self.p, self.nr = p, nr

    def mul(self, a, b):
        p = self.p
        return ((a[0] * b[0] - self.nr * a[1] * b[1]) % p, (a[0] * b[1] + a[1] * b[0]) % p)

    def sqrt(self, a):
        """complex-method square root in Fq[u]/(u^2 + nr)"""
        p = self.p
        a0, a1 = a[0] % p, a[1] % p
        if a1 == 0:
            r = _sqrt_fq(a0, p)
            if r is not None:
                return (r, 0)
            r = _sqrt_fq(a0 * pow(-self.nr, -1, p) % p, p)   # a0 = -nr * t^2  ->  sqrt = t u
            return None if r is None else (0, r)
        norm = (a0 * a0 + self.nr * a1 * a1) % p
        alpha = _sqrt_fq(norm, p)
        if alpha is None:
            return None
        inv2 = pow(2, -1, p)
        delta = (a0 + alpha) * inv2 % p
        x0 = _sqrt_fq(delta, p)
        if x0 is None:
            delta = (a0 - alpha) * inv2 % p
            x0 = _sqrt_fq(delta, p)
            if x0 is None:
                return None
        x1 = a1 * pow(2 * x0, -1, p) % p
        r = (x0, x1)
        return r if self.mul(r, r) == (a0, a1) else None


def _neg_gt(y, p, is_fq2: bool) -> bool:
    """y > -y in ark's ordering (Fq2: compare c1 first, then c0)"""
    if not is_fq2:
        return y % p > (-y) % p
    n = ((-y[0]) % p, (-y[1]) % p)
    return (y[1] % p, y[0] % p) > (n[1], n[0])


# ------------------------------------------------------------------------------------------------------------------
class DeserializeError(ValueError):
    """ark_serialize::SerializationError::InvalidData / UnexpectedFlags / NotEnoughSpace"""


class ArkCodec:
    """serialize / deserialize for one curve"""

    MAX_VEC = 1 << 28   # refuse absurd length prefixes instead of allocating

    def __init__(self, curve, check_subgroup: bool = False):
        self.check_subgroup = check_subgroup
        self.c = get_curve(curve)
        self.q = self.c.q
        self.zcash = self.c.name == "bls12_381"
        self.fq_bytes = (self.q.bit_length() + 2 + 7) // 8 if not self.zcash else 48
        self.g2_fq2 = not self.c.g2_over_fq   # G2 coordinates are Fq2 pairs (otherwise G2 points are encoded like G1's)
        self.fq2 = _Fq2(self.q, _FQ2_NR[self.c.name]) if self.g2_fq2 else None
        self.b1 = _G1_B[self.c.name]
        self.b2 = _g2_b(self.c)

    # ---- scalars ----
    def fr(self, x: int) -> bytes:
        return int(x % self.c.r).to_bytes(8 * self.c.fr_limbs, "little")

    # ---- points ----
    def _coords(self, P, g2):
        """flatten coordinates in wire order (most significant component first for the zcash format)"""
        if not g2:
            return [P[0]], [P[1]]
        if self.zcash:
            return [P[0][1], P[0][0]], [P[1][1], P[1][0]]
        return [P[0][0], P[0][1]], [P[1][0], P[1][1]]

    def point(self, P, g2: bool = False, compress: bool = True) -> bytes:
        nb, q = self.fq_bytes, self.q
        g2 = g2 and self.g2_fq2   # from here on: "the coordinates are Fq2 pairs"
        ncomp = 2 if g2 else 1
        if self.zcash:
            size = nb * ncomp * (1 if compress else 2)
            if P is None:
                out = bytearray(size)
                out[0] = (0x80 if compress else 0) | 0x40
                return bytes(out)
            xs, ys = self._coords(P, g2)
            body = b"".join(int(v % q).to_bytes(nb, "big") for v in (xs if compress else xs + ys))
            out = bytearray(body)
            if compress:
                out[0] |= 0x80
                if _neg_gt(P[1], q, g2):
                    out[0] |= 0x20
            return bytes(out)
        # generic ark-ec encoding
        if P is None:
            out = bytearray(nb * ncomp * (1 if compress else 2))
            out[-1] |= 0x40
            return bytes(out)
        xs, ys = self._coords(P, g2)
        body = bytearray(b"".join(int(v % q).to_bytes(nb, "little") for v in (xs if compress else xs + ys)))
        if _neg_gt(P[1], q, g2):
            body[-1] |= 0x80
        return bytes(body)

    def _read(self, buf, n: int) -> bytearray:
        raw = buf.read(n)
        if len(raw) != n:
            raise DeserializeError(f"truncated input: wanted {n} bytes, got {len(raw)}")
        return bytearray(raw)

    def _on_curve(self, x, y, g2) -> bool:
        q = self.q
        if not g2 or not self.g2_fq2:
            return (y * y - x * x * x - (self.b2 if g2 else self.b1)) % q == 0
        f = self.fq2
        x3 = f.mul(f.mul(x, x), x)
        y2 = f.mul(y, y)
        return (y2[0] - x3[0] - self.b2[0]) % q == 0 and (y2[1] - x3[1] - self.b2[1]) % q == 0

    def _in_subgroup(self, P, g2) -> bool:
        """[r]P == O by double-and-add in affine coordinates (slow; opt-in)"""
        q, r = self.q, self.c.r
        g2 = g2 and self.g2_fq2
        f = self.fq2

        def inv(a):
            if not g2:
                return pow(a, -1, q)
            n = pow((a[0] * a[0] + f.nr * a[1] * a[1]) % q, -1, q)
            return (a[0] * n % q, (-a[1] * n) % q)

        def mul(a, b):
            return f.mul(a, b) if g2 else a * b % q

        def sub(a, b):
            return ((a[0] - b[0]) % q, (a[1] - b[1]) % q) if g2 else (a - b) % q

        def add(A, B):
            if A is None:
                return B
            if B is None:
                return A
            if A[0] == B[0]:
                if A[1] != B[1] or A[1] == ((0, 0) if g2 else 0):
                    return None
                three = (3, 0) if g2 else 3
                two = (2, 0) if g2 else 2
                lam = mul(mul(three, mul(A[0], A[0])), inv(mul(two, A[1])))
            else:
                lam = mul(sub(B[1], A[1]), inv(sub(B[0], A[0])))
            x3 = sub(sub(mul(lam, lam), A[0]), B[0])
            return (x3, sub(mul(lam, sub(A[0], x3)), A[1]))

        acc, base, k = None, P, r
        while k:
            if k & 1:
                acc = add(acc, base)
            base = add(base, base)
            k >>= 1
        return acc is None

    def read_point(self, buf: io.BytesIO, g2: bool = False, compress: bool = True):
        nb, q = self.fq_bytes, self.q
        group2 = g2                 # which curve equation
        g2 = g2 and self.g2_fq2     # the coordinates are Fq2 pairs
        ncomp = 2 if g2 else 1
        raw = self._read(buf, nb * ncomp * (1 if compress else 2))
        if self.zcash:
            flags = raw[0] & 0xE0
            raw[0] &= 0x1F
            if bool(flags & 0x80) != compress:
                raise DeserializeError("compression flag mismatch")
            if flags & 0x40:
                if any(raw) or (flags & 0x20):
                    raise DeserializeError("non-zero bytes in the encoding of the point at infinity")
                return None
            if not compress and (flags & 0x20):
                raise DeserializeError("sort flag set on an uncompressed point")
            vals = [int.from_bytes(raw[i * nb:(i + 1) * nb], "big") for i in range(len(raw) // nb)]
        else:
            flags = raw[-1] & 0xC0
            raw[-1] &= 0x3F
            if flags == 0xC0:
                raise DeserializeError("both SWFlags set")
            if flags & 0x40:
                if any(raw):
                    raise DeserializeError("non-zero bytes in the encoding of the point at infinity")
                return None
            vals = [int.from_bytes(raw[i * nb:(i + 1) * nb], "little") for i in range(len(raw) // nb)]
        if any(v >= q for v in vals):
            raise DeserializeError("non-canonical field element (>= q)")
        if self.zcash:
            x = (vals[1], vals[0]) if g2 else vals[0]
            yraw = ((vals[3], vals[2]) if g2 else vals[1]) if not compress else None
            neg_flag = bool(flags & 0x20)
        else:
            x = (vals[0], vals[1]) if g2 else vals[0]
            yraw = ((vals[2], vals[3]) if g2 else vals[1]) if not compress else None
            neg_flag = bool(flags & 0x80)
        if compress:
            y = self._solve_y(x, group2)
            if _neg_gt(y, q, g2) != neg_flag:
                y = ((-y[0]) % q, (-y[1]) % q) if g2 else (-y) % q
        else:
            y = yraw
            if not self._on_curve(x, y, group2):
                raise DeserializeError("point is not on the curve")
        P = (x, y)
        if self.check_subgroup and not self._in_subgroup(P, group2):
            raise DeserializeError("point is not in the prime-order subgroup")
        return P

    def _solve_y(self, x, g2):
        q = self.q
        if not g2 or not self.g2_fq2:
            y = _sqrt_fq((x * x * x + (self.b2 if g2 else self.b1)) % q, q)
        else:
            f = self.fq2
            x3 = f.mul(f.mul(x, x), x)
            y = f.sqrt(((x3[0] + self.b2[0]) % q, (x3[1] + self.b2[1]) % q))
        if y is None:
            raise DeserializeError("x is not the abscissa of a curve point")
        return y

    # ---- containers ----
    def vec(self, pts: List, g2=False, compress=True) -> bytes:
        return len(pts).to_bytes(8, "little") + b"".join(self.point(P, g2, compress) for P in pts)

    def read_vec(self, buf, g2=False, compress=True) -> List:
        n = int.from_bytes(self._read(buf, 8), "little")
        if n > self.MAX_VEC:
            raise DeserializeError(f"vector length {n} exceeds the limit")
        return [self.read_point(buf, g2, compress) for _ in range(n)]

    def read_fr(self, buf) -> int:
        v = int.from_bytes(self._read(buf, 8 * self.c.fr_limbs), "little")
        if v >= self.c.r:
            raise DeserializeError("non-canonical scalar (>= r)")
        return v

    def read_fr_vec(self, data: bytes) -> List[int]:
        """Vec<Fr>: u64 LE length, then canonical little-endian scalars"""
        buf = io.BytesIO(data)
        n = int.from_bytes(self._read(buf, 8), "little")
        if n > self.MAX_VEC:
            raise DeserializeError(f"vector length {n} exceeds the limit")
        out = [self.read_fr(buf) for _ in range(n)]
        if buf.read(1):
            raise DeserializeError("trailing bytes")
        return out

    def fr_vec(self, xs) -> bytes:
        return len(xs).to_bytes(8, "little") + b"".join(self.fr(x) for x in xs)

    # ---- Groth16 structures (data_structures.rs field order) ----
    def proof(self, a, b, c, compress=True) -> bytes:
        return self.point(a, False, compress) + self.point(b, True, compress) + self.point(c, False, compress)

    def read_proof(self, data: bytes, compress=True):
        buf = io.BytesIO(data)
        out = self.read_point(buf, False, compress), self.read_point(buf, True, compress), self.read_point(buf, False, compress)
        if buf.read(1):
            raise DeserializeError("trailing bytes after the proof")
        return out

    def verifying_key(self, alpha_g1, beta_g2, gamma_g2, delta_g2, gamma_abc_g1, compress=True) -> bytes:
        return (self.point(alpha_g1, False, compress) + self.point(beta_g2, True, compress) + self.point(gamma_g2, True, compress)
                + self.point(delta_g2, True, compress) + self.vec(gamma_abc_g1, False, compress))

    def read_verifying_key(self, buf, compress=True):
        return (self.read_point(buf, False, compress), self.read_point(buf, True, compress), self.read_point(buf, True, compress),
                self.read_point(buf, True, compress), self.read_vec(buf, False, compress))

    def proving_key(self, vk: tuple, beta_g1, delta_g1, a_query, b_g1_query, b_g2_query, h_query, l_query, compress=True) -> bytes:
        return (self.verifying_key(*vk, compress=compress) + self.point(beta_g1, False, compress) + self.point(delta_g1, False, compress)
                + self.vec(a_query, False, compress) + self.vec(b_g1_query, False, compress) + self.vec(b_g2_query, True, compress)
                + self.vec(h_query, False, compress) + self.vec(l_query, False, compress))

    def read_proving_key(self, data: bytes, compress=True):
        buf = io.BytesIO(data)
        vk = self.read_verifying_key(buf, compress)
        beta_g1 = self.read_point(buf, False, compress)
        delta_g1 = self.read_point(buf, False, compress)
        out = (vk, beta_g1, delta_g1, self.read_vec(buf, False, compress), self.read_vec(buf, False, compress),
               self.read_vec(buf, True, compress), self.read_vec(buf, False, compress), self.read_vec(buf, False, compress))
        if buf.read(1):
            raise DeserializeError("trailing bytes after the proving key")
        return out

    # ---- oracle/ark_fixture side files (not arkworks formats: see oracle/ark_fixture/src/main.rs) ----
    def matrices(self, ni: int, nw: int, a_rows, b_rows, c_rows) -> bytes:
        out = bytearray()
        for v in (ni, nw, len(a_rows)):
            out += int(v).to_bytes(8, "little")
        for rows in (a_rows, b_rows, c_rows):
            for row in rows:
                out += len(row).to_bytes(8, "little")
                for coeff, col in row:
                    out += self.fr(coeff) + int(col).to_bytes(8, "little")
        return bytes(out)

    def read_matrices(self, data: bytes):
        """-> (num_instance, num_witness, a_rows, b_rows, c_rows), rows as lists of (coefficient, column)"""
        buf = io.BytesIO(data)
        ni, nw, nc = (int.from_bytes(self._read(buf, 8), "little") for _ in range(3))
        if max(ni, nw, nc) > self.MAX_VEC:
            raise DeserializeError("matrix dimensions exceed the limit")
        mats = []
        for _ in range(3):
            rows = []
            for _ in range(nc):
                ln = int.from_bytes(self._read(buf, 8), "little")
                if ln > ni + nw:
                    raise DeserializeError("row longer than the number of variables")
                row = []
                for _ in range(ln):
                    cf = self.read_fr(buf)
                    col = int.from_bytes(self._read(buf, 8), "little")
                    if col >= ni + nw:
                        raise DeserializeError("column index out of range")
                    row.append((cf, col))
                rows.append(row)
            mats.append(rows)
        if buf.read(1):
            raise DeserializeError("trailing bytes after the matrices")
        return ni, nw, mats[0], mats[1], mats[2]
