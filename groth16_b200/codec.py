"""Python ints <-> the C-ABI memory image (little-endian u64 limbs, Montgomery form), include/g16b200.h.

ark-ff keeps every Fp as a*R mod p with R = 2^(64*N64); scalars handed to an MSM are canonical BigInt<4>
(prover.rs:64,71,82).  Points: affine x||y, infinity = all-zero limbs; G2 coordinates are c0||c1."""
from __future__ import annotations

import numpy as np

from .params import CurveParams


def _nl(p: int) -> int:
    return (p.bit_length() + 63) // 64


def ints_to_limbs(vals, nl: int) -> np.ndarray:
    """canonical ints -> (len, nl) uint64 little-endian limbs"""
    nb = 8 * nl
    buf = b"".join(int(v).to_bytes(nb, "little") for v in vals)
    return np.frombuffer(buf, dtype="<u8").reshape(-1, nl).copy()


def limbs_to_ints(arr: np.ndarray, nl: int):
    a = np.ascontiguousarray(arr, dtype="<u8").reshape(-1, nl)
    raw = a.tobytes()
    nb = 8 * nl
    return [int.from_bytes(raw[i * nb:(i + 1) * nb], "little") for i in range(a.shape[0])]


class FieldCodec:
    def __init__(self, p: int):
        self.p = p
        self.nl = _nl(p)
        self.R = 1 << (64 * self.nl)
        self.Rinv = pow(self.R, -1, p)

    def enc(self, vals) -> np.ndarray:
        """ints -> Montgomery limbs, shape (len, nl)"""
        p, R = self.p, self.R
        return ints_to_limbs([(int(v) % p) * R % p for v in vals], self.nl)

    def dec(self, arr) -> list:
        p, Ri = self.p, self.Rinv
        return [v * Ri % p for v in limbs_to_ints(arr, self.nl)]

    def enc1(self, v) -> np.ndarray:
        return self.enc([v])[0]

    def bigint(self, vals) -> np.ndarray:
        """ints -> canonical limbs (BigInt<N>)"""
        return ints_to_limbs([int(v) % self.p for v in vals], self.nl)


class CurveCodec:
    """G1 points are (x, y) int tuples or None; G2 points are ((x0, x1), (y0, y1)) or None, or (x, y) when G2 is over Fq
    (BW6-761)."""

    def __init__(self, c: CurveParams):
        self.c = c
        self.fr = FieldCodec(c.r)
        self.fq = FieldCodec(c.q)
        self.nq = self.fq.nl

    def enc_g1(self, pts) -> np.ndarray:
        flat = []
        for P in pts:
            flat.extend((0, 0) if P is None else (P[0], P[1]))
        arr = self.fq.enc(flat).reshape(-1, 2 * self.nq)
        for i, P in enumerate(pts):
            if P is None:
                arr[i, :] = 0
        return arr

    def enc_g2(self, pts) -> np.ndarray:
        if self.c.g2_over_fq:
            return self.enc_g1(pts)
        flat = []
        for P in pts:
            flat.extend((0, 0, 0, 0) if P is None else (P[0][0], P[0][1], P[1][0], P[1][1]))
        arr = self.fq.enc(flat).reshape(-1, 4 * self.nq)
        for i, P in enumerate(pts):
            if P is None:
                arr[i, :] = 0
        return arr

    def dec_g1(self, arr) -> list:
        a = np.ascontiguousarray(arr, dtype="<u8").reshape(-1, 2 * self.nq)
        vals = self.fq.dec(a.reshape(-1, self.nq))
        out = []
        for i in range(a.shape[0]):
            out.append(None if not a[i].any() else (vals[2 * i], vals[2 * i + 1]))
        return out

    def dec_g2(self, arr) -> list:
        if self.c.g2_over_fq:
            return self.dec_g1(arr)
        a = np.ascontiguousarray(arr, dtype="<u8").reshape(-1, 4 * self.nq)
        vals = self.fq.dec(a.reshape(-1, self.nq))
        out = []
        for i in range(a.shape[0]):
            out.append(None if not a[i].any() else ((vals[4 * i], vals[4 * i + 1]), (vals[4 * i + 2], vals[4 * i + 3])))
        return out

    def dec_proj_g1(self, arr):
        """normalised Jacobian X||Y||Z -> affine tuple or None"""
        v = self.fq.dec(np.asarray(arr).reshape(3, self.nq))
        return None if v[2] == 0 else (v[0], v[1])

    def dec_proj_g2(self, arr):
        if self.c.g2_over_fq:
            return self.dec_proj_g1(arr)
        v = self.fq.dec(np.asarray(arr).reshape(6, self.nq))
        return None if (v[4] == 0 and v[5] == 0) else ((v[0], v[1]), (v[2], v[3]))
