"""An independent writer and reader of circom .r1cs and .wtns files (iden3 r1csfile / wtnsfile, as circom writes them and
ark-circom's R1CSFile / read_witness read them), restated from the format, not from the CUDA code.  PARITY UNPINNED BY
CIRCOM: no circom artifact is available, so the format is pinned by this restatement and by proofs that verify.

All integers little-endian.
.r1cs: "r1cs", version 1, nSections, then {type u32, size u64, body} records in any order:
  1 header (32 + n8 bytes): n8 u32, prime (n8 bytes), nWires u32, nPubOut u32, nPubIn u32, nPrvIn u32, nLabels u64,
    mConstraints u32
  2 constraints: per constraint the linear combinations A, B, C, each nTerms u32 then nTerms {wire u32, coefficient
    (n8 bytes, canonical)}; A.w * B.w - C.w = 0
  3 the wire-to-label map (nWires u64 labels), 4 / 5 custom gates (PLONK only)
num_inputs = 1 + nPubOut + nPubIn, num_witness = nWires - num_inputs, column = wire.
.wtns: "wtns", version 2, nSections; 1: n8 u32, prime, nWitness u32; 2: nWitness canonical n8-byte values.

A circuit is handled as three CSR triples (row_ptr, col, canonical coefficients as (nnz, n8) bytes), so the writer is
vectorized and writes 2^20-constraint circuits quickly."""
import random
import struct

import numpy as np

from groth16_b200 import ConstraintMatrices, get_curve


def _n8(cp) -> int:
    return 8 * cp.fr_limbs


def _canon_bytes(cp, val) -> np.ndarray:
    """(nnz, n8) canonical little-endian bytes of Montgomery limbs"""
    r, n8 = cp.r, _n8(cp)
    rinv = pow(1 << (8 * n8), -1, r)
    raw = np.ascontiguousarray(val, dtype=np.uint64).reshape(-1, cp.fr_limbs)
    if raw.shape[0] == 0:
        return np.zeros((0, n8), dtype=np.uint8)
    b = raw.tobytes()
    out = b"".join((int.from_bytes(b[k:k + n8], "little") * rinv % r).to_bytes(n8, "little") for k in range(0, len(b), n8))
    return np.frombuffer(out, dtype=np.uint8).reshape(-1, n8)


class Circuit:
    """ni (instance variables, One included), nw, and per matrix (row_ptr u32, col u32, canonical coefficient bytes)"""

    def __init__(self, curve, ni, nw, mats):
        self.cp = get_curve(curve)
        self.ni, self.nw = ni, nw
        self.mats = [(np.asarray(rp, dtype=np.int64), np.asarray(col, dtype=np.uint32), np.asarray(cf, dtype=np.uint8))
                     for rp, col, cf in mats]
        self.m = len(self.mats[0][0]) - 1

    @staticmethod
    def from_matrices(curve, m: ConstraintMatrices) -> "Circuit":
        cp = get_curve(curve)
        return Circuit(curve, m.num_instance_variables, m.num_witness_variables,
                       [(t[0], t[1], _canon_bytes(cp, t[2])) for t in (m.a, m.b, m.c)])

    @staticmethod
    def from_rows(curve, ni, nw, rows) -> "Circuit":
        """rows: per constraint (A, B, C), each a list of (wire, canonical int)"""
        cp = get_curve(curve)
        n8 = _n8(cp)
        mats = []
        for k in range(3):
            rp, col, cf = [0], [], []
            for row in rows:
                for w, c in row[k]:
                    col.append(w)
                    cf.append(c.to_bytes(n8, "little"))
                rp.append(len(col))
            mats.append((rp, col, np.frombuffer(b"".join(cf), dtype=np.uint8).reshape(-1, n8)))
        return Circuit(curve, ni, nw, mats)

    @staticmethod
    def from_r1cs(cs) -> "Circuit":
        """a pyref R1CS (rows of (coefficient, column))"""
        rows = [tuple([(i, cf % cs.curve.r) for cf, i in comb] for comb in (ra, rb, rc)) for ra, rb, rc in zip(cs.a, cs.b, cs.c)]
        return Circuit.from_rows(cs.curve.name, cs.num_instance, cs.num_witness, rows)

    def rows(self):
        out = []
        for i in range(self.m):
            out.append(tuple([(int(col[e]), int.from_bytes(cf[e].tobytes(), "little")) for e in range(rp[i], rp[i + 1])]
                             for rp, col, cf in self.mats))
        return out

    def to_matrices(self) -> ConstraintMatrices:
        """the ABI's ConstraintMatrices (Montgomery limbs), in file order"""
        cp = self.cp
        n8, r, R = _n8(cp), cp.r, 1 << (8 * _n8(cp))
        out = []
        for rp, col, cf in self.mats:
            b = cf.tobytes()
            mont = b"".join((int.from_bytes(b[k:k + n8], "little") * R % r).to_bytes(n8, "little") for k in range(0, len(b), n8))
            val = np.frombuffer(mont, dtype=np.uint64).reshape(-1, cp.fr_limbs).copy()
            out.append((np.asarray(rp, dtype=np.uint32), np.asarray(col, dtype=np.uint32), val))
        return ConstraintMatrices(self.ni, self.nw, self.m, *out)

    def transformed(self, split_seed=None, zero_seed=None, long_row=None) -> "Circuit":
        """split_seed: some terms written as two terms on the same wire whose coefficients add up; zero_seed: zero-coefficient
        terms inserted on random wires; long_row: (constraint, count) -- that constraint's A gets `count` extra terms on wire
        0 whose coefficients sum to zero.  Every variant describes the same constraints."""
        r, nv = self.cp.r, self.ni + self.nw
        rng = random.Random(split_seed if split_seed is not None else zero_seed if zero_seed is not None else 0)
        rows = []
        for i, row in enumerate(self.rows()):
            new = []
            for k, comb in enumerate(row):
                out = []
                for w, c in comb:
                    if split_seed is not None and rng.random() < 0.3:
                        part = rng.randrange(r)
                        out += [(w, part), (w, (c - part) % r)]
                    else:
                        out.append((w, c))
                    if zero_seed is not None and rng.random() < 0.2:
                        out.append((rng.randrange(nv), 0))
                if long_row is not None and long_row[0] == i and k == 0:
                    cs = [rng.randrange(r) for _ in range(long_row[1] - 1)]
                    out += [(0, c) for c in cs] + [(0, -sum(cs) % r)]
                new.append(out)
            rows.append(tuple(new))
        return Circuit.from_rows(self.cp.name, self.ni, self.nw, rows)

    def term_prefix(self) -> np.ndarray:
        """tp[i] = the terms of constraints < i (m + 1 entries)"""
        per = sum(np.diff(rp) for rp, _, _ in self.mats)
        return np.concatenate([[0], np.cumsum(per)]).astype(np.int64)

    def section2(self) -> bytes:
        n8 = _n8(self.cp)
        ts = 4 + n8
        tp = self.term_prefix()
        size = 12 * self.m + ts * int(tp[-1])
        buf = np.zeros(size, dtype=np.uint8)
        cs = 12 * np.arange(self.m, dtype=np.int64) + ts * tp[:-1]
        before = np.zeros(self.m, dtype=np.int64)   # terms of the earlier combinations of the same constraint
        for k, (rp, col, cf) in enumerate(self.mats):
            cnt = np.diff(rp)
            at = cs + 4 * k + ts * before
            buf[at[:, None] + np.arange(4)] = cnt.astype("<u4").view(np.uint8).reshape(-1, 4)
            nnz = int(rp[-1])
            if nnz:
                row = np.repeat(np.arange(self.m), cnt)
                pos = np.arange(nnz) - rp[row]
                off = cs[row] + 4 * (k + 1) + ts * (before[row] + pos)
                rec = np.concatenate([col.astype("<u4").view(np.uint8).reshape(-1, 4), cf.reshape(-1, n8)], axis=1)
                buf[off[:, None] + np.arange(ts)] = rec
            before += cnt
        return buf.tobytes()


def write(c: Circuit, npubin=0, nprvin=None, order=None, extra=(), prime=None, n8=None, nwires=None) -> bytes:
    """The .r1cs of c: its ni - 1 public signals split as nPubOut = ni - 1 - npubin outputs and npubin inputs.  order: the
    section ids in file order (default [1, 2, 3]); extra: (id, body) sections appended; prime / n8 / nwires: header
    overrides."""
    cp = c.cp
    n8v = _n8(cp) if n8 is None else n8
    nw_ = c.ni + c.nw if nwires is None else nwires
    npubout = c.ni - 1 - npubin
    prv = c.nw if nprvin is None else nprvin
    sec = {
        1: struct.pack("<I", n8v) + ((cp.r if prime is None else prime) % (1 << (8 * n8v))).to_bytes(n8v, "little")
           + struct.pack("<IIIIQI", nw_, npubout, npubin, prv, nw_, c.m),
        2: c.section2(),
        3: np.arange(nw_, dtype="<u8").tobytes(),
    }
    ids = list(order) if order is not None else [1, 2, 3]
    body = [struct.pack("<IQ", i, len(sec[i])) + sec[i] for i in ids]
    body += [struct.pack("<IQ", i, len(b)) + b for i, b in extra]
    return b"r1cs" + struct.pack("<II", 1, len(body)) + b"".join(body)


def sections(data: bytes, magic=b"r1cs") -> dict:
    """{id: (body offset, size)} of the section table (first one wins)"""
    assert data[:4] == magic
    nsec = struct.unpack_from("<I", data, 8)[0]
    pos, out = 12, {}
    for _ in range(nsec):
        i, size = struct.unpack_from("<IQ", data, pos)
        out.setdefault(i, (pos + 12, size))
        pos += 12 + size
    assert pos == len(data)
    return out


def header(data: bytes) -> dict:
    off, _ = sections(data)[1]
    n8 = struct.unpack_from("<I", data, off)[0]
    prime = int.from_bytes(data[off + 4:off + 4 + n8], "little")
    nwires, npubout, npubin, nprvin, nlabels, m = struct.unpack_from("<IIIIQI", data, off + 4 + n8)
    return dict(n8=n8, prime=prime, nwires=nwires, npubout=npubout, npubin=npubin, nprvin=nprvin, nlabels=nlabels, m=m)


def read(curve, data: bytes) -> Circuit:
    """the circuit of an .r1cs, as ark-circom's R1CS::from(R1CSFile) builds it (terms in file order)"""
    cp = get_curve(curve)
    h = header(data)
    n8 = h["n8"]
    assert n8 == _n8(cp) and h["prime"] == cp.r
    sec = sections(data)
    assert 4 not in sec and 5 not in sec
    ni = 1 + h["npubout"] + h["npubin"]
    pos, end = sec[2][0], sec[2][0] + sec[2][1]
    rows = []
    for _ in range(h["m"]):
        row = []
        for _k in range(3):
            n = struct.unpack_from("<I", data, pos)[0]
            pos += 4
            comb = []
            for _t in range(n):
                w = struct.unpack_from("<I", data, pos)[0]
                cf = int.from_bytes(data[pos + 4:pos + 4 + n8], "little")
                assert w < h["nwires"] and cf < cp.r
                comb.append((w, cf))
                pos += 4 + n8
            row.append(comb)
        rows.append(tuple(row))
    assert pos == end
    return Circuit.from_rows(curve, ni, h["nwires"] - ni, rows)


def term_offset(data: bytes, constraint: int, matrix: int, k: int) -> int:
    """file offset of term k of matrix (0 A, 1 B, 2 C) of a constraint"""
    n8 = header(data)["n8"]
    pos = sections(data)[2][0]
    for i in range(constraint + 1):
        for mi in range(3):
            n = struct.unpack_from("<I", data, pos)[0]
            if i == constraint and mi == matrix:
                assert k < n
                return pos + 4 + k * (4 + n8)
            pos += 4 + n * (4 + n8)
    raise AssertionError("unreachable")


def satisfied(c: Circuit, z) -> bool:
    """A.z * B.z == C.z for every constraint, z canonical ints"""
    r = c.cp.r
    for row in c.rows():
        e = [sum(cf * z[w] for w, cf in comb) % r for comb in row]
        if e[0] * e[1] % r != e[2]:
            return False
    return True


def write_wtns(curve, values, order=None, extra=(), prime=None, n8=None, version=2) -> bytes:
    """the .wtns of `values` (ints written as they are, so values >= r make refused files)"""
    cp = get_curve(curve)
    n8v = _n8(cp) if n8 is None else n8
    sec = {1: struct.pack("<I", n8v) + ((cp.r if prime is None else prime) % (1 << (8 * n8v))).to_bytes(n8v, "little")
           + struct.pack("<I", len(values)),
           2: b"".join(int(v).to_bytes(n8v, "little") for v in values)}
    ids = list(order) if order is not None else [1, 2]
    body = [struct.pack("<IQ", i, len(sec[i])) + sec[i] for i in ids]
    body += [struct.pack("<IQ", i, len(b)) + b for i, b in extra]
    return b"wtns" + struct.pack("<II", version, len(body)) + b"".join(body)


def read_wtns(curve, data: bytes):
    cp = get_curve(curve)
    sec = sections(data, b"wtns")
    off = sec[1][0]
    n8 = struct.unpack_from("<I", data, off)[0]
    assert n8 == _n8(cp) and int.from_bytes(data[off + 4:off + 4 + n8], "little") == cp.r
    n = struct.unpack_from("<I", data, off + 4 + n8)[0]
    o2 = sec[2][0]
    return [int.from_bytes(data[o2 + k * n8:o2 + (k + 1) * n8], "little") for k in range(n)]


def wtns_from_limbs(curve, z) -> bytes:
    """the .wtns of a full assignment in Montgomery limbs"""
    cp = get_curve(curve)
    return write_wtns(curve, [int.from_bytes(b.tobytes(), "little") for b in _canon_bytes(cp, z)])
