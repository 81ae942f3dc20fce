"""An independent writer and reader of snarkjs Groth16 .zkey files, restated from the format (snarkjs zkey_utils.js /
zkey_new.js, ark-circom zkey.rs), not from the CUDA code.  PARITY UNPINNED BY SNARKJS: no snarkjs artifact or Node runtime
is available, so the format is pinned by this restatement and by proofs that verify; a snarkjs-made fixture is the follow-up.

All integers little-endian.  "zkey", version 1, nSections, then {id u32, size u64, body} records:
  1 protocol = 1 (Groth16)
  2 n8q, q, n8r, r, nVars, nPublic, domainSize, alpha1, beta1, beta2, gamma2, delta1, delta2
  3 IC = gamma_abc_g1 (nPublic + 1 G1)
  4 nCoefs, then {matrix (0 = A, 1 = B), constraint, signal, value = c R_r^2 mod r (n8r bytes)}; A gets the appended rows
    nConstraints + s = {(s, 1)} for s = 0 .. nPublic
  5 A, 6 B1, 7 B2 (nVars points), 8 C = l_query (nVars - nPublic - 1 G1), 9 H = h_query (domainSize G1)
Coordinates are n8q bytes in Montgomery form (R = 2^(8 n8q)), which is exactly the little-endian byte image of the ABI's u64
limbs; G2 is x.c0 || x.c1 || y.c0 || y.c1; the identity is all-zero bytes.  Keys and matrices here are in the ABI form of
groth16_b200 (ProvingKey / ConstraintMatrices with Montgomery limbs)."""
import random
import struct

import numpy as np

from groth16_b200 import ConstraintMatrices, ProvingKey, VerifyingKey, get_curve

SNARKJS_CURVES = ("bn254", "bls12_381")


def _le(x: int, n: int) -> bytes:
    return x.to_bytes(n, "little")


def _limbs_int(row) -> int:
    return int.from_bytes(np.ascontiguousarray(row, dtype=np.uint64).tobytes(), "little")


def _pts(a) -> bytes:
    return np.ascontiguousarray(a, dtype=np.uint64).tobytes()


def coef_records(curve, m: ConstraintMatrices):
    """(matrix, constraint, signal, value) for every entry of A and B plus the appended public-input rows of A"""
    cp = get_curve(curve)
    r = cp.r
    R = 1 << (8 * cp.fr_limbs * 8)
    out = []
    for mi, (rp, col, val) in enumerate((m.a, m.b)):
        rp, col = np.asarray(rp), np.asarray(col)
        for i in range(m.num_constraints):
            for e in range(int(rp[i]), int(rp[i + 1])):
                cm = _limbs_int(val[e])                 # c R mod r
                out.append((mi, i, int(col[e]), cm * R % r))
    one = R % r                                         # 1 in Montgomery form
    for s in range(m.num_instance_variables):
        out.append((0, m.num_constraints + s, s, one * R % r))
    return out


def write(curve, m: ConstraintMatrices, pk: ProvingKey, shuffle_seed=None, order=None, junk10: bytes = b"", records=None,
          split_seed=None) -> bytes:
    """The .zkey of circuit m (CircomReduction key pk, as g16_pk_export writes it).  shuffle_seed: shuffle the coefficient
    records; order: the section ids in file order (default 1 .. 9); junk10: a trailing section 10 with these bytes (b"" =
    none); records: the coefficient records to write instead of coef_records(m); split_seed: split some entries into two
    records whose values add up to the original."""
    cp = get_curve(curve)
    assert cp.name in SNARKJS_CURVES
    nq, nr = 8 * cp.fq_limbs, 8 * cp.fr_limbs
    r = cp.r
    ni, nw = m.num_instance_variables, m.num_witness_variables
    nv = ni + nw
    n = len(pk.h_query)
    recs = list(records) if records is not None else coef_records(curve, m)
    if split_seed is not None:
        rng = random.Random(split_seed)
        out = []
        for rec in recs:
            if rec[1] < m.num_constraints and rng.random() < 0.3:
                part = rng.randrange(r)
                out += [(rec[0], rec[1], rec[2], part), (rec[0], rec[1], rec[2], (rec[3] - part) % r)]
            else:
                out.append(rec)
        recs = out
    if shuffle_seed is not None:
        random.Random(shuffle_seed).shuffle(recs)
    vk = pk.vk
    sec = {
        1: struct.pack("<I", 1),
        2: (struct.pack("<I", nq) + _le(cp.q, nq) + struct.pack("<I", nr) + _le(r, nr) + struct.pack("<III", nv, ni - 1, n)
            + _pts(vk.alpha_g1) + _pts(pk.beta_g1) + _pts(vk.beta_g2) + _pts(vk.gamma_g2) + _pts(pk.delta_g1)
            + _pts(vk.delta_g2)),
        3: _pts(vk.gamma_abc_g1),
        4: struct.pack("<I", len(recs)) + b"".join(struct.pack("<III", a, b, c) + _le(v, nr) for a, b, c, v in recs),
        5: _pts(pk.a_query), 6: _pts(pk.b_g1_query), 7: _pts(pk.b_g2_query), 8: _pts(pk.l_query), 9: _pts(pk.h_query),
    }
    ids = list(order) if order is not None else list(range(1, 10))
    body = []
    for i in ids:
        body.append(struct.pack("<IQ", i, len(sec[i])) + sec[i])
    if junk10:
        body.append(struct.pack("<IQ", 10, len(junk10)) + junk10)
    return b"zkey" + struct.pack("<II", 1, len(body)) + b"".join(body)


def sections(data: bytes) -> dict:
    """{id: (body offset, size)} of the section table (last one wins)"""
    assert data[:4] == b"zkey"
    nsec = struct.unpack_from("<I", data, 8)[0]
    pos, out = 12, {}
    for _ in range(nsec):
        i, size = struct.unpack_from("<IQ", data, pos)
        out[i] = (pos + 12, size)
        pos += 12 + size
    assert pos == len(data)
    return out


def header(data: bytes) -> dict:
    off, _ = sections(data)[2]
    nq = struct.unpack_from("<I", data, off)[0]
    nr = struct.unpack_from("<I", data, off + 4 + nq)[0]
    f = off + 8 + nq + nr
    nv, npub, n = struct.unpack_from("<III", data, f)
    return dict(n8q=nq, n8r=nr, nvars=nv, npub=npub, domain_size=n, points=f + 12, q=int.from_bytes(data[off + 4:off + 4 + nq], "little"),
                r=int.from_bytes(data[off + 8 + nq:f], "little"))


def coef_offset(data: bytes, k: int) -> int:
    """byte offset of coefficient record k"""
    off, _ = sections(data)[4]
    return off + 4 + k * (12 + header(data)["n8r"])


def read(curve, data: bytes):
    """-> (ConstraintMatrices with C empty, ProvingKey), as ark-circom's read_zkey derives them"""
    cp = get_curve(curve)
    nl = cp.fq_limbs
    h = header(data)
    nq, nr, nv, npub, n = h["n8q"], h["n8r"], h["nvars"], h["npub"], h["domain_size"]
    assert nq == 8 * nl and h["q"] == cp.q and h["r"] == cp.r
    sec = sections(data)
    r = cp.r
    Rinv = pow(1 << (8 * nr), -1, r)

    def g1(off, cnt):
        return np.frombuffer(data, dtype=np.uint64, count=cnt * 2 * nl, offset=off).reshape(cnt, 2 * nl).copy()

    def g2(off, cnt):
        return np.frombuffer(data, dtype=np.uint64, count=cnt * 4 * nl, offset=off).reshape(cnt, 4 * nl).copy()

    p = h["points"]
    G1, G2 = 2 * nq, 4 * nq
    alpha1, beta1 = g1(p, 1)[0], g1(p + G1, 1)[0]
    beta2, gamma2 = g2(p + 2 * G1, 1)[0], g2(p + 2 * G1 + G2, 1)[0]
    delta1, delta2 = g1(p + 2 * G1 + 2 * G2, 1)[0], g2(p + 3 * G1 + 2 * G2, 1)[0]
    off4, _ = sec[4]
    ncoef = struct.unpack_from("<I", data, off4)[0]
    recs = []
    for k in range(ncoef):
        o = off4 + 4 + k * (12 + nr)
        mtx, row, sig = struct.unpack_from("<III", data, o)
        v = int.from_bytes(data[o + 12:o + 12 + nr], "little")
        recs.append((mtx, row, sig, v * Rinv % r))          # c R
    nc = max(rec[1] for rec in recs) - npub
    rows = [[{}, {}] for _ in range(nc)]
    for mtx, row, sig, v in recs:
        if row >= nc:
            continue
        d = rows[row][mtx]
        d[sig] = (d.get(sig, 0) + v) % r

    def csr(mi):
        rp, col, val = [0], [], []
        for i in range(nc):
            for s_, v in sorted(rows[i][mi].items()):
                col.append(s_)
                val.append(np.frombuffer(_le(v, 8 * cp.fr_limbs), dtype=np.uint64))
            rp.append(len(col))
        return (np.asarray(rp, dtype=np.uint32), np.asarray(col, dtype=np.uint32),
                np.ascontiguousarray(np.array(val, dtype=np.uint64).reshape(-1, cp.fr_limbs)))

    empty = (np.zeros(nc + 1, dtype=np.uint32), np.zeros(0, dtype=np.uint32), np.zeros((0, cp.fr_limbs), dtype=np.uint64))
    m = ConstraintMatrices(npub + 1, nv - npub - 1, nc, csr(0), csr(1), empty)
    vk = VerifyingKey(alpha1, beta2, gamma2, delta2, g1(sec[3][0], npub + 1))
    pk = ProvingKey(vk, beta1, delta1, g1(sec[5][0], nv), g1(sec[6][0], nv), g2(sec[7][0], nv), g1(sec[9][0], n),
                    g1(sec[8][0], nv - npub - 1))
    return m, pk


def canonical_rows(m: ConstraintMatrices, which, r: int):
    """matrix `which` as a list of {signal: Montgomery int mod r} per row (duplicates summed, zeros dropped), for an
    order-free comparison"""
    rp, col, val = getattr(m, which)
    out = []
    for i in range(m.num_constraints):
        d = {}
        for e in range(int(rp[i]), int(rp[i + 1])):
            d[int(col[e])] = (d.get(int(col[e]), 0) + _limbs_int(val[e])) % r
        out.append({k: v for k, v in d.items() if v})
    return out
