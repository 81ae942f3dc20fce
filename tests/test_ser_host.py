"""CPU tier of the proving-key wire format (csrc/ser.cuh, g16_pk_load_serialized / g16_pk_export_serialized):
tests/host/ser_check.cu, built by nvcc and run without a GPU, checks the chunk planner and the placement rule itself, and runs
the per-point decode and encode functions the kernels run on cases this file writes; every answer is compared with
groth16_b200.serialize.ArkCodec (subgroup check on exactly when G16_SER_VALIDATE is set):
  * random subgroup points and the identity, in both encodings;
  * x = 0 and y = 0 points, cofactor torsion [r]T and Q + T in G1 and G2 (the small-order cases of the subgroup check);
  * each single malformation: every flag error, x >= q, an off-curve point, an x with no curve point."""
import io
import os
import shutil
import subprocess

import pytest

import pyref as P
from groth16_b200.serialize import ArkCodec, DeserializeError

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CURVES = {"bls12_381": 0, "bn254": 1, "bls12_377": 2}
REASONS = {1: "compression flag mismatch", 2: "both SWFlags set", 3: "non-zero bytes in the encoding of the point at infinity",
           4: "sort flag set on an uncompressed point", 5: "non-canonical field element (>= q)",
           6: "x is not the abscissa of a curve point", 7: "point is not on the curve",
           8: "point is not in the prime-order subgroup"}


def _torsion_points(curve, g2):
    """(T0, T, Q + T): a full-group point outside the r-torsion, its cofactor part [r]T0, and a subgroup point plus it"""
    c = P.CURVES[curve]
    cx = P.ctx(c)
    G = cx.G2 if g2 else cx.G1
    k = ArkCodec(curve)
    for x0 in range(1, 200):
        x = (x0, 1) if g2 else x0
        try:
            y = k._solve_y(x, g2)
        except DeserializeError:
            continue
        T0 = (x, y)
        T = G.mul(T0, c.r)
        if T is None:
            continue                   # in the subgroup already (always so for BN254 G1)
        gen = cx.g2_gen() if g2 else cx.g1_gen()
        return [T0, G.neg(T0), T, G.add(G.mul(gen, 12345), T)]
    return []


def _special_points(curve, g2):
    """x = 0 and y = 0 points of the full curve group where they exist (order-3 / order-2 points in G1)"""
    c = P.CURVES[curve]
    k = ArkCodec(curve)
    q = c.q
    out = []
    zero = (0, 0) if g2 else 0
    try:
        y = k._solve_y(zero, g2)
        out += [(zero, y), (zero, ((-y[0]) % q, (-y[1]) % q) if g2 else (-y) % q)]
    except DeserializeError:
        pass
    if not g2:
        # y = 0: x^3 = -b; BLS12-377 G1 has (-1, 0)
        for x in (q - 1,):
            if k._on_curve(x, 0, False):
                out.append((x, 0))
    return out


def _cases():
    """yield (curve, g2, flags, op, payload, expected answer)"""
    rng = P.Rng(2024)
    for curve, cid in CURVES.items():
        c = P.CURVES[curve]
        cx = P.ctx(c)
        q = c.q
        for g2 in (False, True):
            G = cx.G2 if g2 else cx.G1
            gen = cx.g2_gen() if g2 else cx.g1_gen()
            pts = [G.mul(gen, rng.fr(c.r)) for _ in range(3)] + [None, G.mul(gen, c.r - 1)]
            pts += _special_points(curve, g2) + _torsion_points(curve, g2)
            for flags in (0, 1, 2, 3):
                compress, validate = bool(flags & 1), bool(flags & 2)
                k = ArkCodec(curve, check_subgroup=validate)
                streams = []
                for Pt in pts:
                    enc = k.point(Pt, g2, compress)
                    coords = "INF" if Pt is None else " ".join(
                        f"{v:x}" for v in ((Pt[0][0], Pt[0][1], Pt[1][0], Pt[1][1]) if g2 else (Pt[0], Pt[1])))
                    yield cid, g2, flags, "E", coords, "BYTES " + enc.hex()
                    streams.append(enc)
                # single malformations of a good point's encoding
                good = bytearray(k.point(pts[0], g2, compress))
                nb = k.fq_bytes
                bad = []
                if k.zcash:
                    b = bytearray(good); b[0] ^= 0x80; bad.append(b)                       # compression flag
                    b = bytearray(good); b[0] |= 0x40; bad.append(b)                       # infinity flag on a real point
                    inf = bytearray(k.point(None, g2, compress)); inf[0] |= 0x20; bad.append(inf)   # infinity + sort flag
                    inf = bytearray(k.point(None, g2, compress)); inf[-1] = 1; bad.append(inf)      # infinity + payload
                    if not compress:
                        b = bytearray(good); b[0] |= 0x20; bad.append(b)                   # sort flag uncompressed
                    # x >= q in the first wire value (x.c1 for G2): q itself and the largest 381-bit value
                    for v in (q, (1 << 381) - 1):
                        b = bytearray(good); fl = b[0] & 0xE0
                        b[0:nb] = v.to_bytes(nb, "big"); b[0] = (b[0] & 0x1F) | fl; bad.append(b)
                else:
                    b = bytearray(good); b[-1] |= 0xC0; bad.append(b)                      # both SWFlags
                    b = bytearray(good); b[-1] = (b[-1] & 0x3F) | 0x40; bad.append(b)      # infinity flag on a real point
                    inf = bytearray(k.point(None, g2, compress)); inf[0] = 1; bad.append(inf)
                    for v in (q, q + 5):
                        b = bytearray(good); b[0:nb] = v.to_bytes(nb, "little"); bad.append(b)
                    # the spare bits under the flags (BLS12-377: bits 377..381 of the last value)
                    top = q.bit_length() % 8
                    if 0 < top < 6:
                        b = bytearray(good); b[-1] |= 0x3F & ~((1 << top) - 1); bad.append(b)
                if compress:
                    for x0 in range(2, 60):        # an x with no curve point
                        x = (x0, 0) if g2 else x0
                        try:
                            k._solve_y(x, g2)
                        except DeserializeError:
                            b = bytearray(k.point((x, (0, 0) if g2 else 0), g2, True))
                            if k.zcash:
                                b[0] &= ~0x20 & 0xFF
                            else:
                                b[-1] &= 0x3F
                            bad.append(b)
                            break
                else:
                    b = bytearray(good)                                                    # y + 1: off the curve
                    Pt = pts[0]
                    y1 = ((Pt[1][0] + 1) % q, Pt[1][1]) if g2 else (Pt[1] + 1) % q
                    bad.append(bytearray(k.point((Pt[0], y1), g2, False)))
                for raw in streams + [bytes(b) for b in bad]:
                    try:
                        pt = k.read_point(io.BytesIO(bytes(raw)), g2, compress)
                        if pt is None:
                            want = "INF"
                        else:
                            vals = (pt[0][0], pt[0][1], pt[1][0], pt[1][1]) if g2 else pt
                            want = "PT " + " ".join(f"{v:0{2 * k.fq_bytes}x}" for v in vals)
                    except DeserializeError as e:
                        want = ("ERR", str(e))
                    yield cid, g2, flags, "D", bytes(raw).hex(), want


def test_ser_point_codec_and_planner_host(tmp_path):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path / "ser_check")
    subprocess.check_call(["nvcc", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "--expt-relaxed-constexpr",
                           "-o", exe, os.path.join(ROOT, "tests", "host", "ser_check.cu")])
    cases = list(_cases())
    stdin = "".join(f"{op} {cid} {int(g2)} {flags} {payload}\n" for cid, g2, flags, op, payload, _ in cases)
    res = subprocess.run([exe], input=stdin, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    lines = res.stdout.splitlines()
    assert lines[0].startswith("planner: ") and lines[0].endswith(", 0 mismatches"), lines[0]
    assert int(lines[0].split()[1]) > 10000, lines[0]
    answers = lines[1:]
    assert len(answers) == len(cases)
    seen_codes = set()
    for (cid, g2, flags, op, payload, want), got in zip(cases, answers):
        where = f"curve {cid} g2 {g2} flags {flags} {op} {payload[:40]}"
        if isinstance(want, tuple):
            assert got.startswith("ERR "), (where, got, want)
            code = int(got.split()[1])
            seen_codes.add(code)
            assert REASONS[code] == want[1], (where, REASONS[code], want[1])
        else:
            assert got == want, (where, got, want)
    # every check serialize.py makes was met at least once
    assert seen_codes == set(REASONS), sorted(set(REASONS) - seen_codes)
