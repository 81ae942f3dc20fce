"""CPU tier of the .zkey host code (csrc/zkey.cuh) and the Montgomery little-endian point decode (csrc/ser.cuh):
tests/host/zkey_check.cu, built by nvcc and run without a GPU, answers requests that are checked here against
tests/zkey_ref.py and pyref -- the section walk and every refusal it decides on the host, with its message, and the
per-record coefficient and per-point decodes at edge values (0, 1, r - 1, values >= r, q - 1, coordinates >= q)."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import pyref as P
import qap_circom_ref as Q
import zkey_ref as Z
from groth16_b200 import CurveCodec, get_curve
from util import matrices_from_r1cs, pk_to_abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOXIC = (0x1234567, 0x2345678, 0x3456789, 0x456789A, 0x56789AB)


@pytest.fixture(scope="module")
def check(tmp_path_factory):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("zkey") / "zkey_check")
    subprocess.check_call(["nvcc", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "--expt-relaxed-constexpr",
                           "-o", exe, os.path.join(ROOT, "tests", "host", "zkey_check.cu")])
    p = subprocess.Popen([exe], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)

    def ask(line):
        p.stdin.write(line + "\n")
        p.stdin.flush()
        return p.stdout.readline().strip()

    yield ask
    p.stdin.close()
    p.wait(timeout=60)


def _file(curve):
    c = P.CURVES[curve]
    cs = P.silly_circuit(c, 3, 11)
    m = matrices_from_r1cs(cs)
    pk = pk_to_abi(Q.generate_parameters(cs, *TOXIC, qap="circom"))
    return m, pk, Z.write(curve, m, pk)


def _patch(data, off, raw):
    b = bytearray(data)
    b[off:off + len(raw)] = raw
    return bytes(b)


@pytest.mark.parametrize("curve", Z.SNARKJS_CURVES)
def test_walk(check, curve, tmp_path):
    cp = get_curve(curve)
    m, pk, data = _file(curve)
    h = Z.header(data)
    nq, nr = h["n8q"], h["n8r"]
    off2 = Z.sections(data)[2][0]
    off4, size4 = Z.sections(data)[4]

    def walk(d):
        f = tmp_path / "k.zkey"
        f.write_bytes(d)
        return check(f"walk {curve} {f}")

    for kw in ({}, {"shuffle_seed": 1}, {"order": [9, 3, 1, 7, 5, 2, 8, 4, 6]}, {"junk10": b"x" * 17}):
        d = Z.write(curve, m, pk, **kw)
        ncoef = struct.unpack_from("<I", d, Z.sections(d)[4][0])[0]
        assert walk(d) == f"ok {h['nvars']} {h['npub']} {h['domain_size']} {ncoef} {Z.coef_offset(d, 0)}", kw
    other = "bls12_381" if curve == "bn254" else "bn254"
    cases = [
        (data[:11], "truncated input: 11 bytes"),
        (b"zkex" + data[4:], "not a .zkey file"),
        (_patch(data, 4, struct.pack("<I", 2)), "unsupported .zkey version 2 (expected 1)"),
        (data[:-1], "truncated input: section 9"),
        (data + b"\0", "trailing bytes after the last section (1)"),
        (_patch(data, 8, struct.pack("<I", 10)), "truncated input: section 9 of 10 has no complete header"),
        (Z.write(curve, m, pk, order=[1, 2, 3, 4, 5, 6, 7, 8]), "section 9 is missing"),
        (Z.write(curve, m, pk, order=[2, 3, 4, 5, 6, 7, 8, 9]), "section 1 is missing"),
        (Z.write(curve, m, pk, order=[1, 2, 3, 4, 5, 6, 6, 7, 8, 9]), "section 6 appears twice"),
        (_patch(data, Z.sections(data)[1][0], struct.pack("<I", 2)), "section 1: protocol 2 is not Groth16 (1)"),
        (_patch(data, off2, struct.pack("<I", 48 if nq == 32 else 32)), "section 2: n8q = "),
        (_patch(data, off2 + 4, (cp.q + 1).to_bytes(nq, "little")), "section 2: q is not the base field modulus"),
        (_patch(data, off2 + 4 + nq, struct.pack("<I", 48)), "section 2: n8r = 48"),
        (_patch(data, off2 + 8 + nq, (cp.r - 1).to_bytes(nr, "little")), "section 2: r is not the scalar field modulus"),
        (_patch(data, h["points"] - 12, struct.pack("<I", 1)), "section 2: nVars = 1 is below nPublic + 1 = 2"),
        (_patch(data, h["points"] - 4, struct.pack("<I", 0)), "section 2: domainSize = 0 is not a power of two"),
        (_patch(data, h["points"] - 4, struct.pack("<I", 12)), "section 2: domainSize = 12 is not a power of two"),
        (_patch(data, off4, struct.pack("<I", struct.unpack_from("<I", data, off4)[0] + 1)),
         f"section 4 (coefficients): size {size4}, expected {size4 + 12 + nr}"),
        (_patch(data, h["points"] - 8, struct.pack("<I", 2)), "section 3 (IC): size"),
    ]
    for bad, msg in cases:
        got = walk(bad)
        assert got.startswith("err ") and msg in got, (msg, got)
    # a file of the other snarkjs curve
    _, _, od = _file(other)
    assert walk(od).startswith("err section 2: n8q = ") or walk(od).startswith("err section 2: q is not")


@pytest.mark.parametrize("curve", Z.SNARKJS_CURVES)
def test_coefficient_decode(check, curve):
    cp = get_curve(curve)
    r, nr = cp.r, 8 * cp.fr_limbs
    R = 1 << (8 * nr)
    rec = lambda m, i, s, v: (struct.pack("<III", m, i, s) + v.to_bytes(nr, "little")).hex()
    for c in (0, 1, 2, r - 1, 0x1234567890):
        code, val = check(f"coef {curve} 16 10 {rec(1, 15, 9, c * R * R % r)}").split()
        assert code == "0" and int.from_bytes(bytes.fromhex(val), "little") == c * R % r, c
    for v in (r, r + 1, R - 1):
        assert check(f"coef {curve} 16 10 {rec(0, 0, 0, v)}").split()[0] == "4", v
    assert check(f"coef {curve} 16 10 {rec(2, 0, 0, 1)}").split()[0] == "1"
    assert check(f"coef {curve} 16 10 {rec(0, 16, 0, 1)}").split()[0] == "2"
    assert check(f"coef {curve} 16 10 {rec(0, 15, 10, 1)}").split()[0] == "3"
    assert check(f"coef {curve} 16 10 {rec(7, 99, 99, r)}").split()[0] == "1"   # the first failing check wins


@pytest.mark.parametrize("curve", Z.SNARKJS_CURVES)
def test_point_decode(check, curve):
    cp = get_curve(curve)
    cd = CurveCodec(cp)
    c = P.CURVES[curve]
    cx = P.ctx(c)
    nq = 8 * cp.fq_limbs
    q = cp.q
    for g2, G, gen in ((0, cx.G1, cx.g1_gen()), (1, cx.G2, cx.g2_gen())):
        enc = cd.enc_g2 if g2 else cd.enc_g1
        pts = [G.mul(gen, k) for k in (1, 2, 12345)]
        for p in pts:
            raw = enc([p])[0].tobytes()
            code, limbs = check(f"point {curve} {g2} 1 {raw.hex()}").split()
            assert code == "0" and bytes.fromhex(limbs) == raw
        zero = bytes(len(enc([pts[0]])[0].tobytes()))
        code, limbs = check(f"point {curve} {g2} 1 {zero.hex()}").split()
        assert code == "0" and bytes.fromhex(limbs) == zero                     # the identity
        raw = bytearray(enc([pts[0]])[0].tobytes())
        for k in range(4 if g2 else 2):                                         # each coordinate at q and at 2^(8 n8q) - 1
            for v in (q, (1 << (8 * nq)) - 1):
                b = bytearray(raw)
                b[k * nq:(k + 1) * nq] = v.to_bytes(nq, "little")
                assert check(f"point {curve} {g2} 0 {bytes(b).hex()}").split()[0] == "5", (g2, k)
        b = bytearray(raw)
        b[0:nq] = (q - 1).to_bytes(nq, "little")                                # canonical, but off the curve
        assert check(f"point {curve} {g2} 0 {bytes(b).hex()}").split()[0] == "7"
