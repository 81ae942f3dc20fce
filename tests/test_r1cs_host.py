"""CPU tier of the .r1cs / .wtns host code (csrc/r1cs.cuh): tests/host/r1cs_check.cu, built by nvcc and run without a GPU,
answers requests that are checked here against tests/r1cs_ref.py -- the section and term-count walk with its row_ptr and
term prefix, every refusal it decides on the host with its message, on all four curves' scalar fields, and the per-term and
per-element decodes at 0, 1, r - 1, r and 2^(8 n8) - 1, and at wire = nWires - 1 and nWires."""
import os
import random
import shutil
import struct
import subprocess

import pytest

import r1cs_ref as R
from groth16_b200 import get_curve

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CURVES = ["bn254", "bls12_381", "bls12_377", "bw6_761"]


@pytest.fixture(scope="module")
def check(tmp_path_factory):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("r1cs") / "r1cs_check")
    subprocess.check_call(["nvcc", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "--expt-relaxed-constexpr",
                           "-o", exe, os.path.join(ROOT, "tests", "host", "r1cs_check.cu")])
    p = subprocess.Popen([exe], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)

    def ask(line):
        p.stdin.write(line + "\n")
        p.stdin.flush()
        return p.stdout.readline().strip()

    yield ask
    p.stdin.close()
    p.wait(timeout=60)


def circuit(curve, seed=1, ni=3, nw=6, m=7):
    """random constraints with empty combinations, repeated wires and zero coefficients"""
    r = get_curve(curve).r
    rng = random.Random(seed)
    rows = []
    for i in range(m):
        row = []
        for k in range(3):
            n = rng.choice([0, 1, 2, 3, 5]) if i else 0      # constraint 0 is all empty
            row.append([(rng.randrange(ni + nw), rng.choice([0, 1, r - 1, rng.randrange(r)])) for _ in range(n)])
        rows.append(tuple(row))
    return R.Circuit.from_rows(curve, ni, nw, rows)


def _patch(data, off, raw):
    b = bytearray(data)
    b[off:off + len(raw)] = raw
    return bytes(b)


@pytest.mark.parametrize("curve", CURVES)
def test_walk(check, curve, tmp_path):
    cp = get_curve(curve)
    n8 = 8 * cp.fr_limbs
    c = circuit(curve)

    def walk(d):
        f = tmp_path / "c.r1cs"
        f.write_bytes(d)
        return check(f"walk {curve} {f}")

    variants = [dict(), dict(order=[2, 3, 1]), dict(order=[2, 1]), dict(extra=[(6, b"x" * 5), (0, b""), (99, b"\1" * 40)]),
                dict(npubin=1)]
    for kw in variants:
        for cc in (c, c.transformed(split_seed=3), c.transformed(zero_seed=4)):
            got = walk(R.write(cc, **kw)).split(" |")
            assert got[0] == f"ok {cc.ni} {cc.nw} {cc.m} {4 + n8}", kw
            for k in range(3):
                assert [int(x) for x in got[1 + k].split()] == [int(x) for x in cc.mats[k][0]], (kw, k)
            assert [int(x) for x in got[4].split()] == [int(x) for x in cc.term_prefix()], kw
    data = R.write(c)
    h1, s1 = R.sections(data)[1]
    h2, s2 = R.sections(data)[2]
    need = 12 * c.m + (4 + n8) * int(c.term_prefix()[-1])
    assert s2 == need
    other_n8 = 48 if n8 == 32 else 32
    cases = [
        (data[:11], "truncated input: 11 bytes, a .r1cs header is 12"),
        (b"r1cx" + data[4:], "not a .r1cs file"),
        (_patch(data, 4, struct.pack("<I", 2)), "unsupported .r1cs version 2 (expected 1)"),
        (data[:-1], "truncated input: section 3"),
        (data + b"\0", "trailing bytes after the last section (1)"),
        (_patch(data, 8, struct.pack("<I", 4)), "truncated input: section 3 of 4 has no complete header"),
        (R.write(c, order=[2, 3]), "section 1 is missing"),
        (R.write(c, order=[1, 3]), "section 2 is missing"),
        (R.write(c, order=[1, 2, 1]), "section 1 appears twice"),
        (R.write(c, extra=[(2, b"")]), "section 2 appears twice"),
        (R.write(c, extra=[(4, b"gate")]), "section 4: custom gates are not R1CS"),
        (R.write(c, extra=[(5, b"")]), "section 5: custom gates are not R1CS"),
        (R.write(c, n8=other_n8), f"section 1: n8 = {other_n8}, the context's curve has {n8}-byte scalars"),
        (R.write(c, prime=cp.r + 2), "section 1: prime is not the scalar field modulus of this curve"),
        (R.write(c, nwires=c.ni + c.nw - 1), f"section 1: nWires = {c.ni + c.nw - 1} is below 1 + nPubOut + nPubIn + nPrvIn = "
                                             f"{c.ni + c.nw}"),
        (_patch(data, h1 - 8, struct.pack("<Q", s1 + 4)), "truncated input: section "),
        # one more constraint declared than written: the walk runs past the section
        (_patch(data, h1 + 4 + n8 + 24, struct.pack("<I", c.m + 1)), f"section 2 holds {s2} bytes, its constraints need more"),
        # a term count that runs past the end
        (_patch(data, h2, struct.pack("<I", 1 << 30)), "constraint 0's 1073741824 A terms run past its end"),
        # a section 2 with room left over: its constraints need fewer bytes than it holds
        (_patch(data, h1 + 4 + n8 + 24, struct.pack("<I", c.m - 1)), f"section 2 holds {s2} bytes, its constraints need "),
        (_patch(data, h1 + 4 + n8 + 24, struct.pack("<I", 0xFFFFFFFF)), "constraints need at least"),
    ]
    for bad, msg in cases:
        got = walk(bad)
        assert got.startswith("err ") and msg in got, (msg, got)
    # a file of another field
    od = R.write(circuit("bls12_381" if curve != "bls12_381" else "bn254"))
    assert walk(od).startswith("err section 1: ")


@pytest.mark.parametrize("curve", CURVES)
def test_term_and_element_decode(check, curve):
    cp = get_curve(curve)
    r, n8 = cp.r, 8 * cp.fr_limbs
    R_ = 1 << (8 * n8)
    term = lambda w, v: (struct.pack("<I", w) + v.to_bytes(n8, "little")).hex()
    for v in (0, 1, 2, r - 1, 0x1234567890ABCDEF):
        code, wire, val = check(f"term {curve} 10 {term(9, v)}").split()
        assert (code, wire) == ("0", "9") and int.from_bytes(bytes.fromhex(val), "little") == v * R_ % r, v
        code, val = check(f"elem {curve} {v.to_bytes(n8, 'little').hex()}").split()
        assert code == "0" and int.from_bytes(bytes.fromhex(val), "little") == v * R_ % r, v
    for v in (r, r + 1, R_ - 1):
        assert check(f"term {curve} 10 {term(0, v)}").split()[0] == "2", v
        assert check(f"elem {curve} {v.to_bytes(n8, 'little').hex()}").split()[0] == "2", v
    assert check(f"term {curve} 10 {term(10, 1)}").split()[0] == "1"
    assert check(f"term {curve} 10 {term(0xFFFFFFFF, 1)}").split()[0] == "1"
    assert check(f"term {curve} 10 {term(10, r)}").split()[0] == "1"   # the wire is checked first


@pytest.mark.parametrize("curve", CURVES)
def test_wtns_walk(check, curve, tmp_path):
    cp = get_curve(curve)
    n8 = 8 * cp.fr_limbs
    vals = [1, 2, cp.r - 1, 0, 12345]

    def walk(d):
        f = tmp_path / "w.wtns"
        f.write_bytes(d)
        return check(f"wtns {curve} {f}")

    for kw in ({}, {"order": [2, 1]}, {"extra": [(3, b"abc")]}):
        d = R.write_wtns(curve, vals, **kw)
        assert walk(d) == f"ok 5 {R.sections(d, b'wtns')[2][0]}", kw
    d = R.write_wtns(curve, vals)
    assert walk(R.write_wtns(curve, [])) == f"ok 0 {R.sections(R.write_wtns(curve, []), b'wtns')[2][0]}"
    o1 = R.sections(d, b"wtns")[1][0]
    cases = [
        (b"wtnz" + d[4:], "not a .wtns file"),
        (R.write_wtns(curve, vals, version=1), "unsupported .wtns version 1 (expected 2)"),
        (R.write_wtns(curve, vals, order=[1]), "section 2 is missing"),
        (R.write_wtns(curve, vals, order=[1, 2, 2]), "section 2 appears twice"),
        (R.write_wtns(curve, vals, n8=n8 + 8), f"section 1: n8 = {n8 + 8}"),
        (R.write_wtns(curve, vals, prime=cp.r - 2), "section 1: prime is not the scalar field modulus"),
        (_patch(d, o1 + 4 + n8, struct.pack("<I", 6)), f"section 2 holds {5 * n8} bytes, 6 elements need {6 * n8}"),
        (d[:-1], "truncated input"),
    ]
    for bad, msg in cases:
        got = walk(bad)
        assert got.startswith("err ") and msg in got, (msg, got)
