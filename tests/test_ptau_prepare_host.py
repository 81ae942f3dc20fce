"""CPU tier of g16_ptau_prepare's host decisions and of its transform's lane map: tests/host/ptau_prepare_check.cu, built by
nvcc and run without a GPU, answers requests with the library's own functions (csrc/ptau.cuh, csrc/srs.cuh); the answers
are checked here against tests/ptau_ref.py -- the prepared file's size, section count and every section offset and size,
from real files and from the header alone for powers 0-20 on all four curves -- and against the definition of the
radix-2 stages: every butterfly once per stage, one twiddle per warp wherever 32 butterflies share it; and the signed
4-bit recoding of the windowed twiddle product reconstructs every twiddle."""
import os
import re
import shutil
import struct
import subprocess

import numpy as np
import pytest

import ptau_ref as T
from groth16_b200 import get_curve

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CURVES = ["bn254", "bls12_381", "bls12_377", "bw6_761"]


@pytest.fixture(scope="module")
def check(tmp_path_factory):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("ptau_prepare") / "ptau_prepare_check")
    subprocess.check_call(["nvcc", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "--expt-relaxed-constexpr",
                           "-o", exe, os.path.join(ROOT, "tests", "host", "ptau_prepare_check.cu")])
    p = subprocess.Popen([exe], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)

    def ask(line):
        p.stdin.write(line + "\n")
        p.stdin.flush()
        return p.stdout.readline().strip()

    yield ask
    p.stdin.close()
    p.wait(timeout=60)


def transcript(curve, power, seed=3):
    """random limbs: nothing here reads a point"""
    rng = np.random.default_rng(seed)
    n = 1 << power
    lens = dict(tau_g1=2 * n - 1, tau_g2=n, alpha_tau_g1=n, beta_tau_g1=n)
    srs = {m: rng.integers(0, 1 << 63, size=T.points(curve, m, k).shape, dtype=np.uint64) for m, k in lens.items()}
    srs["beta_g2"] = rng.integers(0, 1 << 63, size=T.points(curve, "tau_g2", 1).shape[1], dtype=np.uint64)
    lag = {m: rng.integers(0, 1 << 63, size=v.shape, dtype=np.uint64) for m, v in T.empty_lagrange(curve, power).items()}
    return srs, lag


def file_order(data):
    """section ids in file order"""
    nsec, pos, out = struct.unpack_from("<I", data, 8)[0], 12, []
    for _ in range(nsec):
        i, size = struct.unpack_from("<IQ", data, pos)
        out.append(i)
        pos += 12 + size
    return out


def parse(line):
    parts = line.split(" |")
    size, nsec = (int(x) for x in parts[0].split())
    return size, nsec, [int(x) for x in parts[1].split()], [int(x) for x in parts[2].split()], parts[3:]


@pytest.mark.parametrize("curve", CURVES)
def test_layout_of_files(check, curve, tmp_path):
    """the prepared file laid out from a real input equals ptau_ref.write of the expected output: the kept sections in
    input order (7 and unknown ids included, an input's 12..15 dropped), then 12, 13, 14, 15"""
    f = tmp_path / "in.ptau"
    for power in (0, 1, 2, 4):
        srs, lag = transcript(curve, power)
        extra = [(99, b"\x05" * 13), (0, b"")]
        for prepared in (False, True):
            for order in (None, [6, 15, 2, 1, 14, 7, 3, 13, 5, 4, 12]):
                data = T.write(curve, power, srs, lag if prepared else None, order=order, extra=extra)
                f.write_bytes(data)
                got = check(f"file {curve} {f}")
                assert got.startswith("ok "), got
                size, nsec, off, pts, rest = parse(got[3:])
                s = T.sections(data)
                ids = [i for i in file_order(data) if not 12 <= i <= 15]
                assert [int(x) for x in rest[0].split()] == [s[i][0] - 12 for i in ids]
                lag_secs = [(i, np.ascontiguousarray(lag[m]).tobytes()) for i, m in T.LAG.items()]
                body = b"".join(data[s[i][0] - 12:s[i][0] + s[i][1]] for i in ids)
                body += b"".join(struct.pack("<IQ", i, len(b)) + b for i, b in lag_secs)
                want = b"ptau" + struct.pack("<II", 1, len(ids) + 4) + body
                if order is None:   # input 1..7 (12..15), 99, 0: the output is 1..7, 99, 0, 12..15
                    assert want == T.write(curve, power, srs, None, extra=extra + lag_secs)
                ws = T.sections(want)
                assert (size, nsec) == (len(want), len(ids) + 4), (power, prepared, order)
                assert off == [ws[i][0] for i in (12, 13, 14, 15)]
                w1, w2 = T.widths(curve)
                assert [ws[i][1] for i in (12, 13, 14, 15)] == [p * 8 * (w2 if i == 13 else w1) for p, i in zip(pts, (12, 13, 14, 15))]
                assert pts == [T.lagrange_sizes(power)[i] for i in (12, 13, 14, 15)]


@pytest.mark.parametrize("curve", CURVES)
def test_layout_from_header(check, curve):
    """powers 0-20 from the header alone: an unprepared input with sections 1..7 (section 7 holding one u32)"""
    c = get_curve(curve)
    n8 = 8 * c.fq_limbs
    w1, w2 = (8 * w for w in T.widths(curve))
    for power in range(21):
        n = 1 << power
        kept = [12 + n8, (2 * n - 1) * w1, n * w2, n * w1, n * w1, w2, 4]
        kept_bytes = sum(12 + k for k in kept)
        size, nsec, off, pts, _ = parse(check(f"header {curve} {power} {len(kept)} {kept_bytes}") + " |")
        sizes = T.lagrange_sizes(power)
        want_pts = [sizes[i] for i in (12, 13, 14, 15)]
        assert pts == want_pts
        pos, want_off = 12 + kept_bytes, []
        for i, p in zip((12, 13, 14, 15), want_pts):
            want_off.append(pos + 12)
            pos += 12 + p * (w2 if i == 13 else w1)
        assert (size, nsec, off) == (pos, 11, want_off), power


def test_walk_refusals_are_the_read_walk(check, tmp_path):
    """the layout is only formed for files ptau_walk accepts, with its message"""
    srs, lag = transcript("bn254", 2)
    f = tmp_path / "bad.ptau"
    f.write_bytes(T.write("bn254", 2, srs, lag, drop=[13]))
    assert check(f"file bn254 {f}") == "err sections 12-15 (Lagrange points) appear all four or none: only 12, 14, 15 present"


def test_lane_map(check):
    got = check("map 16")
    m = re.fullmatch(r"map: (\d+) checks, (\d+) mismatches", got)
    assert m and m.group(2) == "0" and int(m.group(1)) > 2_000_000, got


@pytest.mark.parametrize("curve", CURVES)
def test_window_recoding(check, curve):
    """the signed-digit recoding of srs_mul_w4 reconstructs every twiddle of the domains up to 2^14"""
    got = check(f"recode {curve} 14")
    m = re.fullmatch(r"recode: (\d+) checks, (\d+) mismatches", got)
    assert m and m.group(2) == "0" and int(m.group(1)) > 10_000, got
