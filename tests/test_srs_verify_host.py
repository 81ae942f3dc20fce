"""CPU tier of g16_srs_verify_pairs (the transcript check): tests/host/srs_verify_check.cu (built by nvcc, run without a GPU)
checks the chunk cap, the chunk split and the per-point scalars rho^i of csrc/srs.cuh, and the Python side of
Groth16.srs_verification_pairs -- its argument handling, done before the library is called -- is checked without a device."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from groth16_b200 import Srs, SrsPairs
from groth16_b200.api import srs_verify_args
from groth16_b200.params import get_curve

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_srs_verify_host(tmp_path):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path / "srs_verify_check")
    subprocess.check_call(["nvcc", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "--expt-relaxed-constexpr",
                           "-o", exe, os.path.join(ROOT, "tests", "host", "srs_verify_check.cu")])
    res = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    m = re.match(r"srs verify: (\d+) checks, 0 mismatches", res.stdout.strip())
    assert m and int(m.group(1)) >= 400, res.stdout


W1, W2 = 8, 16   # BN254: 4-limb Fq, G1 = 8 limbs, G2 over Fq2 = 16 limbs
R = get_curve("bn254").r


def _srs(n1=5, n2=3, na=3, nb=3):
    z = lambda rows, w: np.arange(rows * w, dtype=np.uint64).reshape(rows, w)
    return Srs(z(n1, W1), z(n2, W2), z(na, W1), z(nb, W1), np.ones(W2, dtype=np.uint64))


def test_arguments_accepted():
    arrs, rho, chunk = srs_verify_args(_srs(), 5, R, W1, W2)
    assert (rho, chunk) == (5, 0)
    assert [arrs[k].shape for k in ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1", "beta_g2")] == \
        [(5, W1), (3, W2), (3, W1), (3, W1), (W2,)]
    # the shortest transcript the check takes, rho reduced mod r (negative values too), the largest chunk cap
    _, rho, chunk = srs_verify_args(_srs(2, 2, 1, 1), R + 7, R, W1, W2, (1 << 64) - 1)
    assert (rho, chunk) == (7, (1 << 64) - 1)
    assert srs_verify_args(_srs(), -1, R, W1, W2)[1] == R - 1


@pytest.mark.parametrize("lens,member", [
    ((1, 3, 3, 3), "tau_g1"), ((0, 3, 3, 3), "tau_g1"), ((5, 1, 3, 3), "tau_g2"), ((5, 0, 3, 3), "tau_g2"),
    ((5, 3, 0, 3), "alpha_tau_g1"), ((5, 3, 3, 0), "beta_tau_g1"),
])
def test_members_too_short(lens, member):
    have = lens[("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1").index(member)]
    with pytest.raises(ValueError, match=rf"srs\.{member} holds {have} points, the check needs at least"):
        srs_verify_args(_srs(*lens), 5, R, W1, W2)


def test_missing_member_is_too_short():
    s = _srs()
    s.alpha_tau_g1 = None
    with pytest.raises(ValueError, match=r"srs\.alpha_tau_g1 holds 0 points"):
        srs_verify_args(s, 5, R, W1, W2)
    s = _srs()
    s.beta_g2 = None
    with pytest.raises(ValueError, match="beta_g2 is missing"):
        srs_verify_args(s, 5, R, W1, W2)


def test_partial_points_refused():
    s = _srs()
    s.tau_g2 = np.zeros((3, W1), dtype=np.uint64)
    with pytest.raises(ValueError, match="tau_g2"):
        srs_verify_args(s, 5, R, W1, W2)


@pytest.mark.parametrize("rho", [0, R, -R, 2 * R])
def test_zero_challenge_refused(rho):
    with pytest.raises(ValueError, match="rho must be non-zero"):
        srs_verify_args(_srs(), rho, R, W1, W2)


@pytest.mark.parametrize("chunk", [-1, 1 << 64])
def test_chunk_points_range(chunk):
    with pytest.raises(ValueError, match="chunk_points"):
        srs_verify_args(_srs(), 5, R, W1, W2, chunk)


def test_srs_pairs_equations():
    g1 = np.arange(10 * W1, dtype=np.uint64).reshape(10, W1)
    g2 = np.arange(10 * W2, dtype=np.uint64).reshape(10, W2)
    p = SrsPairs(g1, g2)
    assert p.members == ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1", "beta_g2")
    for k in range(5):
        P, Q, P2, Q2 = p.equation(k)
        assert np.array_equal(P, g1[2 * k]) and np.array_equal(P2, g1[2 * k + 1])
        assert np.array_equal(Q, g2[2 * k]) and np.array_equal(Q2, g2[2 * k + 1])
