"""CPU tier of g16_srs_contribute (phase-1 contributions): tests/host/srs_contribute_check.cu (built by nvcc, run without a
GPU) checks the chunk split and the per-point power scheme of csrc/srs.cuh, and the Python side of
Groth16.contribute_srs -- how it hands a transcript's arrays to the library -- is checked without a device."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from groth16_b200 import Srs
from groth16_b200.api import srs_arrays

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_srs_contribute_host(tmp_path):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path / "srs_contribute_check")
    subprocess.check_call(["nvcc", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "--expt-relaxed-constexpr",
                           "-o", exe, os.path.join(ROOT, "tests", "host", "srs_contribute_check.cu")])
    res = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    m = re.match(r"srs contribute: (\d+) checks, 0 mismatches", res.stdout.strip())
    assert m and int(m.group(1)) >= 150, res.stdout


W1, W2 = 8, 16   # BN254: 4-limb Fq, G1 = 8 limbs, G2 over Fq2 = 16 limbs


def _srs(n1=5, n2=3):
    z = lambda rows, w: np.arange(rows * w, dtype=np.uint64).reshape(rows, w)
    return Srs(z(n1, W1), z(n2, W2), z(n2, W1), z(n2, W1), np.ones(W2, dtype=np.uint64))


def test_srs_arrays_shapes():
    s = _srs()
    a = srs_arrays(s, W1, W2)
    assert [a[k].shape for k in ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1", "beta_g2")] == \
        [(5, W1), (3, W2), (3, W1), (3, W1), (W2,)]
    assert all(a[k].flags["C_CONTIGUOUS"] and a[k].dtype == np.uint64 for k in a)
    # a flat vector of whole points and a list of Python ints are accepted; a missing vector is empty
    s2 = Srs(s.tau_g1.reshape(-1), s.tau_g2.tolist(), None, s.beta_tau_g1[:0], s.beta_g2.tolist())
    a2 = srs_arrays(s2, W1, W2)
    assert a2["tau_g1"].shape == (5, W1) and np.array_equal(a2["tau_g1"], s.tau_g1)
    assert a2["tau_g2"].shape == (3, W2) and np.array_equal(a2["tau_g2"], s.tau_g2)
    assert a2["alpha_tau_g1"].shape == (0, W1) and a2["beta_tau_g1"].shape == (0, W1)
    assert a2["beta_g2"].shape == (W2,)


def test_srs_arrays_in_place_shares_memory():
    s = _srs()
    a = srs_arrays(s, W1, W2, in_place=True)
    for k in ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1", "beta_g2"):
        assert np.shares_memory(a[k], getattr(s, k)), k
    a["tau_g1"][0, 0] = 99   # a write through the array handed to the library lands in the caller's transcript
    assert s.tau_g1[0, 0] == 99


@pytest.mark.parametrize("member,value,match", [
    ("tau_g1", np.zeros((3, W1 + 1), dtype=np.uint64), "tau_g1"),
    ("tau_g2", np.zeros((2, W1), dtype=np.uint64), "tau_g2"),
    ("alpha_tau_g1", np.zeros(W1 * 2 + 1, dtype=np.uint64), "alpha_tau_g1"),
    ("beta_tau_g1", np.zeros((2, 2, W1), dtype=np.uint64), "beta_tau_g1"),
    ("beta_g2", np.zeros(W2 * 2, dtype=np.uint64), "beta_g2"),
    ("beta_g2", None, "beta_g2 is missing"),
])
def test_srs_arrays_refuses_partial_points(member, value, match):
    s = _srs()
    setattr(s, member, value)
    with pytest.raises(ValueError, match=match):
        srs_arrays(s, W1, W2)


def test_srs_arrays_in_place_needs_writable_uint64():
    s = _srs()
    s.alpha_tau_g1 = s.alpha_tau_g1.astype(np.int64)   # would be converted: a copy, so not in place
    with pytest.raises(ValueError, match="alpha_tau_g1"):
        srs_arrays(s, W1, W2, in_place=True)
    s = _srs()
    s.tau_g2 = np.asfortranarray(np.zeros((3, W2), dtype=np.uint64))
    with pytest.raises(ValueError, match="tau_g2"):
        srs_arrays(s, W1, W2, in_place=True)
    s = _srs()
    s.beta_g2.flags.writeable = False
    with pytest.raises(ValueError, match="beta_g2"):
        srs_arrays(s, W1, W2, in_place=True)
    s = _srs()
    s.tau_g1 = s.tau_g1.tolist()
    with pytest.raises(ValueError, match="tau_g1"):
        srs_arrays(s, W1, W2, in_place=True)
    srs_arrays(s, W1, W2)   # the same transcript is fine out of place
