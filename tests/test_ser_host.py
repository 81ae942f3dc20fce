"""CPU tier of the proving-key stream layout (csrc/ser.cuh, g16_pk_load_serialized / g16_pk_export_serialized):
tests/host/ser_check.cu, built by nvcc and run without a GPU, checks the walk of the length prefixes, the chunk planner and
the placement rule, at the field sizes of all four curves.  The per-point codec is checked in tests/test_ser_codec.py."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_ser_planner_host(tmp_path):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path / "ser_check")
    subprocess.check_call(["nvcc", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "--expt-relaxed-constexpr",
                           "-o", exe, os.path.join(ROOT, "tests", "host", "ser_check.cu")])
    res = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    lines = res.stdout.splitlines()
    assert lines[0].startswith("planner: ") and lines[0].endswith(", 0 mismatches"), lines[0]
    assert int(lines[0].split()[1]) > 15000, lines[0]
