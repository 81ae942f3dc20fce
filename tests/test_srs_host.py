"""CPU tier of the transcript setup's host code and compile evidence: tests/host/srs_plan_check.cu (built by nvcc, run
without a GPU) checks the sparse-sum planner of csrc/srs.cuh, and the ptxas reports of the four k_srs_<curve>.o objects must
show no spills in any kernel or function they compile."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "groth16_b200", "csrc")
CURVES = ("bls381", "bn254", "bls377", "bw6")


def test_srs_planner_host(tmp_path):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path / "srs_plan_check")
    subprocess.check_call(["nvcc", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "--expt-relaxed-constexpr",
                           "-o", exe, os.path.join(ROOT, "tests", "host", "srs_plan_check.cu")])
    res = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    m = re.match(r"srs planner: (\d+) checks, 0 mismatches", res.stdout.strip())
    assert m and int(m.group(1)) > 1000, res.stdout


@pytest.mark.parametrize("curve", CURVES)
def test_srs_kernels_do_not_spill(curve):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    obj = f"k_srs_{curve}.o"
    log = os.path.join(CSRC, f"k_srs_{curve}.ptxas.log")
    subprocess.check_call(["make", "-s", "-C", CSRC, obj])
    if not os.path.exists(log) or os.path.getmtime(log) < os.path.getmtime(os.path.join(CSRC, obj)) - 1:
        os.remove(os.path.join(CSRC, obj))   # the report is written by the compile: make one
        subprocess.check_call(["make", "-s", "-C", CSRC, obj])
    txt = open(log).read()
    entries = re.findall(r"Compiling entry function '(\w+)'", txt)
    assert len(entries) >= (11 if curve == "bw6" else 20), entries
    assert all("srs_" in e for e in entries), entries
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", txt)
    assert spills and all(s == ("0", "0") for s in spills), \
        [ln for ln in txt.splitlines() if "spill" in ln and "0 bytes spill stores, 0 bytes spill loads" not in ln]
