"""CPU tier of batch proving (g16_prove_batch): tests/host/batch_plan_check.cu, built by nvcc and run without a GPU, checks the
bucket-reduction layout of K proofs x ne bucket sets (msm_finish(ws, g, k) is proof k's Horner sum and nothing else), that a
zero-initialised MsmGeom is one MSM, the group-size rule, the proof tail every prover path shares against the prover.rs
order, and that the per-proof workspace bound which sizes an automatic group covers what a group's MSM workspaces reserve."""
import os
import shutil
import subprocess

import pytest

from groth16_b200 import CurveCodec, get_curve
from groth16_b200.params import GENERATORS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _generator_limbs():
    """G1 then G2 generator of BN254 and BLS12-381, as hex Montgomery limbs (the order batch_plan_check reads them)"""
    out = []
    for curve in ("bn254", "bls12_381"):
        cd = CurveCodec(get_curve(curve))
        G = GENERATORS[curve]
        for arr in (cd.enc_g1([G["g1"]])[0], cd.enc_g2([G["g2"]])[0]):
            out.extend(f"{int(x):x}" for x in arr)
    return " ".join(out) + "\n"


def test_batch_plan_and_proof_tail_host(tmp_path):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path / "batch_plan_check")
    subprocess.check_call(["nvcc", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-o", exe,
                           os.path.join(ROOT, "tests", "host", "batch_plan_check.cu")])
    res = subprocess.run([exe], input=_generator_limbs(), capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout + res.stderr
    assert ", 0 mismatches" in res.stdout, res.stdout
    checks = int(res.stdout.split()[0])
    assert checks >= 60, res.stdout          # layout, geometry and group-size checks plus 96 tail cases
    assert "(96 tail cases)" in res.stdout, res.stdout
    assert "workspace bound: 0 group passes over it" in res.stdout, res.stdout
