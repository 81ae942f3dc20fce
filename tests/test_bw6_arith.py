"""CPU tier of BW6-761's arithmetic: the 12-limb Fr and 24-limb Fq of fp.cuh, the safegcd inversion (fp_inv.cuh, checked
against the Fermat inversion at 761 bits) and the XYZZ point operations, on both host back-ends -- the plain 64-bit CIOS and
the device algorithm with emulated PTX carries -- at carry-chain edge operands (tests/bw6_arith.py).  The device build of
the same harness is checked by tests/test_gpu_bw6.py."""
import os
import subprocess

import pytest

import bw6_arith

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "arith_bw6", "bw6_arith.cu")


@pytest.mark.parametrize("flags", [[], ["-DG16_EMULATE_PTX"]], ids=["host_u64", "emulated_ptx"])
def test_bw6_arith_host(tmp_path, flags):
    so = str(tmp_path / "bw6arith.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", SRC, "-o", so] + flags)
    bad = bw6_arith.check_all(bw6_arith.load(so))
    assert not bad, bad[:5]
