"""CPU tests of the product's host-side pieces: field arithmetic back-ends (incl. the device carry-chain algorithm run
under an emulation of the PTX primitives), codecs, and the C ABI surface (symbols, loud failure without a GPU)."""
import ctypes as C
import os
import random
import re
import subprocess

import numpy as np
import pytest

import pyref as P
from groth16_b200 import CurveCodec, FieldCodec, _lib, get_curve

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _vectors():
    random.seed(7)
    names = {"bls12_381": "bls381", "bn254": "bn254", "bls12_377": "bls377"}
    lines = []
    for c in P.CURVES.values():
        for fld, p in (("fr", c.r), ("fq", c.q)):
            R = P.mont_R(p)
            Ri = pow(R, -1, p)
            vals = [0, 1, p - 1, p - 2, R % p, 2] + [random.randrange(p) for _ in range(30)]
            for i, a in enumerate(vals):
                b = vals[(i * 7 + 3) % len(vals)]
                mm = lambda x, y: x * y * Ri % p
                r = None
                for bit in bin(p - 2)[2:]:  # Fp::pow's left-to-right square-and-multiply under Montgomery products
                    if r is not None:
                        r = mm(r, r)
                    if bit == "1":
                        r = a if r is None else mm(r, a)
                lines.append(f"{names[c.name]}_{fld} {a:x} {b:x} {a * b * Ri % p:x} {(a + b) % p:x} {(a - b) % p:x} {r:x}")
    return "\n".join(lines) + "\n"


@pytest.mark.parametrize("flags", [[], ["-DG16_EMULATE_PTX"]], ids=["host_u64", "emulated_ptx"])
def test_fp_backends(tmp_path, flags):
    """fp.cuh: the plain host back-end and the device algorithm (even/odd-column Montgomery product on mad.lo.cc /
    madc.hi.cc chains) executed with emulated PTX carry semantics, both against Python big ints, all six fields."""
    exe = str(tmp_path / "fp_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-x", "c++", os.path.join(ROOT, "tests", "host", "fp_check.cpp"), "-o", exe] + flags)
    out = subprocess.run([exe], input=_vectors(), capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert " 0 mismatches" in out.stdout


def test_codec_roundtrip():
    for name in ("bls12_381", "bn254", "bls12_377"):
        c = P.CURVES[name]
        cd = CurveCodec(get_curve(name))
        vals = [0, 1, c.r - 1, 12345678901234567890123]
        assert cd.fr.dec(cd.fr.enc(vals)) == vals
        assert cd.fr.enc([1])[0].tolist() == [(P.to_mont(1, c.r) >> (64 * i)) & (2**64 - 1) for i in range(4)]
        cx = P.ctx(c)
        pts = [cx.g1_gen(), None, cx.G1.mul(cx.g1_gen(), 5)]
        assert cd.dec_g1(cd.enc_g1(pts)) == pts
        pts2 = [None, cx.g2_gen()]
        assert cd.dec_g2(cd.enc_g2(pts2)) == pts2
        assert not cd.enc_g1([None]).any()


def test_abi_exports_every_declared_symbol():
    """include/g16b200.h <-> libg16b200.so <-> groth16_b200/_lib.py agree on the symbol list."""
    with open(os.path.join(ROOT, "include", "g16b200.h")) as f:
        hdr = f.read()
    declared = set(re.findall(r"\b(g16_[a-z0-9_]+)\s*\(", hdr))
    bound = {n for n, _, _ in _lib.SIGNATURES}
    assert declared == bound, (declared ^ bound)
    lib = _lib.load()
    for n in declared:
        assert hasattr(lib, n), n


def test_no_cpu_fallback_without_gpu():
    """The product path must fail loudly, not fall back, when no CUDA device exists (this container has none)."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.g16_ctx_create(0, 0, C.byref(h)) == _lib.ERR_CUDA
    assert "no CPU fallback" in _lib.last_error()
    from groth16_b200 import CudaError, Groth16
    with pytest.raises(CudaError):
        Groth16("bls12_381")
    # null-context calls are rejected, not crashed
    assert lib.g16_prove(None, None, None, None, 0, None) == _lib.ERR_BAD_ARGUMENT


def test_product_does_not_import_oracle():
    """The shipped package never references oracle/ (SURVEY section 8c / task rule: oracle is test infrastructure)."""
    pkg = os.path.join(ROOT, "groth16_b200")
    for dp, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, fn)).read()
                assert "pyref" not in txt and "liboracle" not in txt and "import orc" not in txt, fn


def _ec_vectors():
    rng = P.Rng(77)
    lines = []

    def fmt1(pt):
        return "inf" if pt is None else f"{pt[0]:x} {pt[1]:x}"

    def fmt2(pt):
        return "inf" if pt is None else f"{pt[0][0]:x} {pt[0][1]:x} {pt[1][0]:x} {pt[1][1]:x}"

    for c in P.CURVES.values():
        cx = P.ctx(c)
        for grp, G, gen, fmt in (("g1", cx.G1, cx.g1_gen(), fmt1), ("g2", cx.G2, cx.g2_gen(), fmt2)):
            for _ in range(3):
                Pt, Q = G.mul(gen, rng.fr(c.r)), G.mul(gen, rng.fr(c.r))
                k = rng.fr(c.r)
                lines.append(f"{c.name} {grp} {fmt(Pt)} {fmt(Q)} {k:x} {fmt(G.add(Pt, Q))} {fmt(G.dbl(Pt))} {fmt(G.mul(Pt, k))}")
    return "\n".join(lines) + "\n"


def test_ec_host_backend(tmp_path):
    """ec.cuh (Fq2 tower, XYZZ group law incl. doubling / inverse / identity cases, scalar multiplication, to_affine):
    the host back-end that assembles the proof (prover.rs:76-131) against the big-int oracle, G1 and G2, three curves."""
    exe = str(tmp_path / "ec_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-x", "c++", os.path.join(ROOT, "tests", "host", "ec_check.cpp"), "-o", exe])
    out = subprocess.run([exe], input=_ec_vectors(), capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "18 vectors, 0 mismatches" in out.stdout


def test_msm_reduction_plan_host(tmp_path):
    """msm.cuh: the bucket-reduction plan (row / column sum tree, array layout) and its host recombination
    (MsmHostRed::T, msm_finish), the window / copies geometry and the entries-per-thread rule -- built by nvcc, executed on
    the CPU only, for bucket counts 2^2 .. 2^13 and 1 or 3 effective windows."""
    import shutil
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path / "msm_plan_check")
    subprocess.check_call(["nvcc", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-o", exe,
                           os.path.join(ROOT, "tests", "host", "msm_plan_check.cu")])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "18 cases, 0 mismatches" in out.stdout


def test_batched_affine_rounds_host(tmp_path):
    """msm_ba.cuh: the per-thread bodies of the batched-affine rounds (forward products, one inversion per combine lane,
    backward additions; tangent / opposite / identity cases; ragged buckets) executed on the CPU for G1 and both Fq2
    towers: every bucket of the reduced list sums to the plain XYZZ sum of its entries, and MsmBaPlan's bounds hold."""
    import shutil
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path / "ba_check")
    subprocess.check_call(["nvcc", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-o", exe,
                           os.path.join(ROOT, "tests", "host", "ba_check.cu")])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "24 cases, 0 mismatches" in out.stdout


def test_prepare_inputs_host_logic():
    """api.Groth16.prepare_inputs (verifier.rs:25-39) with the MSM call replaced by the CPU oracle: scalar conversion
    (ints and Montgomery limbs -> BigInt), the leading 1 for gamma_abc_g1[0], and the MalformedVerifyingKey check."""
    import orc
    import pyref as P
    from groth16_b200 import CurveCodec, Groth16, get_curve
    from util import check_prepare_inputs

    class CpuMsm(Groth16):
        def __init__(self, name):
            self.curve = get_curve(name)
            self.codec = CurveCodec(self.curve)
            self.nq = self.codec.nq
            self._cid = P.CURVES[name].cid

        def msm_g1(self, bases, scalars):
            return orc.msm_g1(self._cid, self.nq, bases, scalars, threads=2)

    for name in ("bn254", "bls12_381"):
        check_prepare_inputs(CpuMsm(name), name)


def test_safegcd_inversion_host(tmp_path):
    """fp_inv.cuh: Bernstein-Yang division-step inversion (signed 30-bit limbs) == Fermat inversion for all six fields:
    random elements, every 2^k and 2^k - 1, p - 1, p - 2, (p +- 1)/2, zero; x * inv(x) == 1."""
    exe = str(tmp_path / "inv_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-x", "c++", os.path.join(ROOT, "tests", "host", "inv_check.cpp"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "total 0 mismatches" in out.stdout
