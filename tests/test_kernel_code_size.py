"""CPU test of the compiled BLS12-381 MSM kernels: every hot kernel calls one out-of-line Fq product body instead of
inlining each product (fp.cuh, Fp::mont_mul_call).  Inlined, the G2 kernels spill and the proof is slower (DESIGN.md
section 3).  Guards against a change that quietly inlines the products again, against register spills in the batched-affine
round kernels, and against hot kernels appearing or disappearing: each object holds exactly the seven listed in HOT."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "groth16_b200", "csrc")


def _cuobjdump():
    for p in (shutil.which("cuobjdump"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")):
        if p and os.path.exists(p):
            return p
    return None


CUOBJDUMP = _cuobjdump()
pytestmark = pytest.mark.skipif(CUOBJDUMP is None, reason="cuobjdump (CUDA toolkit) not found")

# Hot kernels (mangled-name fragments) and the SASS size each must stay under.  A kernel's text includes its copy of the
# out-of-line product and point-operation bodies.  Inlined, these kernels were 60..200 KB (G1) and 140..560 KB (G2).
HOT = ("ba_forward_kernel", "ba_backward_kernel", "ba_combine_kernel", "msm_accum_l0", "msm_accum_ln", "msm_accum_tail",
       "msm_sum_strided")
MAX_KB = {"g1": 64, "g2": 176}
# An inlined 12-limb Montgomery product is ~290 IMAD.WIDE / IMAD.HI; more than two products' worth means inlined copies.
MAX_WIDE_MULS = 2 * 330


def _objects():
    objs = {g: os.path.join(CSRC, f"k_msm_{g}_bls381.o") for g in ("g1", "g2")}
    subprocess.check_call(["make", "-s", "-C", CSRC] + [os.path.basename(o) for o in objs.values()])
    return objs


def _sass(obj):
    """{mangled function name: (bytes of SASS, IMAD.WIDE/IMAD.HI count)} for every kernel in the object."""
    out = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    res, fn = {}, None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            fn = m.group(1)
            res[fn] = [0, 0]
        elif fn and re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
            res[fn][0] += 16
            if "IMAD.WIDE" in line or "IMAD.HI" in line:
                res[fn][1] += 1
    return res


def _res_usage(obj):
    """{mangled function name: {'REG': .., 'STACK': .., 'LOCAL': ..}}"""
    out = subprocess.run([CUOBJDUMP, "-res-usage", obj], capture_output=True, text=True, check=True).stdout
    res, fn = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            fn = m.group(1)
        elif fn and "REG:" in line:
            res[fn] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
    return res


@pytest.fixture(scope="module")
def objects():
    return _objects()


@pytest.mark.parametrize("group", ["g1", "g2"])
def test_hot_kernel_set_and_size(objects, group):
    sass = _sass(objects[group])
    hot = {fn: v for fn, v in sass.items() if any(re.search(rf"\d{h}I", fn) for h in HOT)}
    # exactly one instance of each: the three round kernels and the four accumulation kernels
    assert sorted(next(h for h in HOT if re.search(rf"\d{h}I", fn)) for fn in hot) == sorted(HOT), sorted(sass)
    for fn, (size, wide) in hot.items():
        assert size <= MAX_KB[group] * 1024, f"{fn}: {size / 1024:.1f} KB of SASS (limit {MAX_KB[group]} KB)"
        assert wide <= MAX_WIDE_MULS, f"{fn}: {wide} wide multiplies: Fq products are inlined again"


@pytest.mark.parametrize("group", ["g1", "g2"])
def test_round_kernels_do_not_spill(objects, group):
    use = _res_usage(objects[group])
    rounds = {fn: u for fn, u in use.items() if re.search(r"\d(ba_forward_kernel|ba_backward_kernel)I", fn)}
    assert len(rounds) == 2, sorted(use)
    for fn, u in rounds.items():
        assert u["STACK"] == 0 and u["LOCAL"] == 0, f"{fn}: {u}"
