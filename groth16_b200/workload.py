"""Synthetic R1CS workloads for bench.py and the full-size tests (SURVEY.md section 8d).

* synthetic_r1cs : non-degenerate circuit -- constraint i is (z_p + k_i) * z_q = z_new with p, q uniform over earlier
                   variables; two uniformly random seed witnesses; dense queries, witness values uniform-looking in
                   [0, r).  Sized so that num_constraints + num_instance_variables == 2^log_n exactly (the sizing
                   trick of benches/bench.rs:19-20).
* dummy_r1cs     : the reference's own DummyCircuit (benches/bench.rs:41-64): constant witness, A/B rows touching
                   two variables only (degenerate: almost every a/b query element is the identity).
Both return (ConstraintMatrices, full_assignment as Montgomery limbs, public inputs as ints).
"""
from __future__ import annotations

import numpy as np

from .api import ConstraintMatrices
from .codec import CurveCodec
from .params import get_curve


def _splitmix(seed: int):
    s = seed & 0xFFFFFFFFFFFFFFFF
    M = 0xFFFFFFFFFFFFFFFF
    while True:
        s = (s + 0x9E3779B97F4A7C15) & M
        z = s
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
        yield z ^ (z >> 31)


def _fr(gen, r):
    bits = r.bit_length()
    while True:
        v = next(gen) | (next(gen) << 64) | (next(gen) << 128) | (next(gen) << 192)
        v &= (1 << bits) - 1
        if v < r:
            return v


_WORKLOAD_LIB = None


def _workload_lib():
    """groth16_b200/libg16workload.so: csrc/workload.cu built with the host compiler alone (same generator, no CUDA runtime).
    Preferred when present, so that a process that only needs a circuit -- bench.py's `--impl reference` arm -- never maps the
    CUDA library; falls back to the copy inside libg16b200.so."""
    global _WORKLOAD_LIB
    if _WORKLOAD_LIB is None:
        import ctypes as C
        import os
        p = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libg16workload.so")
        try:
            _WORKLOAD_LIB = C.CDLL(p) if os.path.exists(p) else False
        except OSError:          # unloadable on this host: the copy inside libg16b200.so serves
            _WORKLOAD_LIB = False
    return _WORKLOAD_LIB or None


def synthetic_r1cs(curve, log_n: int, seed: int = 0, num_inputs: int = 1):
    """The synthetic R1CS of SURVEY.md section 8d through g16_synthetic_r1cs (csrc/workload.cu: host code of the library, no
    GPU needed; a Python loop over 2^24 constraints would take minutes).  One public input."""
    import ctypes as C
    from . import _lib
    if num_inputs != 1:
        raise ValueError("the generator has exactly one public input")
    c = get_curve(curve)
    cd = CurveCodec(c)
    ninst = 2
    nc = (1 << log_n) - ninst
    if log_n < 3:
        raise ValueError("domain too small")
    nwit = nc + 1
    a_col = np.empty(2 * nc, dtype=np.uint32)
    a_val = np.empty((2 * nc, cd.fr.nl), dtype=np.uint64)
    b_col = np.empty(nc, dtype=np.uint32)
    c_col = np.empty(nc, dtype=np.uint32)
    z = np.zeros((ninst + nwit, cd.fr.nl), dtype=np.uint64)
    vp = lambda x: x.ctypes.data_as(C.c_void_p)
    lib = _workload_lib()
    fn = (lib or _lib.load()).g16_synthetic_r1cs
    if lib is not None:
        fn.argtypes = [C.c_int, C.c_uint32, C.c_uint64] + [C.c_void_p] * 5
        fn.restype = C.c_int
    rc = fn(c.cid, log_n, seed & 0xFFFFFFFFFFFFFFFF, vp(a_col), vp(a_val), vp(b_col), vp(c_col), vp(z))
    if rc != 0:
        if lib is not None:
            lib.g16_workload_last_error.restype = C.c_char_p
            raise ValueError(lib.g16_workload_last_error().decode())
        raise ValueError(_lib.last_error())
    one = np.ascontiguousarray(cd.fr.enc1(1))
    a_rp = np.arange(0, 2 * nc + 1, 2, dtype=np.uint32)
    b_rp = np.arange(0, nc + 1, dtype=np.uint32)
    ones = np.ascontiguousarray(np.broadcast_to(one, (nc, cd.fr.nl)))
    m = ConstraintMatrices(ninst, nwit, nc, (a_rp, a_col, a_val), (b_rp, b_col, ones), (b_rp.copy(), c_col, ones.copy()))
    return m, z, cd.fr.dec(z[1:ninst])


def dummy_r1cs(curve, num_variables: int, num_constraints: int, seed: int = 0):
    c = get_curve(curve)
    cd = CurveCodec(c)
    r = c.r
    gen = _splitmix(seed)
    a, b = _fr(gen, r), _fr(gen, r)
    nwit = num_variables - 1
    one = cd.fr.enc1(1)
    nc = num_constraints
    rp = np.concatenate([np.arange(0, nc, dtype=np.uint32), np.array([nc - 1], dtype=np.uint32)])  # last row empty
    mk = lambda col: (rp.copy(), np.full(nc - 1, col, dtype=np.uint32), np.ascontiguousarray(np.tile(one, (nc - 1, 1))))
    m = ConstraintMatrices(2, nwit, nc, mk(2), mk(3), mk(1))
    full = [1, a * b % r, a, b] + [a] * (num_variables - 3)
    z = np.ascontiguousarray(cd.fr.enc(full))
    return m, z, full[1:2]
