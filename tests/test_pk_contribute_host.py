"""CPU tier of the phase-2 ceremony calls: tests/host/pk_contribute_check.cu (built by nvcc, run without a GPU) checks the
chunk split and range rule of g16_pk_contribute; the Python argument handling of Groth16.contribute_key and
Groth16.contribution_chain_pairs is checked without a device; and the header, the ctypes binding and the Rust shim must
declare both calls and their structs alike."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from groth16_b200 import ChainPairs, ContributionRecord, ProvingKey, VerifyingKey, _lib
from groth16_b200.api import chain_args, pk_contribute_args
from groth16_b200.params import get_curve
from test_shim_abi import header_functions, header_structs, rust_functions, rust_structs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W1, W2 = 8, 16   # BN254: G1 = 8 limbs, G2 = 16
R = get_curve("bn254").r


def test_pk_contribute_host(tmp_path):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path / "pk_contribute_check")
    subprocess.check_call(["nvcc", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "--expt-relaxed-constexpr",
                           "-o", exe, os.path.join(ROOT, "tests", "host", "pk_contribute_check.cu")])
    res = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    m = re.match(r"pk contribute: (\d+) checks, 0 mismatches", res.stdout.strip())
    assert m and int(m.group(1)) >= 300, res.stdout


def _key(nh=7, nl=5):
    z = lambda rows, w: np.arange(rows * w, dtype=np.uint64).reshape(rows, w)
    vk = VerifyingKey(z(1, W1)[0], z(1, W2)[0], z(1, W2)[0] + 1, z(1, W2)[0] + 2, z(2, W1))
    return ProvingKey(vk, z(1, W1)[0], z(1, W1)[0] + 3, z(7, W1), z(7, W1), z(7, W2), z(nh, W1), z(nl, W1))


def test_pk_contribute_args():
    pk = _key()
    arrs, delta, chunk = pk_contribute_args(pk, R + 5, R, W1, W2, 7)
    assert delta == 5 and chunk == 7
    assert arrs["h_query"].shape == (7, W1) and arrs["l_query"].shape == (5, W1)
    assert arrs["delta_g1"].shape == (W1,) and arrs["delta_g2"].shape == (W2,)
    assert all(a.flags["C_CONTIGUOUS"] and a.dtype == np.uint64 for a in arrs.values())
    # in place: the arrays handed to the library are the key's own
    arrs = pk_contribute_args(pk, 5, R, W1, W2, in_place=True)[0]
    assert np.shares_memory(arrs["h_query"], pk.h_query) and np.shares_memory(arrs["delta_g2"], pk.vk.delta_g2)
    # a flat list of whole points and empty queries are accepted
    pk.h_query, pk.l_query = pk.h_query.reshape(-1).tolist(), np.zeros((0, W1), dtype=np.uint64)
    arrs = pk_contribute_args(pk, 5, R, W1, W2)[0]
    assert arrs["h_query"].shape == (7, W1) and arrs["l_query"].shape == (0, W1)


@pytest.mark.parametrize("edit,match", [
    (lambda pk: setattr(pk, "h_query", np.zeros((3, W1 + 1), dtype=np.uint64)), "h_query of shape"),
    (lambda pk: setattr(pk, "l_query", None), "the key has no l_query"),
    (lambda pk: setattr(pk, "delta_g1", np.zeros(2 * W1, dtype=np.uint64)), "delta_g1 holds 2 points, it is one point"),
    (lambda pk: setattr(pk.vk, "delta_g2", np.zeros(W1, dtype=np.uint64)), "delta_g2 of shape"),
])
def test_pk_contribute_args_refused(edit, match):
    pk = _key()
    edit(pk)
    with pytest.raises(ValueError, match=match):
        pk_contribute_args(pk, 5, R, W1, W2)


@pytest.mark.parametrize("delta", [0, R, -R])
def test_zero_delta_refused(delta):
    with pytest.raises(ValueError, match="UnexpectedIdentity"):
        pk_contribute_args(_key(), delta, R, W1, W2)


def test_pk_contribute_args_chunks_and_in_place():
    for bad in (-1, 1 << 64):
        with pytest.raises(ValueError, match="chunk_points"):
            pk_contribute_args(_key(), 5, R, W1, W2, bad)
    pk = _key()
    pk.l_query = pk.l_query.astype(np.int64)   # converted: a copy, so not in place
    with pytest.raises(ValueError, match="l_query"):
        pk_contribute_args(pk, 5, R, W1, W2, in_place=True)
    pk = _key()
    pk.vk.delta_g2.flags.writeable = False
    with pytest.raises(ValueError, match="delta_g2"):
        pk_contribute_args(pk, 5, R, W1, W2, in_place=True)
    pk_contribute_args(pk, 5, R, W1, W2)   # the same key is fine out of place


def _rec(k=0):
    p = lambda w: np.full(w, k + 1, dtype=np.uint64)
    return ContributionRecord(p(W1), p(W1) + 1, p(W1) + 2, p(W2), p(W2) + 1)


def test_chain_args():
    start, end, recs = chain_args(np.ones(W1, dtype=np.uint64), [2] * W1, [_rec(0), _rec(1)], W1, W2)
    assert start.shape == end.shape == (W1,) and end.dtype == np.uint64
    assert len(recs) == 2 and recs[1]["r_x_g2"].shape == (W2,) and recs[1]["s_g1"][0] == 3
    with pytest.raises(ValueError, match="1 to 2\\^30 - 1 records, not 0"):
        chain_args(np.ones(W1), np.ones(W1), [], W1, W2)
    with pytest.raises(ValueError, match=r"^records\[1\]\.r_g2 holds 8 limbs, one point is 16$"):
        bad = _rec(1)
        bad.r_g2 = np.zeros(W1, dtype=np.uint64)
        chain_args(np.ones(W1), np.ones(W1), [_rec(0), bad], W1, W2)
    with pytest.raises(ValueError, match=r"^start_g1 is missing$"):
        chain_args(None, np.ones(W1), [_rec(0)], W1, W2)
    with pytest.raises(ValueError, match=r"^end_g1 holds 16 limbs"):
        chain_args(np.ones(W1), np.ones(W2), [_rec(0)], W1, W2)


def test_chain_pairs_equations():
    g1 = np.arange(12 * W1, dtype=np.uint64).reshape(12, W1)
    g2 = np.arange(12 * W2, dtype=np.uint64).reshape(12, W2)
    p = ChainPairs(g1, g2)
    assert len(p) == 6
    for k in range(6):
        P, Q, P2, Q2 = p.equation(k)
        assert np.array_equal(P, g1[2 * k]) and np.array_equal(P2, g1[2 * k + 1])
        assert np.array_equal(Q, g2[2 * k]) and np.array_equal(Q2, g2[2 * k + 1])
    with pytest.raises(IndexError):
        p.equation(6)


def test_declarations_agree():
    """header, ctypes and Rust declare both calls alike, and the three structs have the same fields in all three"""
    h, r = header_functions(), rust_functions()
    assert h["g16_pk_contribute"] == r["g16_pk_contribute"] == [True, True, True, False, False, True]
    assert h["g16_contribution_chain_pairs"] == r["g16_contribution_chain_pairs"] == \
        [True, True, True, True, False, False, True, True]
    py = {name: args for name, _, args in _lib.SIGNATURES}
    assert len(py["g16_pk_contribute"]) == 6 and len(py["g16_contribution_chain_pairs"]) == 8
    hs, rs = header_structs(), rust_structs()
    for name, cls in (("g16_pk_delta_desc", _lib.PkDeltaDesc), ("g16_pk_delta_out", _lib.PkDeltaOut),
                      ("g16_contribution_record", _lib.ContributionRecord)):
        assert hs[name] == rs[name] == [f for f, _ in cls._fields_], name
    assert hs["g16_contribution_record"] == ["after_g1", "s_g1", "s_x_g1", "r_g2", "r_x_g2"]
    lib_rs = open(os.path.join(ROOT, "shim", "ark-groth16-b200", "src", "lib.rs")).read()
    for fn in ("pub fn contribute_key", "pub fn contribution_chain_pairs", "pub fn verify_contribution_chain",
               "pub struct ContributionRecord", "pub fn make"):
        assert fn in lib_rs, fn
