"""CPU tier of g16_pk_verify_pairs (the key check): the Python side of Groth16.key_verification_pairs -- its argument
handling, done before the library is called -- without a device, and the declarations of the call in the header, the
ctypes binding and the Rust shim."""
import os
import re

import numpy as np
import pytest

from groth16_b200 import KEY_EQUATIONS, KeyPairs, ProvingKey, Srs, VerifyingKey, _lib
from groth16_b200.api import pk_verify_args
from groth16_b200.params import get_curve
from test_shim_abi import header_functions, header_structs, rust_functions, rust_structs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W1, W2 = 8, 16   # BN254: G1 = 8 limbs, G2 = 16
R = get_curve("bn254").r
NI, NW, LOG_N = 2, 5, 3   # n = 8


def _key(nv=NI + NW, hn=7, nw=NW, ni=NI):
    z = lambda rows, w: np.arange(rows * w, dtype=np.uint64).reshape(rows, w)
    vk = VerifyingKey(z(1, W1)[0], z(1, W2)[0], z(1, W2)[0] + 1, z(1, W2)[0] + 2, z(ni, W1))
    return ProvingKey(vk, z(1, W1)[0], z(1, W1)[0] + 3, z(nv, W1), z(nv, W1), z(nv, W2), z(hn, W1), z(nw, W1))


def _srs(n1=15, n2=8, na=8, nb=8):
    z = lambda rows, w: np.zeros((rows, w), dtype=np.uint64)
    return Srs(z(n1, W1), z(n2, W2), z(na, W1), z(nb, W1), np.ones(W2, dtype=np.uint64))


def _args(pk=None, srs=None, rho=5, qap="libsnark"):
    return pk_verify_args(pk or _key(), srs or _srs(), rho, R, W1, W2, NI, NW, LOG_N, qap)


def test_arguments_accepted():
    keys, arrs, rho = _args()
    assert rho == 5
    assert keys["a_query"].shape == (NI + NW, W1) and keys["b_g2_query"].shape == (NI + NW, W2)
    assert keys["h_query"].shape == (7, W1) and keys["gamma_abc_g1"].shape == (NI, W1)
    assert all(keys[k].shape == (1, W2 if k in ("beta_g2", "gamma_g2", "delta_g2") else W1)
               for k in ("alpha_g1", "beta_g1", "delta_g1", "beta_g2", "gamma_g2", "delta_g2"))
    # CircomReduction: n points of H; a longer transcript; rho reduced mod r
    assert _args(pk=_key(hn=8), qap="circom")[0]["h_query"].shape == (8, W1)
    assert _args(srs=_srs(100, 60, 60, 60), rho=R + 7)[2] == 7
    assert _args(rho=-1)[2] == R - 1


@pytest.mark.parametrize("member,kw,have,need", [
    ("a_query", dict(nv=6), 6, 7), ("h_query", dict(hn=8), 8, 7), ("l_query", dict(nw=4), 4, 5),
    ("gamma_abc_g1", dict(ni=3), 3, 2),
])
def test_key_member_lengths(member, kw, have, need):
    with pytest.raises(ValueError, match=rf"^{member} holds {have} points, the circuit's key has {need}$"):
        _args(pk=_key(**kw))


def test_circom_h_query_length():
    with pytest.raises(ValueError, match=r"^h_query holds 7 points, the circuit's key has 8$"):
        _args(qap="circom")


def test_malformed_key_members():
    pk = _key()
    pk.vk.gamma_abc_g1 = None
    with pytest.raises(ValueError, match="no gamma_abc_g1"):
        _args(pk=pk)
    pk = _key()
    pk.b_g2_query = np.zeros((7, W1), dtype=np.uint64)   # G1-sized points where G2 points belong
    with pytest.raises(ValueError, match=r"b_g2_query of shape \(7, 8\) is not made of points of 16 limbs"):
        _args(pk=pk)
    pk = _key()
    pk.vk.delta_g2 = np.zeros(W2 + 1, dtype=np.uint64)
    with pytest.raises(ValueError, match="delta_g2 of shape"):
        _args(pk=pk)


@pytest.mark.parametrize("lens,member,need", [
    ((14, 8, 8, 8), "tau_g1", 15), ((15, 7, 8, 8), "tau_g2", 8), ((15, 8, 0, 8), "alpha_tau_g1", 8),
    ((15, 8, 8, 7), "beta_tau_g1", 8),
])
def test_transcript_too_short(lens, member, need):
    have = lens[("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1").index(member)]
    with pytest.raises(ValueError, match=rf"srs\.{member} holds {have} points, the circuit \(domain 2\^3\) needs at least {need}"):
        _args(srs=_srs(*lens))


@pytest.mark.parametrize("rho", [0, R, -R, 2 * R])
def test_zero_challenge_refused(rho):
    with pytest.raises(ValueError, match="rho must be non-zero"):
        _args(rho=rho)


def test_key_pairs_equations():
    g1 = np.arange(8 * W1, dtype=np.uint64).reshape(8, W1)
    g2 = np.arange(8 * W2, dtype=np.uint64).reshape(8, W2)
    p = KeyPairs(g1, g2)
    assert p.members == KEY_EQUATIONS == ("delta", "h_query", "l_query", "gamma_abc_g1")
    for k in range(4):
        P, Q, P2, Q2 = p.equation(k)
        assert np.array_equal(P, g1[2 * k]) and np.array_equal(P2, g1[2 * k + 1])
        assert np.array_equal(Q, g2[2 * k]) and np.array_equal(Q2, g2[2 * k + 1])


def test_declarations_agree():
    """header, ctypes and Rust declare the call alike; the key's struct has the export struct's members; the flag has one
    value in all three"""
    h, r = header_functions(), rust_functions()
    assert h["g16_pk_verify_pairs"] == r["g16_pk_verify_pairs"] == [True, True, True, True, False, True, True]
    py = {name: args for name, _, args in _lib.SIGNATURES}
    assert len(py["g16_pk_verify_pairs"]) == 7
    hs, rs = header_structs(), rust_structs()
    assert hs["g16_pk_check_desc"] == rs["g16_pk_check_desc"] == hs["g16_pk_export_desc"]
    assert [f for f, _ in _lib.PkCheckDesc._fields_] == hs["g16_pk_check_desc"]
    hdr = open(os.path.join(ROOT, "include", "g16b200.h")).read()
    sysrs = open(os.path.join(ROOT, "shim", "ark-groth16-b200", "src", "sys.rs")).read()
    flag = int(re.search(r"G16_PK_UNCONTRIBUTED = (\d+)", hdr).group(1))
    assert flag == _lib.PK_UNCONTRIBUTED == int(re.search(r"G16_PK_UNCONTRIBUTED: u32 = (\d+)", sysrs).group(1))
    assert flag & _lib.SER_VALIDATE == 0
    lib_rs = open(os.path.join(ROOT, "shim", "ark-groth16-b200", "src", "lib.rs")).read()
    assert "pub fn key_verification_pairs" in lib_rs and "pub fn verify_key" in lib_rs
