"""CPU tier of CircomReduction (ark-circom's R1CSToQAP): the restatements in qap_circom_ref.py pinned against independent
evaluations, the proof identity the GPU tests rely on, and the shim's Rust source.

The identity: with the same toxic waste, (r, s) and a satisfying witness, the CircomReduction proof equals the
LibsnarkReduction proof.  The H query's scalars L_k are the Lagrange basis of the odd points omega_2n^(2j+1) evaluated at
tau, scaled by delta^-1, so sum_k L_k f(omega_2n^k) = delta^-1 f(tau) for deg f <= 2n - 2; f = ab - c vanishes on the even
points (c = a o b there), hence the H MSM sums to delta^-1 h(tau) Z(tau) G1 under both reductions and every other query is
the same."""
import os

import numpy as np
import pytest

import pyref as P
import qap_circom_ref as Q
from groth16_b200 import CurveCodec, get_curve
from groth16_b200.workload import synthetic_r1cs
from util import ALL_CURVES, matrices_from_r1cs, toxic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _circuits(c):
    rng = P.Rng(40)
    mimc_k = [rng.fr(c.r) for _ in range(6)]
    return {
        "silly": P.silly_circuit(c, rng.fr(c.r), rng.fr(c.r)),
        "mimc": P.mimc_circuit(c, rng.fr(c.r), rng.fr(c.r), mimc_k),
        "synthetic": P.synthetic_circuit(c, 13, seed=41, num_inputs=2),
    }


@pytest.mark.parametrize("curve", ALL_CURVES)
@pytest.mark.parametrize("satisfied", [True, False])
def test_witness_map_matches_naive_interpolation(curve, satisfied):
    """interpolate a, b and a o b by the O(n^2) DFT, then evaluate A B - C at omega_2n^(2j+1) directly"""
    c = P.CURVES[curve]
    cs = P.synthetic_circuit(c, 13, seed=42, num_inputs=2)
    if not satisfied:
        cs.assignment = list(cs.assignment)
        cs.assignment[5] = (cs.assignment[5] + 1) % c.r
        assert not cs.is_satisfied()
    dom, a, b, cc = P.abc_evals(cs)
    ab = [x * y % c.r for x, y in zip(a, b)]
    if not satisfied:
        assert ab != cc   # C z differs from a o b: the map must follow a o b
    # interpolation by the inverse DFT written out: coeff_k = n^-1 sum_i x_i omega^-ik
    inv_dom = P.Domain(c, dom.n)
    inv_dom.omega = dom.omega_inv
    interp = lambda x: [v * dom.n_inv % c.r for v in inv_dom.dft_naive(x)]
    w = Q.omega_2n(dom)
    ev = lambda co, pt: sum(cf * pow(pt, i, c.r) for i, cf in enumerate(co)) % c.r
    coA, coB, coC = interp(a), interp(b), interp(ab)
    want = []
    for j in range(dom.n):
        pt = pow(w, 2 * j + 1, c.r)
        want.append((ev(coA, pt) * ev(coB, pt) - ev(coC, pt)) % c.r)
    assert Q.witness_map(cs) == want
    assert pow(w, dom.n, c.r) == c.r - 1   # a primitive 2n-th root


@pytest.mark.parametrize("curve", ALL_CURVES)
@pytest.mark.parametrize("n_min", [1, 2, 8, 16])
def test_h_query_scalars_closed_form(curve, n_min):
    """the literal size-2n ifft against the closed form the library's setup evaluates, tau = 0 included"""
    c = P.CURVES[curve]
    rng = P.Rng(43 + n_min)
    dom = P.Domain(c, n_min)
    di = rng.fr(c.r)
    for tau in (rng.fr(c.r), 0, 1 + rng.below(1000)):
        assert Q.h_query_scalars(dom, tau, di) == Q.h_query_scalars_closed_form(dom, tau, di)
    assert len(Q.h_query_scalars(dom, 5, di)) == dom.n


@pytest.mark.parametrize("curve", ALL_CURVES)
@pytest.mark.parametrize("circuit", ["silly", "mimc", "synthetic"])
def test_circom_proof_equals_libsnark_proof(curve, circuit):
    c = P.CURVES[curve]
    cs = _circuits(c)[circuit]
    assert cs.is_satisfied()
    tw = toxic(c, 44)
    pk_l = Q.generate_parameters(cs, *tw, qap="libsnark")
    pk_c = Q.generate_parameters(cs, *tw, qap="circom")
    n = P.Domain(c, cs.num_constraints + cs.num_instance).n
    assert len(pk_l.h_query) == n - 1 and len(pk_c.h_query) == n
    for f in ("a_query", "b_g1_query", "b_g2_query", "l_query", "beta_g1", "delta_g1"):
        assert getattr(pk_l, f) == getattr(pk_c, f), f
    rng = P.Rng(45)
    for r_, s_ in ((rng.fr(c.r), rng.fr(c.r)), (0, rng.fr(c.r))):
        pf_l = Q.create_proof(pk_l, cs, r_, s_, qap="libsnark")
        pf_c = Q.create_proof(pk_c, cs, r_, s_, qap="circom")
        assert (pf_c.a, pf_c.b, pf_c.c) == (pf_l.a, pf_l.b, pf_l.c)
        pe = P.proof_in_the_exponent(pk_c, cs, r_, s_, h=Q.witness_map(cs))
        assert (pf_c.a, pf_c.b, pf_c.c) == (pe.a, pe.b, pe.c)
    if circuit == "silly":
        public = cs.assignment[1:cs.num_instance]
        assert P.verify_proof(pk_c.vk, c, pf_c, public)
        assert not P.verify_proof(pk_c.vk, c, pf_c, [(public[0] + 1) % c.r])


@pytest.mark.parametrize("curve", ALL_CURVES)
def test_unsatisfied_witness_is_rejected(curve):
    c = P.CURVES[curve]
    rng = P.Rng(46)
    a, b = rng.fr(c.r), rng.fr(c.r)
    cs = P.silly_circuit(c, a, b)
    cs.assignment = [1, (a * b + 1) % c.r, a, b]   # public c != a b
    assert not cs.is_satisfied()
    tw = toxic(c, 47)
    pk_l = Q.generate_parameters(cs, *tw, qap="libsnark")
    pk_c = Q.generate_parameters(cs, *tw, qap="circom")
    r_, s_ = rng.fr(c.r), rng.fr(c.r)
    pf_l = Q.create_proof(pk_l, cs, r_, s_, qap="libsnark")
    pf_c = Q.create_proof(pk_c, cs, r_, s_, qap="circom")
    assert pf_c.c != pf_l.c and (pf_c.a, pf_c.b) == (pf_l.a, pf_l.b)
    assert not P.verify_proof(pk_c.vk, c, pf_c, cs.assignment[1:2])


@pytest.mark.parametrize("curve", ALL_CURVES)
@pytest.mark.parametrize("satisfied", [True, False])
def test_oracle_transforms_match_pyref(curve, satisfied):
    """the 2^20-capable restatement on the C++ oracle's transforms equals the big-integer one, 1 and 3 threads"""
    c = P.CURVES[curve]
    cd = CurveCodec(get_curve(curve))
    m, z, _ = synthetic_r1cs(curve, 6, seed=48)
    zi = cd.fr.dec(z)
    if not satisfied:
        zi[9] = (zi[9] + 1) % c.r
        z = cd.fr.enc(zi)
    cs = P.R1CS(c, m.num_instance_variables, m.num_witness_variables, *_rows(cd, m), zi)
    assert cs.is_satisfied() == satisfied
    want = Q.witness_map(cs)
    dom = P.Domain(c, cs.num_constraints + cs.num_instance)
    tau, di = 0x1234567, 0x7654321
    want_h = Q.h_query_scalars(dom, tau, di)
    for thr in (1, 3):
        assert cd.fr.dec(Q.orc_witness_map(cd, m, z, threads=thr)) == want
        assert cd.fr.dec(Q.orc_h_query_scalars(cd, dom.log_n, tau, di, threads=thr)) == want_h


def _rows(cd, m):
    out = []
    for rp, col, val in (m.a, m.b, m.c):
        vals = cd.fr.dec(val) if len(col) else []
        out.append([[(vals[e], int(col[e])) for e in range(rp[i], rp[i + 1])] for i in range(m.num_constraints)])
    return out


def test_python_binding_accepts_the_two_reductions_only():
    from groth16_b200 import Groth16, _lib
    assert _lib.QAPS == {"libsnark": 0, "circom": 1}
    with pytest.raises(ValueError):
        Groth16("bn254", 0, qap="groth")


def test_shim_implements_circom_reduction():
    src = open(os.path.join(ROOT, "shim", "ark-groth16-b200", "src", "lib.rs")).read()
    sys_rs = open(os.path.join(ROOT, "shim", "ark-groth16-b200", "src", "sys.rs")).read()
    assert "impl R1CSToQAP for GpuCircomReduction" in src
    assert "sys::g16_circuit_load_qap(" in src
    assert "pub const G16_QAP_LIBSNARK: c_int = 0;" in sys_rs and "pub const G16_QAP_CIRCOM: c_int = 1;" in sys_rs
    header = open(os.path.join(ROOT, "include", "g16b200.h")).read()
    assert "G16_QAP_LIBSNARK = 0" in header and "G16_QAP_CIRCOM = 1" in header
