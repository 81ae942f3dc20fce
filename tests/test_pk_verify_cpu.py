"""CPU tier of the key check (g16_pk_verify_pairs), with big integers in the scalar field of all four curves: the
transcript-side weights the library forms by field transforms (pk_verify_ref.transcript_sides) must equal sum_j rho^j
times the exponents of the directly derived key, under both reductions, on circuits with n = 4 to 64 -- instance-heavy
ones, an unused variable and rows that use the One column among them.  The directly derived key is pk_verify_ref's
Lagrange form, itself checked against pyref's setup, qap_circom_ref's H query and bw6_ref.  Honest keys pass; each
tampering breaks exactly the check or equation pk_verify_ref names."""
import random

import pytest

import bw6_ref as B
import pyref as P
import qap_circom_ref as Q
from pk_verify_ref import (EXPECTED, domain, edited_rows, failing, key_exponents, key_sums, tamperings, transcript_sides,
                           transcript_sums, verdict)

TAU, ALPHA, BETA, GAMMA, DELTA = (0x1234567890ABCDEF1234567, 0x2222222222222222222223, 0x3333333333333333333335,
                                  0x6666666666666666666661, 0x4444444444444444444447)
TAU2 = 0x7777777777777777777779ABC
RHO = 0x5EED5EED5EED5EED5EED5EED5EED5EED1
CURVES4 = ["bls12_381", "bn254", "bls12_377", "bw6_761"]


def field(curve):
    """(r, root(L)); BW6-761 takes its circuits from BLS12-377, whose q is its r"""
    if curve == "bw6_761":
        return B.R, B.domain_root
    c = P.CURVES[curve]
    return c.r, (lambda L: P.Domain(c, 1 << L).omega)


def mixed_circuit(r, ni, nw, nc, seed):
    """random rows over ni instance and nw witness variables: variable ni + 1 unused, every row of C reads One (column 0),
    row 0 of A is One alone"""
    rng = random.Random(seed)
    used = [v for v in range(ni + nw) if v != ni + 1]
    rand_row = lambda k: [(rng.randrange(1, r), v) for v in rng.sample(used, k)]
    a = [[(rng.randrange(1, r), 0)]] + [rand_row(3) for _ in range(nc - 1)]
    b = [rand_row(2) for _ in range(nc)]
    c = [[(1, 0)] + rand_row(2) for _ in range(nc)]
    return (a, b, c), ni, nw


def circuits(curve):
    """(name, (A, B, C), ni, nw): n = 4 .. 64"""
    r = field(curve)[0]
    pc = P.CURVES["bls12_377" if curve == "bw6_761" else curve]
    out = []
    for name, cs in (("silly", P.silly_circuit(pc, 3, 5)), ("synthetic 2^5", P.synthetic_circuit(pc, 30, seed=41, num_inputs=1)),
                     ("synthetic 2^6", P.synthetic_circuit(pc, 60, seed=42, num_inputs=3))):
        out.append((name, (cs.a, cs.b, cs.c), cs.num_instance, cs.num_witness))
    out.append(("instance-heavy", *mixed_circuit(r, 9, 6, 5, 43)))      # n = 16, 9 instance rows
    out.append(("mixed 2^3", *mixed_circuit(r, 2, 9, 6, 44)))
    return out


def ids(curve):
    return [c[0] for c in circuits(curve)]


@pytest.mark.parametrize("qap", ["libsnark", "circom"])
@pytest.mark.parametrize("curve", CURVES4)
def test_transcript_side_equals_key_sums(curve, qap):
    """the identities of DESIGN.md section 16: each transcript-side combination equals sum_j rho^j times the exponents of
    the key g16_setup(alpha, beta, 1, 1, tau), for several rho"""
    r, root = field(curve)
    for name, rows, ni, nw in circuits(curve):
        for rho in (RHO, 1, r - 1):
            got = transcript_sides(r, root, rows, ni, nw, TAU, ALPHA, BETA, rho, qap == "circom")
            assert got == transcript_sums(r, root, rows, ni, nw, TAU, ALPHA, BETA, rho, qap == "circom"), (name, rho)


@pytest.mark.parametrize("curve", CURVES4)
def test_key_exponents_match_the_references(curve):
    """pk_verify_ref.key_exponents is the setup: pyref (LibsnarkReduction), qap_circom_ref's definition of the
    CircomReduction H query (a size-2n inverse transform), bw6_ref on BW6-761"""
    r, root = field(curve)
    di = pow(DELTA, -1, r)
    for name, rows, ni, nw in circuits(curve):
        k = key_exponents(r, root, rows, ni, nw, ALPHA, BETA, GAMMA, DELTA, TAU, False)
        kc = key_exponents(r, root, rows, ni, nw, ALPHA, BETA, GAMMA, DELTA, TAU, True)
        n, L = domain(rows, ni)
        if curve == "bw6_761":
            e = B.query_exponents(list(rows), ni, ni + nw, ALPHA, BETA, DELTA, TAU)
            want = dict(a=e["a"], b=e["b"], l=e["l"], h=e["h"])
            circom_h = [x for x in B.ntt([di * pow(TAU, i, r) % r for i in range(2 * n - 1)] + [0], inverse=True)[1::2]]
        else:
            cs = P.R1CS(P.CURVES[curve], ni, nw, list(rows[0]), list(rows[1]), list(rows[2]))
            e = P.generate_parameters(cs, ALPHA, BETA, GAMMA, DELTA, TAU, scalars_only=True)
            want = dict(a=e["a"], b=e["b"], l=e["l"], h=e["h"])
            assert k["gamma_abc_g1"] == e["gamma_abc"], name
            circom_h = Q.h_query_scalars(P.Domain(P.CURVES[curve], n), TAU, di)
        assert (k["a_query"], k["b_g1_query"], k["b_g2_query"]) == (want["a"], want["b"], want["b"]), name
        assert (k["l_query"], k["h_query"]) == (want["l"], want["h"]), name
        assert kc["h_query"] == circom_h, name
        assert {m: v for m, v in kc.items() if m != "h_query"} == {m: v for m, v in k.items() if m != "h_query"}, name


def check(curve, qap, rows, ni, nw, key_rows=None, key_tau=TAU, key_qap=None, **kw):
    """verdict of the call on a key of (key_rows, key_tau, key_qap) against T(TAU, ALPHA, BETA) and the circuit rows"""
    r, root = field(curve)
    k = key_exponents(r, root, key_rows or rows, ni, nw, ALPHA, BETA, GAMMA, DELTA, key_tau, (key_qap or qap) == "circom")
    ts = transcript_sides(r, root, rows, ni, nw, TAU, ALPHA, BETA, RHO, qap == "circom")
    return k, ts, verdict(k, (TAU, ALPHA, BETA), ts, RHO, r, ni, **kw)


@pytest.mark.parametrize("qap", ["libsnark", "circom"])
@pytest.mark.parametrize("curve", CURVES4)
def test_honest_key_passes(curve, qap):
    r, root = field(curve)
    for name, rows, ni, nw in circuits(curve):
        k, ts, (bad, p, q) = check(curve, qap, rows, ni, nw)
        assert bad is None and failing(p, q, r) == set(), name
        # the uncontributed key of a ceremony: gamma = delta = 1, refused unless accepted explicitly
        k1 = key_exponents(r, root, rows, ni, nw, ALPHA, BETA, 1, 1, TAU, qap == "circom")
        assert verdict(k1, (TAU, ALPHA, BETA), ts, RHO, r, ni)[0] == "gamma_g2"
        bad, p, q = verdict(k1, (TAU, ALPHA, BETA), ts, RHO, r, ni, uncontributed=True)
        assert bad is None and failing(p, q, r) == set(), name
        assert key_sums(k1, RHO, r, ni) == ts   # the transcript's own key has the transcript's sums


def outcome(v, r):
    bad, p, q = v
    return bad if bad is not None else failing(p, q, r)


@pytest.mark.parametrize("qap", ["libsnark", "circom"])
@pytest.mark.parametrize("curve", CURVES4)
def test_tampering(curve, qap):
    r, _ = field(curve)
    for name, rows, ni, nw in circuits(curve):
        k, ts, _ = check(curve, qap, rows, ni, nw)
        for what, t, want in tamperings(k, r):
            assert outcome(verdict(t, (TAU, ALPHA, BETA), ts, RHO, r, ni), r) == want, (name, what)
        # a key for another tau, a key of the other reduction, keys of circuits with one coefficient changed
        assert outcome(check(curve, qap, rows, ni, nw, key_tau=TAU2)[2], r) == "a_query", name
        other = "circom" if qap == "libsnark" else "libsnark"
        assert outcome(check(curve, qap, rows, ni, nw, key_qap=other)[2], r) == {1}, name
        for which in range(4):
            try:
                edited, want = edited_rows(rows, which, ni)
            except ValueError:   # no instance entry in C
                continue
            assert outcome(check(curve, qap, rows, ni, nw, key_rows=edited)[2], r) == want, (name, which)


def test_expected_table_covers_every_member():
    assert set(EXPECTED) == {"a_query", "b_g1_query", "b_g2_query", "h_query", "l_query", "gamma_abc_g1", "alpha_g1",
                             "beta_g1", "beta_g2", "delta_g1", "delta_g2", "gamma_g2"}
