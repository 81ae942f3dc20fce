"""CPU tier of the transcript check (g16_srs_verify_pairs), with big integers and pyref's pairing: transcripts of 7 to 33
points are built as group elements, S, lo and hi are formed by the S-based formulas exactly as the library forms them, and
the five equations are evaluated with pyref's pairing.  Honest transcripts pass every equation; each tampering breaks
exactly the equations srs_verify_ref.expected_failures names, and the pairing agrees with the check in the exponent."""
import pytest

import pyref as P
from groth16_b200.params import GENERATORS
from srs_verify_ref import (MEMBERS, VECS, closed_exponents, failing, pair_exponents, tamperings,
                             transcript_exponents)

TAU, ALPHA, BETA, TAU2 = 0x1234567890ABCDEF1234567, 0x2222222222222222222223, 0x3333333333333333333335, 0x777777777779ABC
RHO = 0x5EED5EED5EED5EED5EED5EED5EED5EED1
SIZES = {"bn254": (33, 17, 17, 17), "bls12_381": (15, 8, 8, 8), "bls12_377": (7, 4, 4, 4)}


class Group:
    """pyref's groups over the library's generators"""

    def __init__(self, curve):
        self.cx = P.ctx(P.CURVES[curve])
        self.r = P.CURVES[curve].r
        self.g1, self.g2 = GENERATORS[curve]["g1"], GENERATORS[curve]["g2"]

    def grp(self, m):
        return self.cx.G2 if m in ("tau_g2", "beta_g2") else self.cx.G1

    def points(self, e):
        out = {}
        for m in MEMBERS:
            G, g = self.grp(m), (self.g2 if m in ("tau_g2", "beta_g2") else self.g1)
            out[m] = G.mul(g, e[m]) if m == "beta_g2" else [G.mul(g, k) for k in e[m]]
        return out

    def msm(self, G, pts, ks):
        acc = None
        for p, k in zip(pts, ks):
            acc = G.add(acc, G.mul(p, k % self.r))
        return acc

    def s_lo_hi(self, G, xs, rho):
        """the library's formulas on points: S = sum rho^i X_i, lo = S - rho^(N-1) X_(N-1), hi = rho^-1 (S - X_0)"""
        r, n = self.r, len(xs)
        s = self.msm(G, xs, [pow(rho, i, r) for i in range(n)])
        lo = G.add(s, G.neg(G.mul(xs[-1], pow(rho, n - 1, r))))
        hi = G.mul(G.add(s, G.neg(xs[0])), pow(rho, -1, r))
        return s, lo, hi

    def pairs(self, pts, rho):
        G1, G2 = self.cx.G1, self.cx.G2
        _, lo1, hi1 = self.s_lo_hi(G1, pts["tau_g1"], rho)
        _, lo2, hi2 = self.s_lo_hi(G2, pts["tau_g2"], rho)
        _, loa, hia = self.s_lo_hi(G1, pts["alpha_tau_g1"], rho)
        _, lob, hib = self.s_lo_hi(G1, pts["beta_tau_g1"], rho)
        t1, t2 = pts["tau_g1"][1], pts["tau_g2"][1]
        ps = [hi1, lo1, self.g1, t1, hia, loa, hib, lob, pts["beta_tau_g1"][0], self.g1]
        qs = [self.g2, t2, hi2, lo2, self.g2, t2, self.g2, t2, self.g2, pts["beta_g2"]]
        return ps, qs

    def pairing_failures(self, ps, qs):
        G1 = self.cx.G1
        return {k for k in range(5)
                if not self.cx.pairing_product_is_one([(ps[2 * k], qs[2 * k]), (G1.neg(ps[2 * k + 1]), qs[2 * k + 1])])}


@pytest.mark.parametrize("curve", list(SIZES))
def test_lo_hi_are_the_direct_sums(curve):
    g = Group(curve)
    r = g.r
    e = transcript_exponents(r, SIZES[curve], TAU, ALPHA, BETA)
    e["alpha_tau_g1"][2] = 12345   # not a geometric member: the identities hold for any points
    pts = g.points(e)
    for m in VECS:
        G, xs = g.grp(m), pts[m]
        s, lo, hi = g.s_lo_hi(G, xs, RHO)
        n = len(xs)
        assert lo == g.msm(G, xs[:-1], [pow(RHO, i, r) for i in range(n - 1)]), m
        assert hi == g.msm(G, xs[1:], [pow(RHO, i, r) for i in range(n - 1)]), m
        assert s == g.msm(G, xs, [pow(RHO, i, r) for i in range(n)]), m
    # one point: lo = hi = the identity
    _, lo, hi = g.s_lo_hi(g.cx.G1, pts["beta_tau_g1"][:1], RHO)
    assert lo is None and hi is None


@pytest.mark.parametrize("curve", list(SIZES))
def test_points_match_the_exponents(curve):
    """the group formulas and pair_exponents (the GPU tier's closed form) name the same twenty points"""
    g = Group(curve)
    e = transcript_exponents(g.r, SIZES[curve], TAU, ALPHA, BETA)
    ps, qs = g.pairs(g.points(e), RHO)
    p, q = pair_exponents(e, RHO, g.r)
    assert ps == [g.cx.G1.mul(g.g1, k) for k in p]
    assert qs == [g.cx.G2.mul(g.g2, k) for k in q]


@pytest.mark.parametrize("curve", list(SIZES))
def test_honest_transcript_passes(curve):
    g = Group(curve)
    e = transcript_exponents(g.r, SIZES[curve], TAU, ALPHA, BETA)
    for rho in (RHO, 2):
        ps, qs = g.pairs(g.points(e), rho)
        assert g.pairing_failures(ps, qs) == set()
        assert failing(*pair_exponents(e, rho, g.r), g.r) == set()


@pytest.mark.parametrize("curve", list(SIZES))
def test_tampering_fails_its_equations(curve):
    g = Group(curve)
    e = transcript_exponents(g.r, SIZES[curve], TAU, ALPHA, BETA)
    for name, t, want in tamperings(e, g.r, TAU2, ALPHA, BETA):
        assert failing(*pair_exponents(t, RHO, g.r), g.r) == want, name
        ps, qs = g.pairs(g.points(t), RHO)
        assert g.pairing_failures(ps, qs) == want, name


@pytest.mark.parametrize("curve", list(SIZES))
def test_closed_form(curve):
    """closed_exponents (the GPU tier's reference for long transcripts) agrees with pair_exponents, ragged lengths too"""
    r = P.CURVES[curve].r
    for lens in (SIZES[curve], (2, 2, 1, 1), (1000, 3, 999, 7)):
        for rho in (RHO, 1, r - 1):
            e = transcript_exponents(r, lens, TAU, ALPHA, BETA)
            assert closed_exponents(r, lens, TAU, ALPHA, BETA, rho) == pair_exponents(e, rho, r), (lens, rho)
