"""CPU tier of the phase-2 ceremony calls, with big integers and pyref's pairing: a delta contribution to
g16_setup(alpha, beta, gamma, delta0, tau) restated in the exponent is g16_setup(.., delta0 delta, ..) on all four scalar
fields; honest chains of contribution records pass every equation of g16_contribution_chain_pairs in the exponent on all
four curves and by pairing on BN254 and BLS12-381; each tampering breaks exactly the equations, or causes exactly the
refusal, contribution_chain_ref names -- in phase 2 and on the three phase-1 chains."""
import pytest

import pyref as P
from contribution_chain_ref import chain, contribute_key, failing, outcome, phase1_chains, tamperings, verdict
from groth16_b200.params import GENERATORS
from pk_verify_ref import key_exponents
from test_pk_verify_cpu import circuits, field

TAU, ALPHA, BETA, GAMMA, DELTA = (0x1234567890ABCDEF1234567, 0x2222222222222222222223, 0x3333333333333333333335,
                                  0x6666666666666666666661, 0x4444444444444444444447)
XS = (0x4444444444444444444449, 0x5555555555555555555559, 0x77777777777777777777771, 0x1357913579135791357913,
      0x2468024680246802468021)
CURVES4 = ["bls12_381", "bn254", "bls12_377", "bw6_761"]
PAIRING = ["bn254", "bls12_381"]


@pytest.mark.parametrize("curve", CURVES4)
@pytest.mark.parametrize("circom", [False, True], ids=["libsnark", "circom"])
def test_contribution_is_setup_of_the_product(curve, circom):
    r, root = field(curve)
    for name, rows, ni, nw in circuits(curve)[:3]:
        k = key_exponents(r, root, rows, ni, nw, ALPHA, BETA, GAMMA, DELTA, TAU, circom)
        got = k
        prod = DELTA
        for x in XS[:3]:
            got = contribute_key(got, x, r)
            prod = prod * x % r
            assert got == key_exponents(r, root, rows, ni, nw, ALPHA, BETA, GAMMA, prod, TAU, circom), (name, x)


@pytest.mark.parametrize("curve", CURVES4)
def test_honest_chains_pass_in_the_exponent(curve):
    r = field(curve)[0]
    for n in range(1, 6):
        end, recs = chain(1, XS[:n], r)
        prod = 1
        for x in XS[:n]:
            prod = prod * x % r
        assert end == prod
        v = verdict(1, end, recs, r)
        assert v[0] == "pairs" and len(v[1]) == len(v[2]) == 4 * n
        assert failing(v[1], v[2], r) == set()


@pytest.mark.parametrize("curve", CURVES4)
def test_tampering_breaks_exactly_its_equations(curve):
    r = field(curve)[0]
    for n in (3, 5):
        for name, start, end, recs, want in tamperings(TAU, XS[:n], r, other_start=ALPHA):
            assert outcome(start, end, recs, r) == want, (n, name)


@pytest.mark.parametrize("curve", CURVES4)
def test_phase1_chains(curve):
    """three contribute_srs-style contributions (tau_k, alpha_k, beta_k) to T(TAU, ALPHA, BETA): each of the three running
    points ends at the transcript's own point of the product secrets, and every tampering of each chain is caught"""
    r = field(curve)[0]
    contribs = [(XS[0], XS[1], XS[2]), (XS[3], XS[4], XS[0]), (XS[1], XS[3], XS[2])]
    chains = phase1_chains(TAU, ALPHA, BETA, contribs, r)
    want_end = [TAU, ALPHA, BETA]
    for j, (start, end, recs) in enumerate(chains.values()):
        for c in contribs:
            want_end[j] = want_end[j] * c[j] % r
        assert end == want_end[j]
        assert outcome(start, end, recs, r) == set()
        xs = [c[j] for c in contribs]
        for name, s2, e2, t, want in tamperings(start, xs, r, other_start=start + 1):
            assert outcome(s2, e2, t, r) == want, name


class Points:
    """pyref's groups over the library's generators: records and equations as points"""

    def __init__(self, curve):
        self.cx = P.ctx(P.CURVES[curve])
        self.r = P.CURVES[curve].r
        self.g1, self.g2 = GENERATORS[curve]["g1"], GENERATORS[curve]["g2"]

    def failures(self, p, q):
        """the equations whose pairings differ, the points formed from the exponents p, q"""
        G1, G2 = self.cx.G1, self.cx.G2
        ps, qs = [G1.mul(self.g1, k) for k in p], [G2.mul(self.g2, k) for k in q]
        return {k for k in range(len(p) // 2)
                if not self.cx.pairing_product_is_one([(ps[2 * k], qs[2 * k]), (G1.neg(ps[2 * k + 1]), qs[2 * k + 1])])}


@pytest.mark.parametrize("curve", PAIRING)
def test_honest_chains_pass_by_pairing(curve):
    g = Points(curve)
    for n in range(1, 6):
        end, recs = chain(TAU, XS[:n], g.r)
        _, p, q = verdict(TAU, end, recs, g.r)
        assert g.failures(p, q) == set(), n


@pytest.mark.parametrize("curve", PAIRING)
def test_tampering_by_pairing(curve):
    """the pairing agrees with the exponent on every tampering of a chain of three that writes equations"""
    g = Points(curve)
    for name, start, end, recs, want in tamperings(TAU, XS[:3], g.r, other_start=ALPHA):
        if isinstance(want, str):
            continue
        _, p, q = verdict(start, end, recs, g.r)
        assert g.failures(p, q) == want, name
