"""CPU tier of the transcript setup (csrc/srs.cuh, Engine::setup_from_srs / setup_contribute): the derivation restated with
big integers over oracle/pyref.py points (tests/bw6_ref.py for BW6-761), step for step as the kernels compute it:
radix-2 group inverse transforms of [tau^i]G1, [tau^i]G2, [alpha tau^i]G1, [beta tau^i]G1, times n^-1; the sparse sums of
the queries; the H query (differences under LibsnarkReduction, the odd-entry identity under CircomReduction); then delta
contributions.  On all four curves, both reductions and circuits with n = 4 .. 32, the key must equal the reference setup
with gamma = 1 and delta = prod delta_k (pyref / qap_circom_ref; bw6_ref's Lagrange coefficients and size-2n transform), and
a longer transcript must give the same key."""
import pytest

import bw6_ref as B
import pyref as P
import qap_circom_ref as Q
from groth16_b200.params import GENERATORS

TAU, ALPHA, BETA = 0x1234567890ABCDEF1234567, 0x2222222222222222222223, 0x3333333333333333333335
DELTAS = (0x4444444444444444444447, 0x5555555555555555555559)
CURVES4 = ["bls12_381", "bn254", "bls12_377", "bw6_761"]


class Bw6Group:
    """bw6_ref's affine arithmetic behind pyref's Group interface (the a = 0 addition law does not depend on b)"""
    add = staticmethod(B.add)
    neg = staticmethod(B.neg)

    @staticmethod
    def mul(p, k):
        return B.mul_proj(k % B.R, p)


def groups(curve):
    """(r, G1, G2, g1, g2, two-adic root of a size-2^L domain)"""
    if curve == "bw6_761":
        G = GENERATORS[curve]
        return B.R, Bw6Group, Bw6Group, G["g1"], G["g2"], B.domain_root
    c = P.CURVES[curve]
    cx = P.ctx(c)
    return c.r, cx.G1, cx.G2, cx.g1_gen(), cx.g2_gen(), lambda L: P.Domain(c, 1 << L).omega


def circuit(curve, log_n):
    """MySillyCircuit at log_n = 2, otherwise pyref's synthetic circuit with one public input filling n = 2^log_n; BW6-761
    takes the rows of BLS12-377's (its r is BLS12-377's q, so the coefficients are canonical there too)"""
    c = P.CURVES["bls12_377" if curve == "bw6_761" else curve]
    if log_n == 2:
        return P.silly_circuit(c, 3, 5)
    return P.synthetic_circuit(c, (1 << log_n) - 2, seed=40 + log_n, num_inputs=1)


def group_ifft(G, pts, w, r):
    """unscaled inverse transform out[j] = sum_i w^(-ij) pts[i]: bit reversal, then radix-2 decimation-in-time stages with
    (P, Q) -> (P + w^-k Q, P - w^-k Q), k = 0 without a product -- srs_bitrev_kernel and srs_butterfly_kernel"""
    n = len(pts)
    L = n.bit_length() - 1
    p = [pts[int(format(i, f"0{L}b")[::-1], 2) if L else 0] for i in range(n)]
    w_inv = pow(w, -1, r)
    h = 1
    while h < n:
        for t in range(n // 2):
            k = t % h
            i0 = (t - k) * 2 + k
            i1 = i0 + h
            q = p[i1] if k == 0 else G.mul(p[i1], pow(w_inv, k * (n // (2 * h)), r))
            p[i0], p[i1] = G.add(p[i0], q), G.add(p[i0], G.neg(q))
        h *= 2
    return p


def derive(curve, cs, srs, deltas, circom):
    r, G1, G2, _, _, root = groups(curve)
    nc, ni = cs.num_constraints, cs.num_instance
    nv = ni + cs.num_witness
    L = max(nc + ni - 1, 0).bit_length()
    n = 1 << L
    w = root(L)
    n_inv = pow(n, -1, r)
    tau_g1, tau_g2, atau, btau, beta_g2 = srs
    lag = lambda G, pts: [G.mul(p, n_inv) for p in group_ifft(G, pts[:n], w, r)]
    L1, L2, aL, bL = lag(G1, tau_g1), lag(G2, tau_g2), lag(G1, atau), lag(G1, btau)

    def ssum(G, mat, src):   # CSC sum: coefficient x point, skipped when the coefficient is One
        out = [None] * nv
        for i, row in enumerate(mat):
            for cf, j in row:
                out[j] = G.add(out[j], src[i] if cf % r == 1 else G.mul(src[i], cf % r))
        return out
    a = ssum(G1, cs.a, L1)
    for j in range(ni):
        a[j] = G1.add(a[j], L1[nc + j])
    b1, b2 = ssum(G1, cs.b, L1), ssum(G2, cs.b, L2)
    t = [G1.add(G1.add(x, y), z) for x, y, z in zip(ssum(G1, cs.a, bL), ssum(G1, cs.b, aL), ssum(G1, cs.c, L1))]
    for j in range(ni):
        t[j] = G1.add(t[j], bL[nc + j])
    if not circom:
        h = [G1.add(tau_g1[n + i], G1.neg(tau_g1[i])) for i in range(n - 1)]
    else:   # 1/(2n) x size-n transform of omega_2n^-i (v_i - v_(i+n)), v_(2n-1) = O
        w2_inv = pow(root(L + 1), -1, r)
        v = tau_g1[:2 * n - 1] + [None]
        d = [G1.mul(G1.add(v[i], G1.neg(v[i + n])), pow(w2_inv, i, r) * pow(2 * n, -1, r) % r) for i in range(n)]
        h = group_ifft(G1, d, w, r)
    key = dict(a=a, b1=b1, b2=b2, gamma_abc=t[:ni], l=t[ni:], h=h, delta_g1=tau_g1[0], delta_g2=tau_g2[0],
               alpha_g1=atau[0], beta_g1=btau[0], beta_g2=beta_g2, gamma_g2=tau_g2[0])
    for dk in deltas:   # g16_setup_contribute
        di = pow(dk, -1, r)
        key.update(delta_g1=G1.mul(key["delta_g1"], dk), delta_g2=G2.mul(key["delta_g2"], dk),
                   l=[G1.mul(p, di) for p in key["l"]], h=[G1.mul(p, di) for p in key["h"]])
    return key


def transcript(curve, n, extra=0):
    r, G1, G2, g1, g2, _ = groups(curve)
    t1 = [G1.mul(g1, pow(TAU, i, r)) for i in range(2 * n - 1 + extra)]
    t2 = [G2.mul(g2, pow(TAU, i, r)) for i in range(n + extra)]
    return t1, t2, [G1.mul(p, ALPHA) for p in t1[:n + extra]], [G1.mul(p, BETA) for p in t1[:n + extra]], G2.mul(g2, BETA)


def reference(curve, cs, delta, circom):
    """the setup with gamma = 1 (pyref / qap_circom_ref; for BW6-761 from bw6_ref's Lagrange coefficients)"""
    if curve != "bw6_761":
        pk = Q.generate_parameters(cs, ALPHA, BETA, 1, delta, TAU, qap="circom" if circom else "libsnark")
        return dict(a=pk.a_query, b1=pk.b_g1_query, b2=pk.b_g2_query, gamma_abc=pk.vk.gamma_abc_g1, l=pk.l_query,
                    h=pk.h_query, delta_g1=pk.delta_g1, delta_g2=pk.vk.delta_g2, alpha_g1=pk.vk.alpha_g1,
                    beta_g1=pk.beta_g1, beta_g2=pk.vk.beta_g2, gamma_g2=pk.vk.gamma_g2)
    r, G1, G2, g1, g2, _ = groups(curve)
    nc, ni = cs.num_constraints, cs.num_instance
    nv = ni + cs.num_witness
    n, L = B.domain_size([cs.a, cs.b, cs.c], ni)
    lag = B.lagrange_at(TAU, L)
    q = [[0] * nv for _ in range(3)]
    for m, mat in enumerate((cs.a, cs.b, cs.c)):
        for i, row in enumerate(mat):
            for cf, var in row:
                q[m][var] = (q[m][var] + lag[i] * cf) % r
    for i in range(ni):
        q[0][i] = (q[0][i] + lag[nc + i]) % r
    di = pow(delta, -1, r)
    t = [(BETA * q[0][i] + ALPHA * q[1][i] + q[2][i]) % r for i in range(nv)]
    if circom:   # the odd entries of the size-2n inverse transform of delta^-1 tau^i, i < 2n - 1
        hs = B.ntt([di * pow(TAU, i, r) % r for i in range(2 * n - 1)] + [0], inverse=True)[1::2]
    else:
        hs = [(pow(TAU, n, r) - 1) * di * pow(TAU, i, r) % r for i in range(n - 1)]
    m1 = lambda e: G1.mul(g1, e)
    return dict(a=[m1(e) for e in q[0]], b1=[m1(e) for e in q[1]], b2=[G2.mul(g2, e) for e in q[1]],
                gamma_abc=[m1(e) for e in t[:ni]], l=[m1(e * di % r) for e in t[ni:]], h=[m1(e) for e in hs],
                delta_g1=m1(delta), delta_g2=G2.mul(g2, delta), alpha_g1=m1(ALPHA), beta_g1=m1(BETA),
                beta_g2=G2.mul(g2, BETA), gamma_g2=g2)


@pytest.mark.parametrize("log_n", [2, 3, 5])
@pytest.mark.parametrize("qap", ["libsnark", "circom"])
@pytest.mark.parametrize("curve", CURVES4)
def test_derived_key_equals_setup(curve, qap, log_n):
    r = groups(curve)[0]
    cs = circuit(curve, log_n)
    n = 1 << max(cs.num_constraints + cs.num_instance - 1, 0).bit_length()
    circom = qap == "circom"
    got = derive(curve, cs, transcript(curve, n), DELTAS, circom)
    want = reference(curve, cs, DELTAS[0] * DELTAS[1] % r, circom)
    for k in want:
        assert got[k] == want[k], k
    if log_n == 2:   # a longer transcript (ceremonies are sized for the largest circuit) gives the same key
        assert derive(curve, cs, transcript(curve, n, extra=3 * n), DELTAS, circom) == got


@pytest.mark.parametrize("log_n", [2, 3, 4, 5])
@pytest.mark.parametrize("curve", ["bls12_381", "bn254", "bls12_377"])
def test_circom_odd_entry_identity(curve, log_n):
    """odd entries of the size-2n inverse transform of v_i = tau^i (i < 2n - 1, v_(2n-1) = 0) equal 1/(2n) times the size-n
    transform of omega_2n^-i (v_i - v_(i+n))"""
    c = P.CURVES[curve]
    r = c.r
    n = 1 << log_n
    w2 = P.Domain(c, 2 * n).omega
    wn = P.Domain(c, n).omega
    v = [pow(TAU, i, r) for i in range(2 * n - 1)] + [0]
    big = [sum(pow(w2, -i * k, r) * v[i] for i in range(2 * n)) * pow(2 * n, -1, r) % r for k in range(2 * n)]
    d = [pow(w2, -i, r) * (v[i] - v[i + n]) for i in range(n)]
    small = [sum(pow(wn, -i * j, r) * d[i] for i in range(n)) * pow(2 * n, -1, r) % r for j in range(n)]
    assert big[1::2] == small
