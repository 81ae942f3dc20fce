"""Reference of the transcript check (g16_srs_verify_pairs) in the exponent, shared by the CPU and GPU tiers.

A transcript is described by the discrete logs of its points: e["tau_g1"][i] is the scalar k with tau_g1[i] = [k]g1, and
so on (beta_g2 is one int).  pair_exponents restates the library's formulas -- S = sum rho^i X_i, lo = S - rho^(N-1)
X_(N-1), hi = rho^-1 (S - X_0) -- on those scalars, so that the ten G1 and ten G2 output points are [p_j]g1 and [q_j]g2, and
equation k holds iff p_2k q_2k = p_2k+1 q_2k+1 mod r (bilinearity)."""

VECS = ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1")
MEMBERS = VECS + ("beta_g2",)


def transcript_exponents(r, lens, tau, alpha, beta) -> dict:
    """T(tau, alpha, beta) with lens = (tau_g1, tau_g2, alpha_tau_g1, beta_tau_g1) points"""
    pw = lambda c, n: [c * pow(tau, i, r) % r for i in range(n)]
    return dict(tau_g1=pw(1, lens[0]), tau_g2=pw(1, lens[1]), alpha_tau_g1=pw(alpha, lens[2]), beta_tau_g1=pw(beta, lens[3]),
                beta_g2=beta % r)


def s_lo_hi(xs, rho, r):
    """(S, lo, hi) of one member by the S-based formulas the library uses"""
    n = len(xs)
    s = sum(pow(rho, i, r) * x for i, x in enumerate(xs)) % r
    lo = (s - pow(rho, n - 1, r) * xs[-1]) % r
    hi = pow(rho, -1, r) * (s - xs[0]) % r
    return s, lo, hi


def pair_exponents(e: dict, rho: int, r: int):
    """(p, q): the exponents of P_0, P'_0, .., P_4, P'_4 over g1 and of Q_0, Q'_0, .., Q_4, Q'_4 over g2"""
    _, lo1, hi1 = s_lo_hi(e["tau_g1"], rho, r)
    _, lo2, hi2 = s_lo_hi(e["tau_g2"], rho, r)
    _, loa, hia = s_lo_hi(e["alpha_tau_g1"], rho, r)
    _, lob, hib = s_lo_hi(e["beta_tau_g1"], rho, r)
    t1, t2 = e["tau_g1"][1], e["tau_g2"][1]
    p = [hi1, lo1, 1, t1, hia, loa, hib, lob, e["beta_tau_g1"][0], 1]
    q = [1, t2, hi2, lo2, 1, t2, 1, t2, 1, e["beta_g2"]]
    return p, q


def failing(p, q, r) -> set:
    """the equations that do not hold"""
    return {k for k in range(5) if p[2 * k] * q[2 * k] % r != p[2 * k + 1] * q[2 * k + 1] % r}


def expected_failures(member: str, idx: int) -> set:
    """The equations a wrong point at `idx` of `member` breaks: its own member's, plus those that read the point itself
    (tau_g1[1] in equation 1, tau_g2[1] in equations 0, 2 and 3, beta_tau_g1[0] in equation 4)."""
    own = {MEMBERS.index(member)}
    if member == "tau_g1" and idx == 1:
        return own | {1}
    if member == "tau_g2" and idx == 1:
        return own | {0, 2, 3}
    if member == "beta_tau_g1" and idx == 0:
        return own | {4}
    return own


def copy_e(e):
    return {k: (list(v) if k != "beta_g2" else v) for k, v in e.items()}


def tamperings(e: dict, r: int, tau2: int, alpha: int, beta: int):
    """(name, tampered exponents, equations expected to fail) for the cases every tier checks.  tau2 is another tau."""
    out = []
    n1, n2 = len(e["tau_g1"]), len(e["tau_g2"])
    t = copy_e(e)
    t["tau_g1"][2], t["tau_g1"][3] = t["tau_g1"][3], t["tau_g1"][2]
    out.append(("tau_g1 points 2 and 3 swapped", t, {0}))
    t = copy_e(e)
    t["tau_g2"][n2 // 2] = pow(tau2, n2 // 2, r)
    out.append(("tau_g2 point of another tau", t, {1}))
    t = copy_e(e)
    t["alpha_tau_g1"] = [alpha * pow(tau2, i, r) % r for i in range(len(e["alpha_tau_g1"]))]
    out.append(("alpha_tau_g1 chain of another ratio", t, {2}))
    for m in VECS:
        t = copy_e(e)
        t[m][-1] = t[m][-1] * 3 % r
        out.append((f"last point of {m} changed", t, expected_failures(m, len(t[m]) - 1)))
    t = copy_e(e)
    t["beta_g2"] = beta * 5 % r
    out.append(("beta_g2 of another beta", t, {4}))
    t = copy_e(e)
    t["tau_g2"] = [pow(tau2, i, r) for i in range(n2)]
    out.append(("tau_g2 of another tau than tau_g1", t, {0, 1, 2, 3}))
    for m, idx in (("tau_g1", 1), ("tau_g2", 1), ("beta_tau_g1", 0), ("tau_g1", n1 // 2)):
        t = copy_e(e)
        t[m][idx] = t[m][idx] * 7 % r
        out.append((f"{m}[{idx}] changed", t, expected_failures(m, idx)))
    return out


def geometric(x, n, r):
    """sum_{i<n} x^i mod r"""
    if n <= 0:
        return 0
    if x % r == 1:
        return n % r
    return (pow(x, n, r) - 1) * pow(x - 1, -1, r) % r


def closed_exponents(r, lens, tau, alpha, beta, rho):
    """pair_exponents of T(tau, alpha, beta) in closed form, for transcripts too long to list: for a member c tau^i of N
    points, lo = c sum_{i<N-1} (rho tau)^i and hi = tau lo."""
    lo = lambda c, n: c * geometric(rho * tau, n - 1, r) % r
    lo1, lo2, loa, lob = lo(1, lens[0]), lo(1, lens[1]), lo(alpha, lens[2]), lo(beta, lens[3])
    p = [tau * lo1 % r, lo1, 1, tau % r, tau * loa % r, loa, tau * lob % r, lob, beta % r, 1]
    q = [1, tau % r, tau * lo2 % r, lo2, 1, tau % r, 1, tau % r, 1, beta % r]
    return p, q
