"""Reference of the key check (g16_pk_verify_pairs) in the exponent, shared by the CPU and GPU tiers.

A key is described by the discrete logs of its points over g1 = tau_g1[0] and g2 = tau_g2[0]: a dict from member name to a
list of ints (the vectors) or an int (the single points).  A transcript T(tau, alpha, beta) by its three secrets.
  key_exponents      the setup written out directly: Lagrange coefficients at tau, the H query of either reduction
  transcript_sides   S_X(T) by the field transforms the library runs (row evaluations of z = rho^j, inverse transforms,
                     the H weights), evaluated at tau: what the MSMs over the transcript compute, in the exponent
  transcript_sums    S_X(T) by the identity the CPU tier proves: the sums of the transcript's own key g16_setup(alpha, beta,
                     1, 1, tau) -- O(n) where transcript_sides is O(n log n), for the GPU tier's large circuits
  verdict            what the call decides: the member it refuses, or the exponents p, q of its eight G1 and eight G2
                     output points; equation k holds iff p_2k q_2k = p_2k+1 q_2k+1 mod r (bilinearity)
  tamperings         the cases every tier checks, each with the refusal or the broken equations it must cause."""

EQUATIONS = ("delta", "h_query", "l_query", "gamma_abc_g1")
VECTORS = ("a_query", "b_g1_query", "b_g2_query", "h_query", "l_query", "gamma_abc_g1")
POINTS = ("alpha_g1", "beta_g1", "delta_g1", "beta_g2", "gamma_g2", "delta_g2")
G2_MEMBERS = ("b_g2_query", "beta_g2", "gamma_g2", "delta_g2")


def batch_inv(xs, r):
    pref, acc = [], 1
    for x in xs:
        pref.append(acc)
        acc = acc * x % r
    inv = pow(acc, -1, r)
    out = [0] * len(xs)
    for i in range(len(xs) - 1, -1, -1):
        out[i] = inv * pref[i] % r
        inv = inv * xs[i] % r
    return out


def powers(x, n, r):
    """x^i, i < n"""
    out, p = [], 1
    for _ in range(n):
        out.append(p)
        p = p * x % r
    return out


def transform(xs, w, r):
    """out[k] = sum_i xs[i] w^(ik) over len(xs) = 2^L points, radix 2"""
    n = len(xs)
    if n == 1:
        return [xs[0] % r]
    ev, od = transform(xs[0::2], w * w % r, r), transform(xs[1::2], w * w % r, r)
    out, t = [0] * n, 1
    for k in range(n // 2):
        x = od[k] * t % r
        out[k], out[k + n // 2] = (ev[k] + x) % r, (ev[k] - x) % r
        t = t * w % r
    return out


def domain(rows, ni):
    """(n, L): the domain of nc + ni points"""
    L = max(len(rows[0]) + ni - 1, 0).bit_length()
    return 1 << L, L


def row_evals(rows, ni, z, n, r):
    """A z, B z, C z over the domain: the constraint rows, then the instance rows a[nc + j] = z_j, then zeros"""
    nc = len(rows[0])
    out = []
    for m, mat in enumerate(rows):
        ev = [sum(cf * z[v] for cf, v in row) % r for row in mat] + [0] * (n - nc)
        if m == 0:
            for j in range(ni):
                ev[nc + j] = z[j] % r
        out.append(ev)
    return out


def key_exponents(r, root, rows, ni, nw, alpha, beta, gamma, delta, tau, circom):
    """g16_setup(alpha, beta, gamma, delta, tau) of the circuit `rows` = (A, B, C) (lists of (coefficient, variable)
    rows), under LibsnarkReduction or CircomReduction; root(L) is the 2^L-th root of unity of the scalar field"""
    n, L = domain(rows, ni)
    nc, nv = len(rows[0]), ni + nw
    w = root(L)
    zt = (pow(tau, n, r) - 1) % r
    pw = powers(w, n, r)
    zn = zt * pow(n, -1, r) % r
    u = [zn * p % r * d % r for p, d in zip(pw, batch_inv([(tau - p) % r for p in pw], r))]
    q = [[0] * nv for _ in range(3)]
    for m, mat in enumerate(rows):
        for i, row in enumerate(mat):
            for cf, v in row:
                q[m][v] = (q[m][v] + u[i] * cf) % r
    for j in range(ni):
        q[0][j] = (q[0][j] + u[nc + j]) % r
    di, gi = pow(delta, -1, r), pow(gamma, -1, r)
    t = [(beta * q[0][j] + alpha * q[1][j] + q[2][j]) % r for j in range(nv)]
    if circom:   # the odd entries of the size-2n inverse transform of tau^i (i < 2n - 1), in closed form
        w2 = root(L + 1)
        t2n, t2n1 = pow(tau, 2 * n, r), pow(tau, 2 * n - 1, r)
        ks = [w2 * x % r for x in powers(w2 * w2 % r, n, r)]              # w2^(2j + 1)
        kis = [pow(w2, -1, r) * x % r for x in powers(pow(w2, -2, r), n, r)]
        dens = batch_inv([(tau * ki - 1) % r for ki in kis], r)
        c = di * pow(2 * n, -1, r) % r
        h = [c * ((t2n - 1) * d - t2n1 * k) % r for d, k in zip(dens, ks)]
    else:
        h = [zt * di * x % r for x in powers(tau, n - 1, r)]
    return dict(a_query=q[0], b_g1_query=list(q[1]), b_g2_query=list(q[1]), h_query=h,
                l_query=[x * di % r for x in t[ni:]], gamma_abc_g1=[x * gi % r for x in t[:ni]],
                alpha_g1=alpha % r, beta_g1=beta % r, delta_g1=delta % r, beta_g2=beta % r, gamma_g2=gamma % r,
                delta_g2=delta % r)


def combination(xs, rho, r, first=0):
    """sum_j rho^(first + j) xs[j]"""
    acc, p = 0, pow(rho, first, r)
    for x in xs:
        acc = (acc + p * x) % r
        p = p * rho % r
    return acc


def key_sums(k, rho, r, ni):
    """S_X(K) of every member the call combines: a_query, b_g1_query, b_g2_query, h_query, l_query (from rho^ni),
    gamma_abc_g1"""
    return dict(a=combination(k["a_query"], rho, r), b1=combination(k["b_g1_query"], rho, r),
                b2=combination(k["b_g2_query"], rho, r), h=combination(k["h_query"], rho, r),
                l=combination(k["l_query"], rho, r, ni), ic=combination(k["gamma_abc_g1"], rho, r))


def h_weights(r, rho, n, w2, circom):
    """the weights on tau_g1[0 .. 2n - 1) of srs_h_weights_kernel"""
    if not circom:
        return [-pow(rho, k, r) % r for k in range(n - 1)] + [0] + [pow(rho, k, r) for k in range(n - 1)]
    F = transform([pow(rho, i, r) for i in range(n)], pow(w2 * w2 % r, -1, r), r)   # n x the inverse transform
    c, wi = pow(2 * n, -1, r), pow(w2, -1, r)
    return [c * pow(wi, k, r) * F[k % n] % r for k in range(2 * n - 1)]


def transcript_sides(r, root, rows, ni, nw, tau, alpha, beta, rho, circom):
    """S_X(T) as the library forms it: z = rho^j, z^I (instance variables), z^L (the rest); a^, b^, c^ = the inverse
    transforms (with n^-1) of A z, B z, C z; a_query / b queries: sum_k a^_k tau^k, sum_k b^_k tau^k; l_query and
    gamma_abc_g1: beta sum a^_k tau^k + alpha sum b^_k tau^k + sum c^_k tau^k over z^L and z^I; h_query: sum_k s_k tau^k"""
    n, L = domain(rows, ni)
    nv = ni + nw
    w, ninv = root(L), pow(n, -1, r)
    z = [pow(rho, j, r) for j in range(nv)]
    hat = lambda zz: [[x * ninv % r for x in transform(v, pow(w, -1, r), r)] for v in row_evals(rows, ni, zz, n, r)]
    at_tau = lambda xs: combination(xs, tau, r)
    ah, bh, _ = hat(z)
    a, b = at_tau(ah), at_tau(bh)
    side = lambda zz: (lambda h: (beta * at_tau(h[0]) + alpha * at_tau(h[1]) + at_tau(h[2])) % r)(hat(zz))
    zi = z[:ni] + [0] * nw
    zl = [0] * ni + z[ni:]
    return dict(a=a, b1=b, b2=b, h=at_tau(h_weights(r, rho, n, root(L + 1), circom)), l=side(zl), ic=side(zi))


def transcript_sums(r, root, rows, ni, nw, tau, alpha, beta, rho, circom):
    """S_X(T) by the identity the CPU tier proves: the sums of g16_setup(alpha, beta, 1, 1, tau) under rho"""
    return key_sums(key_exponents(r, root, rows, ni, nw, alpha, beta, 1, 1, tau, circom), rho, r, ni)


def verdict(k, secrets, ts, rho, r, ni, uncontributed=False):
    """(refused member or None, p, q) of the call on the key with exponents k against T(*secrets) whose sums are ts"""
    _, alpha, beta = secrets
    for m, want in (("alpha_g1", alpha), ("beta_g1", beta), ("beta_g2", beta)):
        if k[m] % r != want % r:
            return m, None, None
    for m in ("delta_g1", "delta_g2", "gamma_g2"):
        if k[m] % r == 0:
            return m, None, None
    if not uncontributed and k["gamma_g2"] % r == k["delta_g2"] % r:
        return "gamma_g2", None, None
    ks = key_sums(k, rho, r, ni)
    for m, s in (("a_query", "a"), ("b_g1_query", "b1"), ("b_g2_query", "b2")):
        if ks[s] != ts[s]:
            return m, None, None
    d2 = k["delta_g2"]
    p = [k["delta_g1"], 1, ks["h"], ts["h"], ks["l"], ts["l"], ks["ic"], ts["ic"]]
    q = [1, d2, d2, 1, d2, 1, k["gamma_g2"], 1]
    return None, p, q


def failing(p, q, r) -> set:
    """the equations that do not hold"""
    return {k for k in range(4) if p[2 * k] * q[2 * k] % r != p[2 * k + 1] * q[2 * k + 1] % r}


# a wrong point of each member: the refusal it causes (a name) or the equations it breaks (a set)
EXPECTED = dict(a_query="a_query", b_g1_query="b_g1_query", b_g2_query="b_g2_query", h_query={1}, l_query={2},
                gamma_abc_g1={3}, alpha_g1="alpha_g1", beta_g1="beta_g1", beta_g2="beta_g2", delta_g1={0},
                delta_g2={0, 1, 2}, gamma_g2={3})


def copy_k(k):
    return {m: (list(v) if isinstance(v, list) else v) for m, v in k.items()}


def tamperings(k, r):
    """(name, tampered exponents, refusal or broken equations) for a wrong point of every member -- at index 0, the middle
    and the last of a vector -- plus a zero delta and gamma = delta"""
    out = []
    for m in VECTORS:
        n = len(k[m])
        for idx in sorted({0, n // 2, n - 1}):
            t = copy_k(k)
            t[m][idx] = t[m][idx] * 3 % r if t[m][idx] else 3
            out.append((f"{m}[{idx}] changed", t, EXPECTED[m]))
    for m in POINTS:
        t = copy_k(k)
        t[m] = t[m] * 5 % r
        out.append((f"{m} changed", t, EXPECTED[m]))
    t = copy_k(k)
    t["delta_g1"] = 0
    out.append(("delta_g1 the identity", t, "delta_g1"))
    t = copy_k(k)
    t["gamma_g2"] = t["delta_g2"]
    out.append(("gamma_g2 = delta_g2", t, "gamma_g2"))
    return out


def edited_rows(rows, which, ni):
    """The circuit with one coefficient changed, and the refusal or broken equations a key of it causes against the
    original: which = 0, 1: the first witness entry of A, B; 2: of C; 3: the first instance entry of C."""
    rows = [[list(row) for row in mat] for mat in rows]
    for row in rows[min(which, 2)]:
        for e, (cf, v) in enumerate(row):
            if (v < ni) == (which == 3):
                row[e] = (cf + 1, v)
                return rows, {0: "a_query", 1: "b_g1_query", 2: {2}, 3: {3}}[which]
    raise ValueError("no such entry")
