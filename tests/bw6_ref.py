"""Big-integer reference for BW6-761, written from the curve's definition alone (no import from groth16_b200's CUDA side).

BW6-761 is the outer curve of BLS12-377 recursion: its scalar field is BLS12-377's base field.  Both groups are over Fq:
G1 is y^2 = x^3 - 1, G2 is y^2 = x^3 + 4.  There is no pairing here; a Groth16 proof is checked by the closed form "proof in
the exponent" (`expected_proof`): with the toxic waste known, A, B and C are fixed multiples of the two generators.

Points are affine (x, y) int tuples, None for the identity, as in groth16_b200.codec."""
import math
import random

R = 258664426012969094010652733694893533536393512754914660539884262666720468348340822774968888139573360124440321458177
Q = int("122e824fb83ce0ad187c94004faff3eb926186a81d14688528275ef8087be41707ba638e584e91903cebaff25b423048689c8ed12f9fd9071dc"
        "d3dc73ebff2e98a116c25667a8f8160cf8aeeaf0a437e6913e6870000082f49d00000000008b", 16)
X377 = 0x8508C00000000001          # the BLS12-377 seed
B1, B2 = Q - 1, 4                  # curve coefficients of G1 and G2
FR_GENERATOR, TWO_ADICITY = 15, 46


def is_probable_prime(n, rounds=32, seed=1):
    if n < 4:
        return n in (2, 3)
    d, s = n - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    rng = random.Random(seed)
    for _ in range(rounds):
        y = pow(rng.randrange(2, n - 1), d, n)
        if y in (1, n - 1):
            continue
        for _ in range(s - 1):
            y = y * y % n
            if y == n - 1:
                break
        else:
            return False
    return True


def cm_orders(q=Q):
    """The six group orders q + 1 - t of the j = 0 curves over Fq: 4q = t^2 + 3y^2 solved by Cornacchia."""
    s = pow(q - 3, (q + 1) // 4, q)           # sqrt(-3) (q = 3 mod 4)
    assert s * s % q == q - 3
    if s % 2 != q % 2:
        s = q - s
    a, b, lim = 2 * q, s, math.isqrt(4 * q)
    while b > lim:
        a, b = b, a % b
    t = b
    y2 = (4 * q - t * t) // 3
    y = math.isqrt(y2)
    assert 3 * y * y == 4 * q - t * t
    traces = (t, -t, (t + 3 * y) // 2, -(t + 3 * y) // 2, (t - 3 * y) // 2, -(t - 3 * y) // 2)
    return [q + 1 - tr for tr in traces]


# ---- curve arithmetic (affine, one inversion per operation) ------------------------------------------------------------
def on_curve(P, b):
    return P is None or (P[1] * P[1] - P[0] ** 3 - b) % Q == 0


def add(P, Qp):
    if P is None:
        return Qp
    if Qp is None:
        return P
    if P[0] == Qp[0]:
        if (P[1] + Qp[1]) % Q == 0:
            return None
        lam = 3 * P[0] * P[0] * pow(2 * P[1], -1, Q) % Q
    else:
        lam = (Qp[1] - P[1]) * pow(Qp[0] - P[0], -1, Q) % Q
    x = (lam * lam - P[0] - Qp[0]) % Q
    return x, (lam * (P[0] - x) - P[1]) % Q


def neg(P):
    return None if P is None else (P[0], (-P[1]) % Q)


def mul(k, P):
    acc = None
    for bit in bin(k)[2:] if k > 0 else "":
        acc = add(acc, acc)
        if bit == "1":
            acc = add(acc, P)
    return acc


def msm(bases, scalars):
    acc = None
    for P, k in zip(bases, scalars):
        acc = add(acc, mul(k % R, P))
    return acc


def _jdbl(X, Y, Z):
    """2 (X : Y : Z) in Jacobian coordinates (a = 0; Z = 0 is the identity)"""
    A, B = X * X % Q, Y * Y % Q
    C = B * B % Q
    D = 2 * ((X + B) ** 2 - A - C) % Q
    E = 3 * A % Q
    X3 = (E * E - 2 * D) % Q
    return X3, (E * (D - X3) - 8 * C) % Q, 2 * Y * Z % Q


def mul_proj(k, P):
    """k P for any k >= 0 with one inversion: left-to-right double-and-add in Jacobian coordinates, adding the affine P"""
    if P is None or k == 0:
        return None
    x, y = P
    X, Y, Z = 0, 1, 0
    for bit in bin(k)[2:]:
        if Z:
            X, Y, Z = _jdbl(X, Y, Z)
        if bit == "1":
            if not Z:
                X, Y, Z = x, y, 1
                continue
            ZZ = Z * Z % Q
            H = (x * ZZ - X) % Q
            S = (y * ZZ * Z - Y) % Q
            if H == 0:
                if S == 0:
                    X, Y, Z = _jdbl(X, Y, Z)
                else:
                    X, Y, Z = 0, 1, 0
                continue
            HH = H * H % Q
            HHH = H * HH % Q
            V = X * HH % Q
            X3 = (S * S - HHH - 2 * V) % Q
            X, Y, Z = X3, (S * (V - X3) - Y * HHH) % Q, Z * H % Q
    if not Z:
        return None
    zi = pow(Z, -1, Q)
    zi2 = zi * zi % Q
    return X * zi2 % Q, Y * zi2 * zi % Q


def sqrt_fq(a):
    y = pow(a, (Q + 1) // 4, Q)
    return y if y * y % Q == a % Q else None


def order_of_curve(b):
    """The CM order whose multiple annihilates two points of y^2 = x^3 + b: the group order."""
    rng = random.Random(b)
    pts = []
    while len(pts) < 2:
        x = rng.randrange(Q)
        y = sqrt_fq((x ** 3 + b) % Q)
        if y is not None:
            pts.append((x, y))
    found = [n for n in cm_orders() if all(mul(n, P) is None for P in pts)]
    assert len(found) == 1, found
    return found[0]


def hash_to_subgroup(b, order, tag):
    """The first x = H(tag, i) with a curve point, times the cofactor.  H is sha512 repeated to 1024 bits, little-endian, mod
    q: the other curves' generators hash with sha256, which is too short for a 761-bit x, so BW6-761 has this recipe of its
    own."""
    import hashlib
    h = order // R
    for i in range(1000):
        x = int.from_bytes(hashlib.sha512(f"{tag}:{i}".encode()).digest() * 2, "little") % Q
        y = sqrt_fq((x ** 3 + b) % Q)
        if y is None:
            continue
        P = mul(h, (x, min(y, Q - y)))
        if P is not None:
            return P
    raise AssertionError("no point")


# ---- scalar field: domain, QAP at tau, closed-form proof -------------------------------------------------------------
def domain_root(log_n):
    w = pow(FR_GENERATOR, (R - 1) >> TWO_ADICITY, R)
    return pow(w, 1 << (TWO_ADICITY - log_n), R)


def ntt(vals, inverse=False, coset=False):
    """domain.fft / ifft (coset: over g * domain, g = FR_GENERATOR), naive O(n^2)"""
    n = len(vals)
    L = n.bit_length() - 1
    w = domain_root(L)
    if not inverse:
        if coset:
            vals = [v * pow(FR_GENERATOR, i, R) % R for i, v in enumerate(vals)]
        return [sum(v * pow(w, i * k, R) for i, v in enumerate(vals)) % R for k in range(n)]
    wi, ni = pow(w, -1, R), pow(n, -1, R)
    out = [sum(v * pow(wi, i * k, R) for i, v in enumerate(vals)) * ni % R for k in range(n)]
    if coset:
        gi = pow(FR_GENERATOR, -1, R)
        out = [v * pow(gi, i, R) % R for i, v in enumerate(out)]
    return out


def lagrange_at(tau, log_n):
    """L_j(tau) over the domain of size 2^log_n, j < n (one batch inversion)"""
    n = 1 << log_n
    w = domain_root(log_n)
    zt = (pow(tau, n, R) - 1) % R
    pw, dens = 1, []
    for _ in range(n):
        dens.append((tau - pw) % R)
        pw = pw * w % R
    pref, acc = [], 1
    for d in dens:
        pref.append(acc)
        acc = acc * d % R
    inv = pow(acc, -1, R)
    invs = [0] * n
    for j in range(n - 1, -1, -1):
        invs[j] = inv * pref[j] % R
        inv = inv * dens[j] % R
    c = zt * pow(n, -1, R) % R
    out, pw = [], 1
    for j in range(n):
        out.append(c * pw % R * invs[j] % R)
        pw = pw * w % R
    return out


def fft(vals, inverse=False, coset=False):
    """the same transforms as `ntt` in O(n log n): iterative radix-2 over the bit-reversed input"""
    n = len(vals)
    L = n.bit_length() - 1
    a = [v % R for v in vals]
    if coset and not inverse:
        gp = 1
        for i in range(n):
            a[i] = a[i] * gp % R
            gp = gp * FR_GENERATOR % R
    j = 0
    for i in range(1, n):
        bit = n >> 1
        while j & bit:
            j ^= bit
            bit >>= 1
        j |= bit
        if i < j:
            a[i], a[j] = a[j], a[i]
    w = domain_root(L)
    if inverse:
        w = pow(w, -1, R)
    m = 1
    while m < n:
        wm = pow(w, n // (2 * m), R)
        tw = [1] * m
        for k in range(1, m):
            tw[k] = tw[k - 1] * wm % R
        for st in range(0, n, 2 * m):
            for k in range(m):
                u, t = a[st + k], a[st + k + m] * tw[k] % R
                a[st + k], a[st + k + m] = (u + t) % R, (u - t) % R
        m *= 2
    if inverse:
        ni, gi = pow(n, -1, R), pow(FR_GENERATOR, -1, R) if coset else 1
        c = ni
        for i in range(n):
            a[i] = a[i] * c % R
            c = c * gi % R
    return a


def domain_size(rows, num_inputs):
    """(n, log n) of the QAP domain: the constraints plus one instance copy per input"""
    n, L = 1, 0
    while n < len(rows[0]) + num_inputs:
        n, L = 2 * n, L + 1
    return n, L


def row_evals(rows, num_inputs, z):
    """LibsnarkReduction's evaluations of A, B, C on the domain: row j of each matrix at z, the instance copy
    a[nc + i] = z_i (r1cs_to_qap.rs), zero above"""
    n, _ = domain_size(rows, num_inputs)
    nc = len(rows[0])
    out = []
    for m, mat in enumerate(rows):
        ev = [sum(cf * z[var] for cf, var in row) % R for row in mat] + [0] * (n - nc)
        if m == 0:
            for i in range(num_inputs):
                ev[nc + i] = z[i] % R
        out.append(ev)
    return out


def witness_map(a, b, c):
    """LibsnarkReduction's h (n coefficients) from the row evaluations: coset-ifft((A B - C) / Z) with X = coset-fft(ifft(x));
    Z is g^n - 1 at every point of the coset"""
    n = len(a)
    ac, bc, cc = (fft(fft(x, inverse=True), coset=True) for x in (a, b, c))
    zi = pow((pow(FR_GENERATOR, n, R) - 1) % R, -1, R)
    return fft([(x * y - z) * zi % R for x, y, z in zip(ac, bc, cc)], inverse=True, coset=True)


def query_exponents(rows, num_inputs, num_vars, alpha, beta, delta, tau):
    """The discrete logs of the five queries of a key g16_setup makes from this toxic waste: every point is [d]G with
    a: a_i(tau) and b: b_i(tau) for every variable (b_g1_query and b_g2_query alike), l: (beta a_i + alpha b_i + c_i)(tau) /
    delta for i >= num_inputs, h: tau^i Z(tau) / delta for i < n - 1."""
    n, L = domain_size(rows, num_inputs)
    nc = len(rows[0])
    lag = lagrange_at(tau, L)
    q = [[0] * num_vars for _ in range(3)]
    for m, mat in enumerate(rows):
        for j, row in enumerate(mat):
            for cf, var in row:
                q[m][var] += lag[j] * cf
    for i in range(num_inputs):
        q[0][i] += lag[nc + i]
    qa, qb, qc = ([v % R for v in x] for x in q)
    di = pow(delta, -1, R)
    zd = (pow(tau, n, R) - 1) * di % R
    h, p = [], zd
    for _ in range(n - 1):
        h.append(p)
        p = p * tau % R
    return dict(a=qa, b=qb, l=[(beta * qa[i] + alpha * qb[i] + qc[i]) * di % R for i in range(num_inputs, num_vars)], h=h)


def msm_exponents(d, h, z, num_inputs):
    """The exponents of the prover's five MSMs over a key with discrete logs d (`query_exponents`, possibly edited): H over
    the first n - 1 coefficients of h, L over the witness, A, B in G1 and B in G2 over every variable but the constant One"""
    dot = lambda xs, ys: sum(x * y for x, y in zip(xs, ys)) % R
    b1, b2 = (d[k] if k in d else d["b"] for k in ("b_g1", "b_g2"))   # one b for both groups unless edited apart
    return dict(h=dot(d["h"], h), l=dot(d["l"], z[num_inputs:]), a=dot(d["a"][1:], z[1:]), b_g1=dot(b1[1:], z[1:]),
                b_g2=dot(b2[1:], z[1:]))


def proof_from_msms(e, d0, alpha, beta, delta, r, s):
    """A, B, C exponents as the prover assembles them from its MSM exponents e and the first entries d0 = (a_0, b_g1_0,
    b_g2_0) of the queries (the constant One): A = alpha + a + r delta, B = beta + b + s delta, C = h + l + s A + r B_1 -
    r s delta"""
    a_s = (alpha + d0[0] + e["a"] + r * delta) % R
    b1 = (beta + d0[1] + e["b_g1"] + s * delta) % R
    b_s = (beta + d0[2] + e["b_g2"] + s * delta) % R
    return a_s, b_s, (e["h"] + e["l"] + s * a_s + r * b1 - r * s * delta) % R


def proof_exponents(rows, num_inputs, z, alpha, beta, delta, tau, r, s):
    """A, B, C of a Groth16 proof (libsnark QAP) as exponents of the generators, for ANY assignment z, in O(n):
    A = alpha + a(tau) + r delta, B = beta + b(tau) + s delta, with x(tau) = sum_i z_i x_i(tau), and
    C = sum_{i >= ni} z_i (beta a_i + alpha b_i + c_i)(tau) / delta + H + s A + r B - r s delta.
    H is what the prover's H MSM gives, sum_{i < n-1} h_i tau^i Z(tau) / delta.  With the row evaluations e_j = a_j b_j - c_j
    and rem(X) = sum_j e_j L_j(X) (a b - c mod Z), the witness map's h interpolates (a b - c) / (g^n - 1) on the coset, so
    h = (a b - c - rem) / Z + rem / (g^n - 1), of degree < n, with top coefficient h_{n-1} = (sum_j e_j w^j) / (n (g^n - 1));
    h_query has n - 1 points, so H = (h(tau) - h_{n-1} tau^{n-1}) Z(tau) / delta.  For a satisfying z, rem = 0 and
    H = (a(tau) b(tau) - c(tau)) / delta."""
    n, L = domain_size(rows, num_inputs)
    lag = lagrange_at(tau, L)
    ev = row_evals(rows, num_inputs, z)
    at, bt, ct = (sum(l * v for l, v in zip(lag, e)) % R for e in ev)
    # the instance part of a(tau), b(tau), c(tau): only z_i with i < ni, the instance copies included
    inst = []
    nc = len(rows[0])
    for m, mat in enumerate(rows):
        tot = sum(lag[j] * sum(cf * z[var] for cf, var in row if var < num_inputs) for j, row in enumerate(mat))
        if m == 0:
            tot += sum(lag[nc + i] * z[i] for i in range(num_inputs))
        inst.append(tot % R)
    e = [(x * y - w) % R for x, y, w in zip(*ev)]
    rem = sum(l * v for l, v in zip(lag, e)) % R
    w, wp, top = domain_root(L), 1, 0
    for v in e:
        top += v * wp
        wp = wp * w % R
    gn1 = (pow(FR_GENERATOR, n, R) - 1) % R
    top = top * pow(n * gn1, -1, R) % R
    zt = (pow(tau, n, R) - 1) % R
    h_tau = ((at * bt - ct - rem) * pow(zt, -1, R) + rem * pow(gn1, -1, R)) % R
    di = pow(delta, -1, R)
    hh = (h_tau - top * pow(tau, n - 1, R)) * zt % R
    a_s = (alpha + at + r * delta) % R
    b_s = (beta + bt + s * delta) % R
    wit = (beta * (at - inst[0]) + alpha * (bt - inst[1]) + (ct - inst[2])) % R
    c_s = ((wit + hh) * di + s * a_s + r * b_s - r * s * delta) % R
    return a_s, b_s, c_s


def expected_proof(rows, num_inputs, z, alpha, beta, delta, tau, r, s, g1, g2):
    """A, B, C of a Groth16 proof from the toxic waste (`proof_exponents`; CircomReduction gives the same points for a
    satisfying z).  rows = (A, B, C), each a list of constraints [(coeff, var), ...]."""
    a_s, b_s, c_s = proof_exponents(rows, num_inputs, z, alpha, beta, delta, tau, r, s)
    return mul_proj(a_s, g1), mul_proj(b_s, g2), mul_proj(c_s, g1)


def csr_rows(m):
    """groth16_b200 ConstraintMatrices -> rows (A, B, C) of (coeff, var) with canonical coefficients"""
    from groth16_b200.codec import FieldCodec
    fr = FieldCodec(R)
    out = []
    for rp, col, val in (m.a, m.b, m.c):
        vals = fr.dec(val) if len(col) else []
        out.append([[(vals[e], int(col[e])) for e in range(int(rp[i]), int(rp[i + 1]))] for i in range(len(rp) - 1)])
    return out
