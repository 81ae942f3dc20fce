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


def expected_proof(rows, num_inputs, z, alpha, beta, delta, tau, r, s, g1, g2):
    """A, B, C of a Groth16 proof (libsnark QAP; CircomReduction gives the same points) from the toxic waste:
    A = [alpha + a(tau) + r delta]_1, B = [beta + b(tau) + s delta]_2,
    C = [(sum_{i >= ni} z_i (beta a_i + alpha b_i + c_i)(tau) + a(tau) b(tau) - c(tau)) / delta + s A + r B - r s delta]_1
    with x(tau) = sum_i z_i x_i(tau).  rows = (A, B, C), each a list of constraints [(coeff, var), ...]."""
    nc = len(rows[0])
    n, L = 1, 0
    while n < nc + num_inputs:
        n, L = 2 * n, L + 1
    lag = lagrange_at(tau, L)
    ev = []       # a(tau), b(tau), c(tau)
    inst = []     # sum_{i < ni} z_i x_i(tau)
    for m, mat in enumerate(rows):
        tot, ins = 0, 0
        for j, row in enumerate(mat):
            v = sum(cf * z[var] for cf, var in row) % R
            tot += lag[j] * v
            ins += lag[j] * sum(cf * z[var] for cf, var in row if var < num_inputs)
        if m == 0:   # the instance copy a[nc + i] = z_i (r1cs_to_qap.rs)
            for i in range(num_inputs):
                tot += lag[nc + i] * z[i]
                ins += lag[nc + i] * z[i]
        ev.append(tot % R)
        inst.append(ins % R)
    a_s = (alpha + ev[0] + r * delta) % R
    b_s = (beta + ev[1] + s * delta) % R
    wit = (beta * (ev[0] - inst[0]) + alpha * (ev[1] - inst[1]) + (ev[2] - inst[2])) % R
    c_s = ((wit + ev[0] * ev[1] - ev[2]) * pow(delta, -1, R) + s * a_s + r * b_s - r * s * delta) % R
    return mul(a_s, g1), mul(b_s, g2), mul(c_s, g1)


def csr_rows(m):
    """groth16_b200 ConstraintMatrices -> rows (A, B, C) of (coeff, var) with canonical coefficients"""
    from groth16_b200.codec import FieldCodec
    fr = FieldCodec(R)
    out = []
    for rp, col, val in (m.a, m.b, m.c):
        vals = fr.dec(val) if len(col) else []
        out.append([[(vals[e], int(col[e])) for e in range(int(rp[i]), int(rp[i + 1]))] for i in range(len(rp) - 1)])
    return out
