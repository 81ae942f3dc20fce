"""ark-circom's CircomReduction restated for the tests, from its definition (not from the CUDA code).

n is the domain size D::new(num_constraints + num_inputs), as in LibsnarkReduction; omega_2n is element(1) of the domain of
size 2n.
  witness_map_from_matrices: a, b are the row evaluations (plus the instance copy into a) of LibsnarkReduction; c = a o b
    (matrix C is never read); each of a, b, c goes through ifft on the domain, X[i] *= omega_2n^i, fft on the domain (the
    evaluations at the odd powers omega_2n^(2j+1), natural order); h[j] = A[j] B[j] - C[j]: n evaluations, no division.
  h_query_scalars(n - 1, tau, _, delta^-1): the odd entries 1, 3, .., 2n - 1 of the size-2n ifft of v, v[i] = delta^-1 tau^i
    for i < 2n - 1, v[2n - 1] = 0: n scalars.
Two restatements of each: big-integer Python on pyref's domain (any size a test can afford), and one built on the C++
oracle's transforms (orc.ntt), which reaches 2^20: the odd-point evaluations are the odd entries of a size-2n fft of the
coefficients padded with n zeros, a route independent of the pre-scaling the definition uses."""
import dataclasses

import numpy as np

import orc
import pyref as P


def omega_2n(dom: "P.Domain") -> int:
    return P.Domain(dom.c, 2 * dom.n).omega


def witness_map_from_evals(dom: "P.Domain", a, b):
    r = dom.r
    c = [x * y % r for x, y in zip(a, b)]
    w = omega_2n(dom)
    out = []
    for x in (a, b, c):
        coeffs = dom.ifft(x)
        p = 1
        for i in range(dom.n):                 # distribute_powers_and_mul_by_const(X, omega_2n, 1)
            coeffs[i] = coeffs[i] * p % r
            p = p * w % r
        out.append(dom.fft(coeffs))
    A, B, C = out
    return [(x * y - z) % r for x, y, z in zip(A, B, C)]


def witness_map(cs: "P.R1CS"):
    dom, a, b, _ = P.abc_evals(cs)
    return witness_map_from_evals(dom, a, b)


def h_query_scalars(dom: "P.Domain", tau: int, delta_inv: int):
    """the literal definition: a size-2n ifft"""
    r, n = dom.r, dom.n
    v = [delta_inv * pow(tau, i, r) % r for i in range(2 * n - 1)] + [0]
    return P.Domain(dom.c, 2 * n).ifft(v)[1::2]


def h_query_scalars_closed_form(dom: "P.Domain", tau: int, delta_inv: int):
    """the closed form the library's setup evaluates (one batch inversion):
    L_{2j+1} = delta^-1 / (2n) [(tau^2n - 1) / (tau w^-(2j+1) - 1) - tau^(2n-1) w^(2j+1)],  w = omega_2n"""
    r, n = dom.r, dom.n
    w = omega_2n(dom)
    wi = pow(w, -1, r)
    t2n = pow(tau, 2 * n, r)
    assert t2n != 1, "tau lies in the domain of size 2n"
    dens = [(tau * pow(wi, 2 * j + 1, r) - 1) % r for j in range(n)]
    invs = P.batch_inv(dens, r)
    c = delta_inv * pow(2 * n, -1, r) % r
    return [c * ((t2n - 1) * invs[j] - pow(tau, 2 * n - 1, r) * pow(w, 2 * j + 1, r)) % r for j in range(n)]


def generate_parameters(cs: "P.R1CS", alpha, beta, gamma, delta, tau, qap="libsnark"):
    """pyref.generate_parameters under either reduction: CircomReduction's key differs in the H query alone
    (instance_map_with_evaluation is LibsnarkReduction's)."""
    pk = P.generate_parameters(cs, alpha, beta, gamma, delta, tau)
    if qap == "libsnark":
        return pk
    assert qap == "circom"
    dom = P.Domain(cs.curve, cs.num_constraints + cs.num_instance)
    hs = h_query_scalars(dom, tau, pow(delta, -1, cs.curve.r))
    G1, g1 = P.ctx(cs.curve).G1, pk.toxic["g1"]
    return dataclasses.replace(pk, h_query=[G1.mul(g1, s) for s in hs], toxic=dict(pk.toxic, h=hs))


def create_proof(pk: "P.ProvingKey", cs: "P.R1CS", r_: int, s_: int, qap="libsnark"):
    if qap == "libsnark":
        return P.create_proof(pk, cs, r_, s_)
    assert qap == "circom"
    z = cs.assignment
    return P.create_proof_with_assignment(pk, r_, s_, witness_map(cs), z[1:cs.num_instance], z[cs.num_instance:])


# ---- the same on the C++ oracle's transforms (ABI arrays in and out) ---------------------------------------------------


def _ints(cd, arr):
    return cd.fr.dec(np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1, 4))


def row_evals(cd, m, z):
    """a, b of LibsnarkReduction's row evaluation (r1cs_to_qap.rs:183-199) as ints, padded to the domain size"""
    r = cd.c.r
    zi = _ints(cd, z)
    n = 1 << max(m.num_constraints + m.num_instance_variables - 1, 0).bit_length()
    out = []
    for rp, col, val in (m.a, m.b):
        vals = _ints(cd, val) if len(col) else []
        rp, col = np.asarray(rp).tolist(), np.asarray(col).tolist()
        x = [sum(vals[e] * zi[col[e]] for e in range(rp[i], rp[i + 1])) % r for i in range(m.num_constraints)]
        out.append(x + [0] * (n - m.num_constraints))
    for i in range(m.num_instance_variables):
        out[0][m.num_constraints + i] = zi[i]
    return out[0], out[1]


def orc_witness_map(cd, m, z, threads=1):
    """CircomReduction::witness_map_from_matrices on ABI arrays -> n Montgomery limbs"""
    r = cd.c.r
    a, b = row_evals(cd, m, z)
    n = len(a)
    log_n = n.bit_length() - 1
    c = [x * y % r for x, y in zip(a, b)]
    ev = []
    for x in (a, b, c):
        coeffs = orc.ntt(cd.c.cid, log_n, cd.fr.enc(x), inverse=True, threads=threads)
        padded = np.concatenate([coeffs, np.zeros_like(coeffs)])
        ev.append(_ints(cd, orc.ntt(cd.c.cid, log_n + 1, padded, threads=threads)[1::2]))
    A, B, C = ev
    return cd.fr.enc([(x * y - w) % r for x, y, w in zip(A, B, C)])


def orc_h_query_scalars(cd, log_n, tau, delta_inv, threads=1):
    """CircomReduction::h_query_scalars on the oracle's size-2n ifft -> n Montgomery limbs"""
    r, n = cd.c.r, 1 << log_n
    v, p = [], delta_inv % r
    for _ in range(2 * n - 1):
        v.append(p)
        p = p * tau % r
    v.append(0)
    return orc.ntt(cd.c.cid, log_n + 1, cd.fr.enc(v), inverse=True, threads=threads)[1::2].copy()
