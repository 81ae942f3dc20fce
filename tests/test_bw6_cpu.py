"""CPU tier for BW6-761: re-derives every constant the library uses for the curve from its definition (primality, the CM
orders, the cofactors, the generators, the two-adic data), checks the generated header against them, and runs the host
codec on BW6 points: round trips and every rejection."""
import io
import os
import random
import re

import pytest

import bw6_ref as ref
from groth16_b200 import BW6_761, BLS12_377, CurveCodec, get_curve
from groth16_b200.params import GENERATORS
from groth16_b200.serialize import ArkCodec, DeserializeError

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fields():
    x = ref.X377
    assert (x ** 6 - 2 * x ** 5 + 2 * x ** 3 + x + 1) % 3 == 0
    assert (x ** 6 - 2 * x ** 5 + 2 * x ** 3 + x + 1) // 3 == ref.R == BLS12_377.q   # Fr is BLS12-377's Fq
    assert ref.is_probable_prime(ref.Q) and ref.is_probable_prime(ref.R)
    assert ref.Q.bit_length() == 761 and ref.R.bit_length() == 377 and ref.Q % 4 == 3
    s, t = 0, ref.R - 1
    while t % 2 == 0:
        s, t = s + 1, t // 2
    assert s == ref.TWO_ADICITY == 46
    assert pow(ref.FR_GENERATOR, (ref.R - 1) // 2, ref.R) == ref.R - 1   # a quadratic non-residue
    c = get_curve("bw6_761")
    assert c is BW6_761 and (c.r, c.q, c.fr_generator, c.two_adicity, c.cid) == (ref.R, ref.Q, 15, 46, 3)
    assert (c.fr_limbs, c.fq_limbs, c.g2_limbs) == (6, 12, 24)


def test_curve_orders_and_generators():
    orders = ref.cm_orders()
    assert len(set(orders)) == 6 and sum(1 for n in orders if n % ref.R == 0) == 2
    for b, name in ((ref.B1, "g1"), (ref.B2, "g2")):
        n = ref.order_of_curve(b)
        assert n in orders and n % ref.R == 0 and (n // ref.R).bit_length() == 384
        P = GENERATORS["bw6_761"][name]
        assert ref.on_curve(P, b) and P is not None
        assert ref.mul(ref.R, P) is None
        assert P == ref.hash_to_subgroup(b, n, f"bw6_761-{name}")


def _header_struct(name):
    txt = open(os.path.join(ROOT, "groth16_b200", "csrc", "g16_constants.h")).read()
    body = re.search(r"struct %s \{(.*?)\n\};" % name, txt, flags=re.S).group(1)
    out = {}
    for fn, arr in re.findall(r"uint32_t (\w+)\(int i\) \{ constexpr uint32_t t\[\d+\] = \{([^}]*)\}", body):
        out[fn] = sum(int(w.strip().rstrip("u"), 16) << (32 * i) for i, w in enumerate(arr.split(",")))
    for k, v in re.findall(r"static constexpr (?:int|uint32_t) (\w+) = (0x[0-9a-f]+|\d+)u?;", body):
        out[k] = int(v, 0)
    return out, body


def test_generated_header():
    fr, _ = _header_struct("BW6_FrP")
    fq, _ = _header_struct("BW6_FqP")
    _, params = _header_struct("BW6_Params")
    for h, p, n in ((fr, ref.R, 12), (fq, ref.Q, 24)):
        R = 1 << (32 * n)
        assert h["N"] == n and h["BITS"] == p.bit_length() and h["mod"] == p
        assert h["one"] == R % p and h["r2"] == R * R % p
        assert (h["INV32"] * p) % (1 << 32) == (1 << 32) - 1
    Rr, Rq = 1 << 384, 1 << 768
    assert fr["TWO_ADICITY"] == 46 and fr["generator"] == 15 * Rr % ref.R
    assert fr["two_adic_root"] == pow(15, (ref.R - 1) >> 46, ref.R) * Rr % ref.R
    assert fq["curve_b"] == (ref.Q - 1) * Rq % ref.Q and fq["twist_b0"] == 4 * Rq % ref.Q and "twist_b1" not in fq
    assert "CURVE_ID = 3" in params and "using G2F = Fp<BW6_FqP>;" in params


def _non_subgroup_point(b, seed):
    rng = random.Random(seed)
    while True:
        x = rng.randrange(ref.Q)
        y = ref.sqrt_fq((x ** 3 + b) % ref.Q)
        if y is not None and ref.mul(ref.R, (x, y)) is not None:
            return x, y


@pytest.mark.parametrize("g2", [False, True])
def test_codec_round_trips_and_rejections(g2):
    cd = CurveCodec(BW6_761)
    ac = ArkCodec("bw6_761", check_subgroup=True)
    b = ref.B2 if g2 else ref.B1
    gen = GENERATORS["bw6_761"]["g2" if g2 else "g1"]
    rng = random.Random(g2)
    pts = [None, gen] + [ref.mul(rng.randrange(ref.R), gen) for _ in range(4)]
    enc, dec = (cd.enc_g2, cd.dec_g2) if g2 else (cd.enc_g1, cd.dec_g1)
    assert enc(pts).shape == (len(pts), 24) and dec(enc(pts)) == pts
    for compress in (True, False):
        for P in pts:
            raw = ac.point(P, g2, compress)
            assert len(raw) == 96 * (1 if compress else 2)
            assert ac.read_point(io.BytesIO(raw), g2, compress) == P
        P = pts[2]
        raw = bytearray(ac.point(P, g2, compress))
        bad = bytearray(raw)
        bad[-1] |= 0xC0
        with pytest.raises(DeserializeError, match="both SWFlags"):
            ac.read_point(io.BytesIO(bytes(bad)), g2, compress)
        bad = bytearray(ac.point(None, g2, compress))
        bad[0] = 1
        with pytest.raises(DeserializeError, match="infinity"):
            ac.read_point(io.BytesIO(bytes(bad)), g2, compress)
        bad = bytearray((ref.Q + 1).to_bytes(96, "little")) + raw[96:]
        with pytest.raises(DeserializeError, match="non-canonical"):
            ac.read_point(io.BytesIO(bytes(bad)), g2, compress)
        with pytest.raises(DeserializeError, match="subgroup"):
            ac.read_point(io.BytesIO(ac.point(_non_subgroup_point(b, 3), g2, compress)), g2, compress)
        with pytest.raises(DeserializeError, match="truncated"):
            ac.read_point(io.BytesIO(bytes(raw[:-1])), g2, compress)
    # off the curve (uncompressed) and no root (compressed)
    P = pts[3]
    with pytest.raises(DeserializeError, match="not on the curve"):
        ac.read_point(io.BytesIO(ac.point((P[0], (P[1] + 1) % ref.Q), g2, False)), g2, False)
    x = 5
    while ref.sqrt_fq((x ** 3 + b) % ref.Q) is not None:
        x += 1
    with pytest.raises(DeserializeError, match="abscissa"):
        ac.read_point(io.BytesIO(x.to_bytes(96, "little")), g2, True)
    # G1 and G2 differ in b: a G2 point is not a G1 point
    if g2:
        with pytest.raises(DeserializeError):
            ac.read_point(io.BytesIO(ac.point(gen, True, False)), False, False)


def test_scalars_and_host_msm_reference():
    ac = ArkCodec("bw6_761")
    assert len(ac.fr(ref.R - 1)) == 48 and ac.read_fr(io.BytesIO(ac.fr(12345))) == 12345
    g = GENERATORS["bw6_761"]["g1"]
    # the reference's MSM agrees with a plain scalar multiple, at the edge scalars the GPU tests use
    for k in (0, 1, ref.R - 1, (1 << 376) | 0xFFFF):
        assert ref.msm([g, g], [k, 1]) == ref.add(ref.mul(k % ref.R, g), g)
    assert ref.mul(ref.R - 1, g) == ref.neg(g)


def test_ntt_reference_round_trip():
    rng = random.Random(2)
    x = [rng.randrange(ref.R) for _ in range(16)]
    for coset in (False, True):
        assert ref.ntt(ref.ntt(x, coset=coset), inverse=True, coset=coset) == x
    assert pow(ref.domain_root(4), 16, ref.R) == 1 and pow(ref.domain_root(4), 8, ref.R) != 1


def test_projective_mul_and_fast_ntt():
    """mul_proj (one inversion) against the affine double-and-add, at scalars beyond r too; fft against the naive ntt"""
    rng = random.Random(4)
    for name in ("g1", "g2"):
        g = GENERATORS["bw6_761"][name]
        for k in (0, 1, 2, 3, ref.R - 1, ref.R, ref.R + 1, (1 << 384) - 1, rng.randrange(1 << 40)):
            assert ref.mul_proj(k, g) == ref.mul(k, g), (name, k)
    assert ref.mul_proj(2, (7, 0)) is None and ref.mul_proj(5, None) is None
    for log_n in range(7):
        x = [rng.randrange(ref.R) for _ in range(1 << log_n)]
        x[0] = ref.R - 1
        for inverse in (False, True):
            for coset in (False, True):
                assert ref.fft(x, inverse, coset) == ref.ntt(x, inverse, coset), (log_n, inverse, coset)


def _random_r1cs(rng, nc, ni, nw):
    """nc random constraints over One, ni - 1 inputs and nw witnesses: one to three terms per row, coefficients at the
    edges (1, r - 1) and random"""
    nv = ni + nw
    coeff = lambda: rng.choice([1, ref.R - 1, rng.randrange(ref.R)])
    rows = tuple([[(coeff(), rng.randrange(nv)) for _ in range(rng.randrange(1, 4))] for _ in range(nc)] for _ in range(3))
    return rows, nv


def _witness_map_naive(a, b, c):
    n = len(a)
    ac, bc, cc = (ref.ntt(ref.ntt(x, inverse=True), coset=True) for x in (a, b, c))
    zi = pow((pow(ref.FR_GENERATOR, n, ref.R) - 1) % ref.R, -1, ref.R)
    return ref.ntt([(x * y - z) * zi % ref.R for x, y, z in zip(ac, bc, cc)], inverse=True, coset=True)


@pytest.mark.parametrize("nc,ni,nw", [(1, 1, 1), (2, 2, 3), (5, 2, 6), (13, 3, 9), (29, 2, 20), (60, 4, 40)])
def test_closed_form_proof_any_assignment(nc, ni, nw):
    """proof_exponents (O(n) closed form, for any assignment) against the prover's definition: the five MSMs over the
    key's discrete logs with h from the naive-NTT witness map, at domains 2 .. 2^6 and random assignments that do not
    satisfy the circuit; a satisfying assignment (c = a * b by construction) as well"""
    rng = random.Random(nc * 100 + ni)
    rows, nv = _random_r1cs(rng, nc, ni, nw)
    alpha, beta, _gamma, delta, tau = (rng.randrange(1, ref.R) for _ in range(5))
    d = ref.query_exponents(rows, ni, nv, alpha, beta, delta, tau)
    n, _ = ref.domain_size(rows, ni)
    assert len(d["a"]) == len(d["b"]) == nv and len(d["l"]) == nv - ni and len(d["h"]) == n - 1
    for k in range(4):
        z = [1] + [rng.randrange(ref.R) for _ in range(nv - 1)]
        if k == 3:   # satisfy every row: a fresh witness variable per row would be needed, so make C's rows A * B directly
            ev = ref.row_evals(rows, ni, z)
            rows = (rows[0], rows[1], [[(ev[0][j] * ev[1][j] % ref.R, 0)] for j in range(nc)])
            d = ref.query_exponents(rows, ni, nv, alpha, beta, delta, tau)
        ev = ref.row_evals(rows, ni, z)
        h = _witness_map_naive(*ev)
        assert h == ref.witness_map(*ev)
        if k == 3:
            assert all((x * y - w) % ref.R == 0 for x, y, w in zip(*ev)) and h[-1] == 0
        else:
            assert any((x * y - w) % ref.R for x, y, w in zip(*ev))
        r, s = (0, rng.randrange(ref.R)) if k == 1 else (rng.randrange(ref.R), rng.randrange(ref.R))
        e = ref.msm_exponents(d, h, z, ni)
        want = ref.proof_from_msms(e, (d["a"][0], d["b"][0], d["b"][0]), alpha, beta, delta, r, s)
        assert ref.proof_exponents(rows, ni, z, alpha, beta, delta, tau, r, s) == want, k
