"""GPU tier of g16_ptau_prepare (snarkjs `powersoftau prepare phase2` on the GPU): the prepared file of the transcript
T(TAU, ALPHA, BETA) must equal, byte for byte, ptau_ref.write of the expected Lagrange levels, every expected point formed
without any group transform:
  levels 1 .. power   ptau_ref.lagrange_from_setup (the library's g16_setup of diagonal circuits);
  level 0             X_0;
  level power + 1 of tauG1 (the missing last power taken as the identity): entry i is
      [L_i^(2n)(tau) - (omega_2n^i / 2n) tau^(2n-1)]G1, n = 2^power, made by ptau_ref.points_from_scalars (g16_setup);
      its odd entries are also the CircomReduction H query at delta = 1, as a cross-check.
Then: the prepared file round-trips through g16_ptau_read and g16_setup_from_lagrange to the key g16_setup_from_srs makes;
section 7 and unknown ids are kept in input order; an input's sections 12..15 never change the output; every refusal
writes nothing; the resident circuit and key are untouched; Python's out= writes the same bytes."""
import ctypes as C

import numpy as np
import pytest

import ptau_ref as T
import pyref as P
from groth16_b200 import Groth16, _lib
from groth16_b200.api import PolynomialDegreeTooLarge
from groth16_b200.params import GENERATORS
from groth16_b200.serialize import DeserializeError
from groth16_b200.workload import synthetic_r1cs

pytestmark = pytest.mark.gpu

CURVES4 = ["bls12_381", "bn254", "bls12_377", "bw6_761"]
TAU, ALPHA, BETA = 0x1234567890ABCDEF1234567, 0x2222222222222222222223, 0x3333333333333333333335
RHO = 0x5A5A5A5A5A5A5A5A5A5A5A5A5A5A5A5A5
KEY_MEMBERS = ("a_query", "b_g1_query", "b_g2_query", "h_query", "l_query", "beta_g1", "delta_g1")

_ENG = {}
_LEVELS = {}


def engine(curve, qap="libsnark") -> Groth16:
    for key in [k for k in _ENG if k[0] != curve]:
        _ENG.pop(key).close()
    if (curve, qap) not in _ENG:
        _ENG[(curve, qap)] = Groth16(curve, 0, qap=qap)
    return _ENG[(curve, qap)]


@pytest.fixture(scope="module", autouse=True)
def _engines():
    yield
    for g in _ENG.values():
        g.close()
    _ENG.clear()


def gens(curve):
    G = GENERATORS[curve]
    return G["g1"], G["g2"]


def members_of(g, power):
    n = 1 << power
    srs = g.srs_from_secrets(2 * n - 1, n, TAU, ALPHA, BETA, *gens(g.curve.name))
    m = {k: getattr(srs, k) for k in T.MEMBERS}
    m["beta_g2"] = srs.beta_g2
    return m, srs


def ptau_file(g, power, lag=None, **kw):
    """the .ptau of T(TAU, ALPHA, BETA) at `power` (as tests/test_gpu_ptau.py writes it), unprepared without lag"""
    m, srs = members_of(g, power)
    return T.write(g.curve.name, power, m, lag, **kw), srs


def level(curve, k):
    """level k >= 1 of every member (a Lagrange of the library's g16_setup), cached per curve"""
    if (curve, k) not in _LEVELS:
        _LEVELS[(curve, k)] = T.lagrange_from_setup(engine(curve, "libsnark"), engine(curve, "circom"), k, TAU, ALPHA, BETA)
    return _LEVELS[(curve, k)]


def top_level(curve, power):
    """level power + 1 of tauG1 over the 2^(power+1) - 1 powers, by its closed form"""
    g = engine(curve)
    r, n2 = g.curve.r, 2 << power
    lc = T.lagrange_coefficients(curve, power + 1, TAU)
    w = T.root(curve, power + 1)
    c = pow(TAU, n2 - 1, r) * pow(n2, -1, r) % r
    s = [(lc[i] - pow(w, i, r) * c) % r for i in range(n2)]
    return T.points_from_scalars(g, power + 1, s, TAU)


def expected(g, power):
    curve = g.curve.name
    m, _ = members_of(g, power)
    lag = T.empty_lagrange(curve, power)
    T.place_level(lag, 0, {k: m[k][:1] for k in T.MEMBERS})
    for k in range(1, power + 1):
        lv = level(curve, k)
        T.place_level(lag, k, {x: getattr(lv, x) for x in T.MEMBERS})
    top = top_level(curve, power)
    if power >= 1:   # the odd entries are the CircomReduction H query at delta = 1
        assert np.array_equal(top[1::2], level(curve, power).tau_g1_h)
    lag["tau_g1"][T.level_start(power + 1):] = top
    return T.write(curve, power, m, lag)


@pytest.mark.parametrize("power", [0, 1, 2, 5, 8, 12])
@pytest.mark.parametrize("curve", CURVES4)
def test_levels_exact(curve, power):
    if power == 12 and curve not in ("bn254", "bls12_381"):
        pytest.skip("2^12 on BN254 and BLS12-381 only")
    g = engine(curve)
    data, _ = ptau_file(g, power)
    got = g.prepare_ptau(data)
    want = expected(g, power)
    assert len(got) == len(want)
    assert got == want
    assert g.prepare_ptau(data, validate=True) == want
    assert g.prepare_ptau(got) == want   # a prepared input: its sections 12..15 are recomputed
    t = g.timings()
    assert t["total_ms"] > 0 and t["h2d_ms"] > 0 and t["launches"] > 0
    assert t["h2d_bytes"] > 0 and t["d2h_bytes"] > 0
    tm = t["msm_ms"]
    assert tm["h"] > 0 and (power == 0 or min(tm["l"], tm["a"], tm["b_g1"]) > 0) and tm["b_g2"] == 0
    assert t["witness_map_ms"] == 0 and t["host_finish_ms"] == 0
    assert all(v == 0 for d in ("msm_accum_ms", "msm_pairs", "msm_entries", "msm_begin_ms", "msm_end_ms") for v in t[d].values())


def assert_same_key(g, key_a, bytes_a):
    k = g.export_proving_key()
    for name in KEY_MEMBERS:
        assert np.array_equal(getattr(k, name), getattr(key_a, name)), name
    assert g.export_proving_key_bytes(compress=False) == bytes_a


@pytest.mark.parametrize("qap", ["libsnark", "circom"])
@pytest.mark.parametrize("curve", CURVES4)
def test_round_trip(curve, qap):
    power = 6
    g = engine(curve, qap)
    data, _ = ptau_file(g, power)
    prepared = g.prepare_ptau(data)
    for log_n in (power, power - 2):
        m, _, _ = synthetic_r1cs(curve, log_n, seed=600 + log_n)
        p = g.read_ptau(prepared, log_n)
        assert p.prepared and p.lagrange is not None
        g.generate_parameters_from_ptau(m, prepared, rho=RHO, validate=True)   # the Lagrange path and its check
        key, kb = g.export_proving_key(), g.export_proving_key_bytes(compress=False)
        g.generate_parameters_from_srs(None, p.srs)
        assert_same_key(g, key, kb)


def test_sections_kept_in_order():
    g = engine("bn254")
    power = 3
    base = g.prepare_ptau(ptau_file(g, power)[0])
    bs = T.sections(base)
    lag_bytes = b"".join(base[bs[i][0] - 12:bs[i][0] + bs[i][1]] for i in (12, 13, 14, 15))
    extra = [(99, b"\x07" * 21), (8, b"")]
    for order in (None, [6, 7, 2, 1, 5, 3, 4], [7, 1, 2, 3, 4, 5, 6]):
        data, _ = ptau_file(g, power, order=order, extra=extra)
        s = T.sections(data)
        ids = [i for i in (order or [1, 2, 3, 4, 5, 6, 7])] + [99, 8]
        want = b"ptau" + np.array([1, len(ids) + 4], dtype="<u4").tobytes()
        want += b"".join(data[s[i][0] - 12:s[i][0] + s[i][1]] for i in ids) + lag_bytes
        assert g.prepare_ptau(data) == want, order
    # a prepared input whose sections 12..15 hold the identity everywhere, in any order: the unprepared form's output
    m, _ = members_of(g, power)
    zero = T.write("bn254", power, m, T.empty_lagrange("bn254", power))
    assert g.prepare_ptau(zero) == base
    mixed = T.write("bn254", power, m, T.empty_lagrange("bn254", power), order=[15, 1, 13, 2, 3, 12, 4, 5, 14, 6, 7])
    assert g.prepare_ptau(mixed) == base


def raw_prepare(g, data, flags=0, out=None, cap=None):
    """the C call: (rc, *len_out)"""
    n = C.c_uint64(0xDEAD)
    src = np.frombuffer(data, dtype=np.uint8) if isinstance(data, bytes) else data
    optr = None if out is None else out.ctypes.data_as(C.c_void_p)
    rc = g._lib.g16_ptau_prepare(g._ctx, src.ctypes.data_as(C.c_void_p), src.size, flags, optr,
                                 (0 if out is None else out.size) if cap is None else cap, C.byref(n))
    return rc, n.value


def _off_curve(arr, idx):
    arr[idx][-1] ^= np.uint64(1)   # y's top limb: off the curve, still below q


@pytest.mark.parametrize("curve", ["bn254", "bls12_381"])
def test_refusals_write_nothing(curve):
    g = engine(curve)
    power = 4
    m, _ = members_of(g, power)
    good = T.write(curve, power, m)
    size = len(g.prepare_ptau(good))

    def refused(data, exc, match, flags=0):
        out = np.full(size + 64, 0xAB, dtype=np.uint8)
        with pytest.raises(exc, match=match):
            g.prepare_ptau(data, validate=bool(flags), out=out)
        assert (out == 0xAB).all()

    for k in T.MEMBERS:   # a late point of each member, named
        bad = {x: v.copy() for x, v in m.items()}
        idx = len(bad[k]) - 2
        _off_curve(bad[k], idx)
        refused(T.write(curve, power, bad), DeserializeError, rf"^{k}\[{idx}\]: point is not on the curve$")
    # non-canonical: x = q
    bad = {x: v.copy() for x, v in m.items()}
    nq = g.curve.fq_limbs
    bad["alpha_tau_g1"][9][:nq] = [(g.curve.q >> (64 * i)) & ((1 << 64) - 1) for i in range(nq)]
    refused(T.write(curve, power, bad), DeserializeError, r"^alpha_tau_g1\[9\]: non-canonical field element \(>= q\)$")
    # malformed container and header
    refused(good[:-1], DeserializeError, "truncated input")
    refused(T.write(curve, power, m, drop=[4]), DeserializeError, "section 4 is missing")
    # size protocol and argument errors, on the raw call
    rc, n = raw_prepare(g, good)
    assert (rc, n) == (_lib.G16_OK, size)
    out = np.full(size, 0xAB, dtype=np.uint8)
    rc, n = raw_prepare(g, good, out=out, cap=size - 1)
    assert (rc, n) == (_lib.ERR_BAD_ARGUMENT, size) and (out == 0xAB).all()
    assert "needs " + str(size) in _lib.last_error()
    rc, _ = raw_prepare(g, good, flags=0x40, out=out)
    assert rc == _lib.ERR_BAD_ARGUMENT and (out == 0xAB).all()
    both = np.zeros(len(good) + size, dtype=np.uint8)
    both[:len(good)] = np.frombuffer(good, dtype=np.uint8)
    rc = g._lib.g16_ptau_prepare(g._ctx, both.ctypes.data_as(C.c_void_p), len(good), 0,
                                 C.c_void_p(both.ctypes.data + len(good) - 1), size, C.byref(C.c_uint64()))
    assert rc == _lib.ERR_BAD_ARGUMENT and "overlaps" in _lib.last_error()
    assert g._lib.g16_ptau_prepare(g._ctx, None, 0, 0, None, 0, C.byref(C.c_uint64())) == _lib.ERR_BAD_ARGUMENT
    rc, n = raw_prepare(g, good, out=out)
    assert (rc, n) == (_lib.G16_OK, size) and out.tobytes() == g.prepare_ptau(good)


def test_power_above_two_adicity():
    """BN254 at power 28: refused from section 1 alone, before the sections' sizes are compared"""
    g = engine("bn254")
    m, _ = members_of(g, 2)
    data = T.write("bn254", 28, m)
    out = np.full(1024, 0xAB, dtype=np.uint8)
    with pytest.raises(PolynomialDegreeTooLarge, match="two-adicity 28"):
        g.prepare_ptau(data, out=out)
    assert (out == 0xAB).all()
    with pytest.raises(DeserializeError, match="section 2 holds"):   # power 27 is sized as usual
        g.prepare_ptau(T.write("bn254", 27, m))


def test_torsion_point_needs_validate():
    """an on-curve G2 point outside the prime-order subgroup: refused with validate only"""
    curve = "bls12_381"
    g = engine(curve)
    c = P.CURVES[curve]
    Gp = P.ctx(c).G2
    F = Gp.F
    x = F.from_int(1)
    while True:
        y = F.sqrt(F.add(F.mul(F.mul(x, x), x), Gp.b))
        if y is not None:
            break
        x = F.add(x, F.from_int(1))
    assert Gp.mul((x, y), c.r) is not None
    m, _ = members_of(g, 3)
    m["tau_g2"] = m["tau_g2"].copy()
    m["tau_g2"][5] = g.codec.enc_g2([(x, y)])[0]
    data = T.write(curve, 3, m)
    with pytest.raises(DeserializeError, match=r"^tau_g2\[5\]: point is not in the prime-order subgroup$"):
        g.prepare_ptau(data, validate=True)
    assert len(g.prepare_ptau(data)) == len(g.prepare_ptau(T.write(curve, 3, members_of(g, 3)[0])))


def test_resident_state_untouched():
    curve = "bn254"
    g = engine(curve)
    mtx, z, _ = synthetic_r1cs(curve, 6, seed=610)
    g.generate_parameters_with_qap(mtx, ALPHA, BETA, 1, 5, TAU, *gens(curve), export=False)
    prove = lambda: g.create_proof_with_reduction_and_matrices(None, 5, 7, None, mtx.num_instance_variables,
                                                               mtx.num_constraints, z)
    before = prove()
    key = g.export_proving_key_bytes(compress=False)
    g.prepare_ptau(ptau_file(g, 7)[0])
    after = prove()
    assert all(np.array_equal(getattr(before, k), getattr(after, k)) for k in "abc")
    assert g.export_proving_key_bytes(compress=False) == key
    # a proof in flight refuses the call
    r_, s_ = (np.ascontiguousarray(g.codec.fr.enc1(v)) for v in (5, 7))
    g.prove_submit_raw(0, r_, s_, z.ctypes.data, 0)
    try:
        with pytest.raises(ValueError, match="in flight"):
            g.prepare_ptau(ptau_file(g, 2)[0])
    finally:
        out = np.zeros_like(np.concatenate([before.a, before.b, before.c]))
        g.prove_wait_raw(0, out)
    assert np.array_equal(out, np.concatenate([before.a, before.b, before.c]))


def test_out_memmap(tmp_path):
    g = engine("bls12_377")
    data, _ = ptau_file(g, 5)
    want = g.prepare_ptau(data)
    path = tmp_path / "prepared.ptau"
    mm = np.memmap(path, dtype=np.uint8, mode="w+", shape=(len(want),))
    assert g.prepare_ptau(data, out=mm) == len(want)
    mm.flush()
    del mm
    assert path.read_bytes() == want

