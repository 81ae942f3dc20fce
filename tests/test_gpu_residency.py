"""What a context holds resident across loads: a rejected circuit or key leaves the previous one proving as before, and
loading a circuit or key discards everything derived from the previous key (here the products of
g16_prove_assemble_prepare).  Every proof is checked against g16_prove under the intended key and the CPU oracle."""
import ctypes as C
import dataclasses
import random

import numpy as np
import pytest

import orc
from groth16_b200 import Groth16, MalformedKey, _lib
from groth16_b200.api import _check, _ptr, _u64p
from groth16_b200.params import GENERATORS
from groth16_b200.workload import synthetic_r1cs

pytestmark = pytest.mark.gpu

LOG_N = 8
TOXIC1 = (0x1111111111111111111111, 0x2222222222222222222223, 0x3333333333333333333335, 0x4444444444444444444447,
          0x5555555555555555555559)
TOXIC2 = (0x6666666666666666666661, 0x7777777777777777777773, 0x8888888888888888888885, 0x9999999999999999999997,
          0xAAAAAAAAAAAAAAAAAAAAA9)
THREADS = 8

_ENGINES = {}


def engine(curve) -> Groth16:
    if curve not in _ENGINES:
        _ENGINES[curve] = Groth16(curve, 0)
    return _ENGINES[curve]


@pytest.fixture(scope="module", autouse=True)
def _engines():
    yield
    for g in _ENGINES.values():
        g.close()
    _ENGINES.clear()


def _rs(g, seed):
    rng = random.Random(seed)
    return tuple(np.ascontiguousarray(g.codec.fr.enc1(rng.randrange(1, g.curve.r))) for _ in range(2))


def _prove(g, r, s, z):
    """g16_prove on the resident circuit and key"""
    out = np.zeros(4 * g.nq + g.ng2, dtype=np.uint64)
    g.prove_raw(r, s, np.ascontiguousarray(z).ctypes.data, 0, out)
    return out


def _oracle(g, pk, m, z, r, s):
    return orc.prove(g.curve.cid, g.nq, pk, m, z, r, s, threads=THREADS)[0]


def _setup_only(g, toxic):
    """g16_setup on the resident circuit (generate_parameters_with_qap loads the circuit first); returns the exported key"""
    G = GENERATORS[g.curve.name]
    cd = g.codec
    sc = [np.ascontiguousarray(cd.fr.enc1(x)) for x in toxic]
    g1 = np.ascontiguousarray(cd.enc_g1([G["g1"]])[0])
    g2 = np.ascontiguousarray(cd.enc_g2([G["g2"]])[0])
    _check(g._lib.g16_setup(g._ctx, *[_ptr(x) for x in sc], _ptr(g1), _ptr(g2)))
    return g.export_proving_key()


@pytest.mark.parametrize("bad", ["c_column", "b_row_ptr"])
@pytest.mark.parametrize("curve", ["bn254", "bls12_381"])
def test_rejected_circuit_keeps_the_resident_one(curve, bad):
    """A circuit of the same shape with other A and B and one bad matrix (a column out of range in C, or a decreasing
    row_ptr in B) is rejected before any of its matrices replaces the resident circuit: proving again gives the first
    proof."""
    g = engine(curve)
    G = GENERATORS[curve]
    m1, z1, _ = synthetic_r1cs(curve, LOG_N, seed=1)
    pk1 = g.generate_parameters_with_qap(m1, *TOXIC1, G["g1"], G["g2"])
    r, s = _rs(g, 1)
    first = _prove(g, r, s, z1)
    assert np.array_equal(first, _oracle(g, pk1, m1, z1, r, s))
    m2, _, _ = synthetic_r1cs(curve, LOG_N, seed=2)
    shape = lambda m: (m.num_instance_variables, m.num_witness_variables, m.num_constraints)
    assert shape(m2) == shape(m1)
    assert not np.array_equal(m2.a[1], m1.a[1]) and not np.array_equal(m2.b[1], m1.b[1])
    if bad == "c_column":
        col = m2.c[1].copy()
        col[len(col) // 2] = m2.num_instance_variables + m2.num_witness_variables
        m2 = dataclasses.replace(m2, c=(m2.c[0], col, m2.c[2]))
    else:
        rp = m2.b[0].copy()
        rp[len(rp) // 2] = rp[len(rp) // 2 - 1] - 1
        m2 = dataclasses.replace(m2, b=(rp, m2.b[1], m2.b[2]))
    with pytest.raises(ValueError, match="out of range" if bad == "c_column" else "non-decreasing"):
        g.load_matrices(m2)
    assert np.array_equal(_prove(g, r, s, z1), first)


@pytest.mark.parametrize("how", ["setup", "pk_load", "pk_load_serialized", "circuit"])
def test_prepared_products_are_dropped_with_the_key(how):
    """g16_prove_assemble_prepare(r, s) under key 1, then key 2 made resident (by g16_setup with other toxic waste,
    g16_pk_load, g16_pk_load_serialized, or with a new circuit): g16_prove_partial + g16_prove_assemble(r, s) prove under
    key 2, not with key 1's products."""
    curve = "bn254"
    g = engine(curve)
    G = GENERATORS[curve]
    m, z, _ = synthetic_r1cs(curve, LOG_N, seed=3)
    pk2 = g.generate_parameters_with_qap(m, *TOXIC2, G["g1"], G["g2"])
    pk2_bytes = g.export_proving_key_bytes()
    g.generate_parameters_with_qap(m, *TOXIC1, G["g1"], G["g2"])
    r, s = _rs(g, 2)
    g.prove_assemble_prepare(r, s)
    if how == "setup":
        pk2 = _setup_only(g, TOXIC2)
    elif how == "pk_load":
        g.load_proving_key(pk2)
    elif how == "pk_load_serialized":
        g.load_proving_key_bytes(pk2_bytes)
    else:
        m, z, _ = synthetic_r1cs(curve, LOG_N, seed=4)
        pk2 = g.generate_parameters_with_qap(m, *TOXIC2, G["g1"], G["g2"])
    part = np.zeros(g.partial_limbs(), dtype=np.uint64)
    g.prove_partial_raw(r, np.ascontiguousarray(z).ctypes.data, 0, part)
    pf = g.prove_assemble(r, s, part[None])
    got = np.concatenate([pf.a, pf.b, pf.c])
    assert np.array_equal(got, _prove(g, r, s, z))
    assert np.array_equal(got, _oracle(g, pk2, m, z, r, s))


def test_malformed_key_keeps_the_resident_one():
    """g16_pk_load with an empty a_query is G16_ERR_MALFORMED_KEY, found before the resident key is released."""
    curve = "bn254"
    g = engine(curve)
    G = GENERATORS[curve]
    m, z, _ = synthetic_r1cs(curve, LOG_N, seed=5)
    other = g.generate_parameters_with_qap(m, *TOXIC2, G["g1"], G["g2"])
    pk = g.generate_parameters_with_qap(m, *TOXIC1, G["g1"], G["g2"])
    r, s = _rs(g, 3)
    first = _prove(g, r, s, z)
    assert np.array_equal(first, _oracle(g, pk, m, z, r, s))
    # what g.load_proving_key(other) passes, but with a_len = 0 over a non-null a_query (the wrapper passes NULL when empty)
    d = _lib.PkDesc()
    keep = []
    for name in ("a_query", "b_g1_query", "b_g2_query", "h_query", "l_query"):
        arr = np.ascontiguousarray(getattr(other, name), dtype=np.uint64)
        keep.append(arr)
        setattr(d, name, _u64p(arr))
        setattr(d, name.replace("_query", "_len"), arr.reshape(-1, g.ng2 if name == "b_g2_query" else 2 * g.nq).shape[0])
    d.a_len = 0
    for k, v in dict(alpha_g1=other.vk.alpha_g1, beta_g1=other.beta_g1, delta_g1=other.delta_g1, beta_g2=other.vk.beta_g2,
                     delta_g2=other.vk.delta_g2).items():
        keep.append(np.ascontiguousarray(v, dtype=np.uint64))
        setattr(d, k, _u64p(keep[-1]))
    with pytest.raises(MalformedKey):
        _check(g._lib.g16_pk_load(g._ctx, C.byref(d), 0, 1))
    assert np.array_equal(_prove(g, r, s, z), first)
