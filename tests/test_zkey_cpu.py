"""CPU tier of the .zkey format restatement (tests/zkey_ref.py), pinned to pyref: writing a CircomReduction key and its
circuit and reading the file back returns the same matrices and key, whatever the record order, section order, split
records or trailing section 10, and a proof under the read key verifies by pyref's pairing while a wrong public input does
not.  BN254 and BLS12-381, the curves snarkjs writes.  PARITY UNPINNED BY SNARKJS: no snarkjs-made file is available."""
import numpy as np
import pytest

import pyref as P
import qap_circom_ref as Q
import zkey_ref as Z
from util import matrices_from_r1cs, pk_from_abi, pk_to_abi

TOXIC = (0x1234567, 0x2345678, 0x3456789, 0x456789A, 0x56789AB)


def circuits(c):
    rng = P.Rng(3)
    yield "silly", P.silly_circuit(c, 3, 11)
    yield "mimc", P.mimc_circuit(c, rng.fr(c.r), rng.fr(c.r), [rng.fr(c.r) for _ in range(6)])
    yield "npub0", P.synthetic_circuit(c, 5, seed=7, num_inputs=0)
    for log_n in (4, 6):
        yield f"2^{log_n}", P.synthetic_circuit(c, (1 << log_n) - 2, seed=log_n, num_inputs=1)


def _same_key(a, b):
    for name in ("beta_g1", "delta_g1", "a_query", "b_g1_query", "b_g2_query", "h_query", "l_query"):
        assert np.array_equal(np.asarray(getattr(a, name)), np.asarray(getattr(b, name))), name
    for name in ("alpha_g1", "beta_g2", "gamma_g2", "delta_g2", "gamma_abc_g1"):
        assert np.array_equal(np.asarray(getattr(a.vk, name)), np.asarray(getattr(b.vk, name))), name


@pytest.mark.parametrize("curve", Z.SNARKJS_CURVES)
def test_write_read_roundtrip(curve):
    c = P.CURVES[curve]
    for name, cs in circuits(c):
        if name.startswith("2^6") and curve == "bls12_381":
            continue   # the pure-Python setup of the larger circuit is the slow part; one curve covers it
        m = matrices_from_r1cs(cs)
        pk = pk_to_abi(Q.generate_parameters(cs, *TOXIC, qap="circom"))
        base = None
        for kw in ({}, {"shuffle_seed": 1}, {"order": [9, 3, 1, 7, 5, 2, 8, 4, 6]}, {"split_seed": 2}, {"junk10": b"\x07" * 40}):
            m2, pk2 = Z.read(curve, Z.write(curve, m, pk, **kw))
            assert (m2.num_instance_variables, m2.num_witness_variables, m2.num_constraints) == \
                (m.num_instance_variables, m.num_witness_variables, m.num_constraints), (name, kw)
            for which in ("a", "b"):
                assert Z.canonical_rows(m2, which, c.r) == Z.canonical_rows(m, which, c.r), (name, kw, which)
            assert int(m2.c[0][-1]) == 0
            _same_key(pk2, pk)
            if base is None:
                base = (m2, pk2)


@pytest.mark.parametrize("curve", Z.SNARKJS_CURVES)
def test_proof_under_the_read_key_verifies(curve):
    c = P.CURVES[curve]
    cs = P.silly_circuit(c, 5, 9)
    opk = Q.generate_parameters(cs, *TOXIC, qap="circom")
    m = matrices_from_r1cs(cs)
    _, pk2 = Z.read(curve, Z.write(curve, m, pk_to_abi(opk), shuffle_seed=5))
    rpk = pk_from_abi(curve, pk2)
    proof = Q.create_proof(rpk, cs, 77, 88, qap="circom")
    pub = cs.assignment[1:cs.num_instance]
    assert P.verify_proof(rpk.vk, c, proof, pub)
    assert not P.verify_proof(rpk.vk, c, proof, [(pub[0] + 1) % c.r])


def test_header_fields():
    c = P.CURVES["bn254"]
    cs = P.silly_circuit(c, 3, 11)
    m = matrices_from_r1cs(cs)
    data = Z.write("bn254", m, pk_to_abi(Q.generate_parameters(cs, *TOXIC, qap="circom")))
    h = Z.header(data)
    assert (h["n8q"], h["n8r"], h["q"], h["r"]) == (32, 32, c.q, c.r)
    assert (h["nvars"], h["npub"], h["domain_size"]) == (4, 1, 8)
    assert sorted(Z.sections(data)) == list(range(1, 10))
