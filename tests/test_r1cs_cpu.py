"""CPU tier of the .r1cs / .wtns format restatement (tests/r1cs_ref.py), pinned to pyref: writing a circuit (from pyref's
R1CS or from ConstraintMatrices) and reading the file back returns the same constraints with ark-circom's sizes, whatever
the section order, unknown sections, split terms or zero coefficients; the read-back circuit is satisfied by the witness
read back from its .wtns.  PARITY UNPINNED BY CIRCOM: no circom-made file is available."""
import pytest

import pyref as P
import r1cs_ref as R
from groth16_b200 import get_curve
from util import matrices_from_r1cs


def circuits(c):
    rng = P.Rng(3)
    yield "silly", P.silly_circuit(c, 3, 11)
    yield "mimc", P.mimc_circuit(c, rng.fr(c.r), rng.fr(c.r), [rng.fr(c.r) for _ in range(6)])
    yield "npub0", P.synthetic_circuit(c, 5, seed=7, num_inputs=0)
    yield "2^5", P.synthetic_circuit(c, 30, seed=5, num_inputs=2)


def _canon(c: R.Circuit):
    """per constraint and matrix: {wire: sum of coefficients} without zeros, an order-free view"""
    r = c.cp.r
    out = []
    for row in c.rows():
        rr = []
        for comb in row:
            d = {}
            for w, cf in comb:
                d[w] = (d.get(w, 0) + cf) % r
            rr.append({k: v for k, v in d.items() if v})
        out.append(rr)
    return out


@pytest.mark.parametrize("curve", list(P.CURVES))
def test_roundtrip(curve):
    c = P.CURVES[curve]
    for name, cs in circuits(c):
        assert cs.is_satisfied()
        base = R.Circuit.from_r1cs(cs)
        via_m = R.Circuit.from_matrices(curve, matrices_from_r1cs(cs))
        assert _canon(via_m) == _canon(base), name
        for cc in (base, base.transformed(split_seed=1), base.transformed(zero_seed=2), base.transformed(long_row=(1, 9))):
            assert _canon(cc) == _canon(base), name
            for kw in ({}, {"order": [3, 2, 1]}, {"extra": [(9, b"junk"), (0, b"")]}, {"npubin": min(1, cs.num_instance - 1)}):
                data = R.write(cc, **kw)
                h = R.header(data)
                back = R.read(curve, data)
                # ark-circom's sizes: num_inputs = 1 + nPubOut + nPubIn, num_witness = nWires - num_inputs
                assert (1 + h["npubout"] + h["npubin"], h["nwires"] - 1 - h["npubout"] - h["npubin"], h["m"]) == \
                    (cs.num_instance, cs.num_witness, cs.num_constraints), (name, kw)
                assert (back.ni, back.nw, back.m) == (cs.num_instance, cs.num_witness, cs.num_constraints)
                assert back.rows() == cc.rows(), (name, kw)   # terms exactly as written, in file order
                z = R.read_wtns(curve, R.write_wtns(curve, cs.assignment))
                assert z == [v % c.r for v in cs.assignment]
                assert R.satisfied(back, z), (name, kw)


@pytest.mark.parametrize("curve", list(P.CURVES))
def test_matrices_roundtrip(curve):
    """to_matrices gives the ABI's ConstraintMatrices of the file's terms, in file order"""
    c = P.CURVES[curve]
    cs = P.silly_circuit(c, 5, 7)
    m = matrices_from_r1cs(cs)
    back = R.read(curve, R.write(R.Circuit.from_matrices(curve, m))).to_matrices()
    for k in ("a", "b", "c"):
        for x, y in zip(getattr(back, k), getattr(m, k)):
            assert (x == y).all(), k
    assert (back.num_instance_variables, back.num_witness_variables, back.num_constraints) == \
        (m.num_instance_variables, m.num_witness_variables, m.num_constraints)


def test_header_fields():
    c = P.CURVES["bn254"]
    cs = P.silly_circuit(c, 3, 11)
    data = R.write(R.Circuit.from_r1cs(cs))
    h = R.header(data)
    assert (h["n8"], h["prime"], h["nwires"], h["npubout"], h["npubin"], h["nprvin"], h["nlabels"], h["m"]) == \
        (32, get_curve("bn254").r, 4, 1, 0, 2, 4, cs.num_constraints)
    assert sorted(R.sections(data)) == [1, 2, 3]
