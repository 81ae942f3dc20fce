"""CPU tier of the witness check's ABI: g16_witness_report and the constants G16_ERR_UNSATISFIED, G16_CHECK_WITNESS and
G16_NONE agree between include/g16b200.h, groth16_b200/_lib.py and the Rust shim's sys.rs."""
import ctypes
import os
import re

import groth16_b200
from groth16_b200 import _lib
from test_shim_abi import _strip_comments, header_structs, rust_structs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ["first_unsatisfied", "num_unsatisfied", "first_malformed"]


def _read(*parts):
    return open(os.path.join(ROOT, *parts)).read()


def test_witness_report_fields_agree():
    assert header_structs()["g16_witness_report"] == FIELDS
    assert rust_structs()["g16_witness_report"] == FIELDS
    assert [f for f, _ in _lib.WitnessReport._fields_] == FIELDS
    assert all(t is ctypes.c_uint64 for _, t in _lib.WitnessReport._fields_)
    h = _strip_comments(_read("include", "g16b200.h"))
    body = re.search(r"typedef struct\s*\{([^{}]*)\}\s*g16_witness_report\s*;", h, flags=re.S).group(1)
    assert re.findall(r"(\w+)\s+\w+\s*;", body) == ["uint64_t"] * 3
    rs = _strip_comments(_read("shim", "ark-groth16-b200", "src", "sys.rs"))
    body = re.search(r"pub struct g16_witness_report\s*\{(.*?)\}", rs, flags=re.S).group(1)
    assert re.findall(r"pub \w+\s*:\s*(\w+)", body) == ["u64"] * 3


def test_witness_check_constants_agree():
    h = _strip_comments(_read("include", "g16b200.h"))
    rs = _strip_comments(_read("shim", "ark-groth16-b200", "src", "sys.rs"))
    hval = lambda name: int(re.search(rf"\b{name}\s*=\s*(\d+)", h).group(1))
    rval = lambda name: re.search(rf"pub const {name}\s*:\s*\w+\s*=\s*([^;]+);", rs).group(1).strip()
    assert hval("G16_ERR_UNSATISFIED") == _lib.ERR_UNSATISFIED == int(rval("G16_ERR_UNSATISFIED")) == 6
    assert hval("G16_CHECK_WITNESS") == _lib.CHECK_WITNESS == int(rval("G16_CHECK_WITNESS")) == 4
    assert re.search(r"#define\s+G16_NONE\s+UINT64_MAX\b", h)
    assert rval("G16_NONE") == "u64::MAX" and _lib.NONE == (1 << 64) - 1
    # the new flag is its own bit, beside the prover flags it ors with
    assert _lib.CHECK_WITNESS & (_lib.ASSIGNMENT_ON_DEVICE | _lib.SERIAL_MSMS) == 0
    assert groth16_b200.CHECK_WITNESS == _lib.CHECK_WITNESS and groth16_b200.ERR_UNSATISFIED == _lib.ERR_UNSATISFIED
    assert issubclass(groth16_b200.Unsatisfiable, groth16_b200.SynthesisError)


def test_unsatisfied_status_maps_to_unsatisfiable(monkeypatch):
    from groth16_b200 import api
    monkeypatch.setattr(_lib, "last_error", lambda: "constraint 3 unsatisfied (1 in all)")
    try:
        api._check(_lib.ERR_UNSATISFIED)
    except groth16_b200.Unsatisfiable as e:
        assert str(e) == "constraint 3 unsatisfied (1 in all)"
    else:
        raise AssertionError("ERR_UNSATISFIED did not raise")
    # the shim maps the code explicitly, not through its catch-all arm
    lib_rs = _read("shim", "ark-groth16-b200", "src", "lib.rs")
    assert re.search(r"sys::G16_ERR_UNSATISFIED\s*=>", lib_rs)
    for fn in ("pub fn is_satisfied", "pub fn which_is_unsatisfied", "pub fn check_witness", "pub fn set_check_witness"):
        assert fn in lib_rs, fn
