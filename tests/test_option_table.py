"""The tuning options are listed in three places that users and the engine read: the engine's option table
(groth16_b200/csrc/engine.cuh, which g16_set_option, g16_get_option and g16_ctx_create's environment reading all loop
over), the comment above g16_set_option in include/g16b200.h, and the table of INTEGRATION.md section 6.  They must name
the same options."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _read(*path):
    with open(os.path.join(ROOT, *path)) as f:
        return f.read()


def _engine_options():
    return set(re.findall(r'\{"(\w+)", &Tune::', _read("groth16_b200", "csrc", "engine.cuh")))


def _header_options():
    h = _read("include", "g16b200.h")
    block = h[h.index("/* Tuning options"):h.index("int g16_set_option(")]
    return set(re.findall(r'"(\w+)"', block))


def _integration_options():
    doc = _read("INTEGRATION.md")
    section = re.search(r"^## 6\..*?(?=^## |\Z)", doc, re.M | re.S).group(0)
    names = set()
    for row in re.findall(r"^\| (`[^|]+) \|", section, re.M):
        names |= set(re.findall(r"`(\w+)`", row))
    return names


def test_option_lists_agree():
    engine = _engine_options()
    assert len(engine) == 18, sorted(engine)
    assert _header_options() == engine
    assert _integration_options() == engine
