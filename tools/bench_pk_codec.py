#!/usr/bin/env python3
"""bench_pk_codec.py -- ark-serialized proving keys on the GPU: g16_pk_load_serialized against g16_pk_load of the same key
from limbs, and g16_pk_export_serialized, on 2^20-constraint synthetic keys.

  python tools/bench_pk_codec.py [--curve bls12_381 bn254 bls12_377] [--log-n 20] [--repeat 3] [--json FILE]

Per curve: one g16_setup, the key exported as limbs and in both encodings, then --repeat rounds that each time, in this
order, g16_pk_load of the limbs and g16_pk_load_serialized in {compressed, uncompressed} x {validate, not}.  A call is timed
with the host clock; each ends in a device synchronise.  Reported: the median and the spread (min .. max) over rounds,
points/s (all points of the key over the median), and g16_pk_export_serialized per encoding.  The card name, power limit
and maximum SM clock come from a read-only `nvidia-smi --query-gpu` in the same run."""
import argparse
import json
import os
import statistics
import sys
import time

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batch import TOXIC, gpu_info  # noqa: E402
from groth16_b200 import Groth16  # noqa: E402
from groth16_b200.params import GENERATORS  # noqa: E402
from groth16_b200.workload import synthetic_r1cs  # noqa: E402


def timed(fn):
    t = time.perf_counter()
    out = fn()
    return time.perf_counter() - t, out


def summary(xs):
    return {"median_s": statistics.median(xs), "min_s": min(xs), "max_s": max(xs)}


def run_curve(curve, log_n, repeat):
    g = Groth16(curve, 0)
    m, _, _ = synthetic_r1cs(curve, log_n, seed=1)
    G = GENERATORS[curve]
    pk = g.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=True)
    npts = 6 + sum(x.shape[0] for x in (pk.a_query, pk.b_g1_query, pk.b_g2_query, pk.h_query, pk.l_query, pk.vk.gamma_abc_g1))
    out = {"curve": curve, "log_n": log_n, "points": npts, "export": {}, "load": {}}
    blobs = {}
    for cp in (True, False):
        secs = [timed(lambda: g.export_proving_key_bytes(cp))[0] for _ in range(repeat)]
        blobs[cp] = g.export_proving_key_bytes(cp)
        out["export"]["compressed" if cp else "uncompressed"] = dict(summary(secs), bytes=len(blobs[cp]),
                                                                     points_per_s=npts / statistics.median(secs))
    g.load_proving_key_bytes(blobs[True], compress=True, validate=False)   # warm-up: module loads, first allocations
    modes = [("limbs", None, None)] + [(f"{'compressed' if cp else 'uncompressed'}{'+validate' if v else ''}", cp, v)
                                       for cp in (True, False) for v in (False, True)]
    secs = {name: [] for name, _, _ in modes}
    for _ in range(repeat):
        for name, cp, v in modes:
            if cp is None:
                secs[name].append(timed(lambda: g.load_proving_key(pk))[0])
            else:
                secs[name].append(timed(lambda: g.load_proving_key_bytes(blobs[cp], compress=cp, validate=v))[0])
    for name, _, _ in modes:
        out["load"][name] = dict(summary(secs[name]), points_per_s=npts / statistics.median(secs[name]))
    g.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curve", nargs="+", default=["bls12_381", "bn254", "bls12_377"])
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    res = {"gpu": gpu_info(), "rows": []}
    for curve in a.curve:
        row = run_curve(curve, a.log_n, a.repeat)
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"gpu": res["gpu"]}))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
