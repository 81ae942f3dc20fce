#!/usr/bin/env python3
"""bench_qap.py -- the two R1CS-to-QAP reductions side by side: LibsnarkReduction (7 transforms + a fused (ab - c)/Z) and
CircomReduction (6 transforms, c = a o b and A B - C fused into loads / stores), on the same synthetic circuit and key.

  python tools/bench_qap.py [--curve bls12_381 bn254] [--log-n 20] [--rounds 5] [--proofs 20] [--json FILE]

Per curve: one context per reduction, both set up with the same toxic waste, so the satisfying witness gives the same proof
bytes under both (checked).  Then --rounds rounds alternate the two reductions; each round measures, per reduction:
  witness_map_ms   g16_get_timings' witness_map_ms (row evaluation + transforms) of a proof with G16_SERIAL_MSMS, so that no
                   MSM shares the GPU with the witness map; median over --proofs proofs
  latency_ms       host wall time of one g16_prove (upload to proof), median over --proofs proofs
  proofs_per_s     --proofs proofs with two in flight (g16_prove_submit / g16_prove_wait over the two slots)
Reported: the median over rounds of each figure, and the spread (min .. max) of the rounds.  The card name, power limit and
maximum SM clock come from a read-only `nvidia-smi --query-gpu` in the same run."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batch import TOXIC, gpu_info  # noqa: E402
from groth16_b200 import Groth16, _lib  # noqa: E402
from groth16_b200.params import GENERATORS  # noqa: E402
from groth16_b200.workload import synthetic_r1cs  # noqa: E402

QAPS = ("libsnark", "circom")


def measure(g, m, z, r, s, proofs):
    nq = g.nq
    out = np.zeros(8 * nq, dtype=np.uint64)
    zp = z.ctypes.data
    wm, lat = [], []
    for _ in range(proofs):
        g.prove_raw(r, s, zp, _lib.SERIAL_MSMS, out)
        wm.append(g.timings()["witness_map_ms"])
    for _ in range(proofs):
        t0 = time.perf_counter()
        g.prove_raw(r, s, zp, 0, out)
        lat.append((time.perf_counter() - t0) * 1e3)
    outs = [np.zeros(8 * nq, dtype=np.uint64) for _ in range(2)]
    t0 = time.perf_counter()
    for k in range(proofs + 1):   # proof k is submitted before proof k - 1 is waited for
        if k < proofs:
            g.prove_submit_raw(k & 1, r, s, zp, 0)
        if k >= 1:
            g.prove_wait_raw((k - 1) & 1, outs[(k - 1) & 1])
    pps = proofs / (time.perf_counter() - t0)
    return dict(witness_map_ms=statistics.median(wm), latency_ms=statistics.median(lat), proofs_per_s=pps), out


def run_curve(curve, log_n, rounds, proofs):
    m, z, _ = synthetic_r1cs(curve, log_n, seed=log_n)
    G = GENERATORS[curve]
    gs = {q: Groth16(curve, 0, qap=q) for q in QAPS}
    try:
        for g in gs.values():
            g.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=False)
        cd = gs["libsnark"].codec
        r, s = np.ascontiguousarray(cd.fr.enc1(123456789)), np.ascontiguousarray(cd.fr.enc1(987654321))
        per = {q: [] for q in QAPS}
        proof = {}
        for q in QAPS:   # warm-up of every path the rounds time
            measure(gs[q], m, z, r, s, 2)
        for _ in range(rounds):
            for q in QAPS:
                x, proof[q] = measure(gs[q], m, z, r, s, proofs)
                per[q].append(x)
        assert np.array_equal(proof["libsnark"], proof["circom"]), f"{curve}: the two reductions' proofs differ"
        res = dict(curve=curve, log_n=log_n, rounds=rounds, proofs=proofs)
        for q in QAPS:
            for k in ("witness_map_ms", "latency_ms", "proofs_per_s"):
                v = [x[k] for x in per[q]]
                res[f"{q}_{k}"] = statistics.median(v)
                res[f"{q}_{k}_range"] = [min(v), max(v)]
        return res
    finally:
        for g in gs.values():
            g.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curve", nargs="+", default=["bls12_381", "bn254"], choices=["bls12_381", "bn254", "bls12_377"])
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--proofs", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    info = gpu_info()
    print(json.dumps(dict(gpu=info)), flush=True)
    res = []
    for curve in a.curve:
        x = run_curve(curve, a.log_n, a.rounds, a.proofs)
        res.append(x)
        print(json.dumps(x), flush=True)
        for q in QAPS:
            print(f"{curve:>9} 2^{a.log_n} {q:>8}: witness map {x[f'{q}_witness_map_ms']:.3f} ms, one proof "
                  f"{x[f'{q}_latency_ms']:.2f} ms, two in flight {x[f'{q}_proofs_per_s']:.1f} proofs/s", flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(gpu=info, results=res), f, indent=1)


if __name__ == "__main__":
    main()
