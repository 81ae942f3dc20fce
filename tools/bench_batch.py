#!/usr/bin/env python3
"""bench_batch.py -- throughput of batch proving (g16_prove_batch) against the two-slot pipelined single-proof loop
(g16_prove_submit / g16_prove_wait) on the same inputs, for small synthetic circuits.

  python tools/bench_batch.py [--curve bls12_381] [--log-n 10 12 14 16] [--count 1 16 64 256] [--seconds 1] [--json FILE]

For every (log n, count): one key (GPU setup), `count` proofs with distinct r, s and assignments, one warm-up of each arm,
then the two arms alternate until each has run at least --seconds.  Every proof of both arms must be byte-equal.  Reported per
shape: proofs/s of each arm, kernel launches per proof and the host tail (host time after the GPU work: for the batch,
g16_get_timings' host_finish_ms of the whole call, i.e. the tail of its last group; for the loop, the mean per proof).
The card name, power limit and maximum SM clock come from a read-only `nvidia-smi --query-gpu` in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from groth16_b200 import Groth16  # noqa: E402
from groth16_b200.params import GENERATORS  # noqa: E402
from groth16_b200.workload import synthetic_r1cs  # noqa: E402

TOXIC = (0x1111111111111111111111, 0x2222222222222222222223, 0x3333333333333333333335, 0x4444444444444444444447,
         0x5555555555555555555559)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [x.strip() for x in out[0].split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:   # noqa: BLE001 -- the numbers are still worth printing without the card's description
        return dict(error=str(e))


def random_fr(rng, shape):
    """uniform-ish Montgomery limbs below 2^252 (every such value is a field element of all three scalar fields)"""
    x = rng.integers(0, 1 << 63, size=shape + (4,), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=shape + (4,), dtype=np.uint64)
    x[..., 3] &= np.uint64((1 << 60) - 1)
    return np.ascontiguousarray(x)


def run_shape(curve, log_n, count, seconds, rng):
    g = Groth16(curve, 0)
    try:
        G = GENERATORS[curve]
        m, z0, _ = synthetic_r1cs(curve, log_n, seed=log_n)
        g.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=False)
        nv = m.num_instance_variables + m.num_witness_variables
        r, s = random_fr(rng, (count,)), random_fr(rng, (count,))
        z = random_fr(rng, (count, nv))
        z[:, 0] = z0[0]   # the constant One
        nq = g.nq
        out_b = np.zeros((count, 8 * nq), dtype=np.uint64)
        out_p = np.zeros((count, 8 * nq), dtype=np.uint64)
        rows = [(np.ascontiguousarray(r[k]), np.ascontiguousarray(s[k]), np.ascontiguousarray(z[k])) for k in range(count)]

        def batch():
            g.prove_batch_raw(count, r, s, z.ctypes.data, 0, 0, out_b)
            t = g.timings()
            return t["launches"], t["host_finish_ms"]

        def pipelined():
            launches, host = 0, 0.0
            for k in range(count + 1):   # proof k is submitted before proof k - 1 is waited for
                if k < count:
                    g.prove_submit_raw(k & 1, rows[k][0], rows[k][1], rows[k][2].ctypes.data, 0)
                if k >= 1:
                    g.prove_wait_raw((k - 1) & 1, out_p[k - 1])
                    t = g.timings()
                    launches += t["launches"]
                    host += t["host_finish_ms"]
            return launches, host

        lb, hb = batch()
        lp, hp = pipelined()
        assert np.array_equal(out_b, out_p), f"{curve} 2^{log_n} x {count}: batch and single proofs differ"
        tb = tp = 0.0
        nb = np_ = 0
        while tb < seconds or tp < seconds:
            t0 = time.perf_counter()
            lb, hb = batch()
            tb += time.perf_counter() - t0
            nb += 1
            t0 = time.perf_counter()
            lp, hp = pipelined()
            tp += time.perf_counter() - t0
            np_ += 1
        assert np.array_equal(out_b, out_p), f"{curve} 2^{log_n} x {count}: batch and single proofs differ"
        return dict(curve=curve, log_n=log_n, count=count, batch_proofs_per_s=count * nb / tb,
                    pipelined_proofs_per_s=count * np_ / tp, speedup=(count * nb / tb) / (count * np_ / tp),
                    batch_launches_per_proof=lb / count, pipelined_launches_per_proof=lp / count,
                    batch_host_tail_ms_call=hb, pipelined_host_tail_ms_per_proof=hp / count)
    finally:
        g.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curve", default="bls12_381", choices=["bls12_381", "bn254", "bls12_377"])
    ap.add_argument("--log-n", type=int, nargs="+", default=[10, 12, 14, 16])
    ap.add_argument("--count", type=int, nargs="+", default=[1, 16, 64, 256])
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    rng = np.random.default_rng(1)
    info = gpu_info()
    print(json.dumps(dict(gpu=info)), flush=True)
    res = []
    print(f"{'log n':>5} {'count':>5} {'batch/s':>10} {'pipelined/s':>12} {'speedup':>8} {'launch/pf b':>11} {'launch/pf p':>11} "
          f"{'host tail ms (b, call)':>22} {'host tail ms/pf (p)':>19}", flush=True)
    for log_n in a.log_n:
        for count in a.count:
            x = run_shape(a.curve, log_n, count, a.seconds, rng)
            res.append(x)
            print(f"{log_n:>5} {count:>5} {x['batch_proofs_per_s']:>10.1f} {x['pipelined_proofs_per_s']:>12.1f} {x['speedup']:>8.2f} "
                  f"{x['batch_launches_per_proof']:>11.2f} {x['pipelined_launches_per_proof']:>11.2f} "
                  f"{x['batch_host_tail_ms_call']:>22.2f} {x['pipelined_host_tail_ms_per_proof']:>19.3f}", flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(gpu=info, results=res), f, indent=1)


if __name__ == "__main__":
    main()
