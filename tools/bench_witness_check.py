#!/usr/bin/env python3
"""Cost of the witness check (g16_check_witness and the G16_CHECK_WITNESS prover flag) on the synthetic circuit: per curve,

  * check_ms: one g16_check_witness of a device-resident assignment, synchronised after every call (median, min, max of
    --calls calls after --warmup);
  * proofs/s of the two-slot pipelined loop (g16_prove_submit / g16_prove_wait, host assignment) without and with the flag,
    alternated --reps times in the same run; every proof must equal the first one.

Prints the card (name, power limit, max SM clock, read with nvidia-smi in the same run) and one JSON line per curve.

  python tools/bench_witness_check.py [--curves bls12_381 bn254 bls12_377 bw6_761] [--log-n 20] [--steps 20] [--reps 3]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from groth16_b200 import CHECK_WITNESS, Groth16, _lib  # noqa: E402
from groth16_b200.params import GENERATORS  # noqa: E402
from groth16_b200.workload import synthetic_r1cs  # noqa: E402

TOXIC = (11, 22, 33, 44, 55)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # report, do not guess
        return f"nvidia-smi unavailable: {e}"


def pipelined(g, r, s, z, flags, steps, nout, want):
    outs = [np.zeros(nout, dtype=np.uint64) for _ in range(2)]
    t = time.perf_counter()
    g.prove_submit_raw(0, r, s, z.ctypes.data, flags)
    for i in range(1, steps):
        g.prove_submit_raw(i & 1, r, s, z.ctypes.data, flags)
        g.prove_wait_raw((i - 1) & 1, outs[(i - 1) & 1])
        assert np.array_equal(outs[(i - 1) & 1], want)
    g.prove_wait_raw((steps - 1) & 1, outs[(steps - 1) & 1])
    dt = time.perf_counter() - t
    assert np.array_equal(outs[(steps - 1) & 1], want)
    return steps / dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", nargs="+", default=["bls12_381", "bn254", "bls12_377", "bw6_761"])
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import torch
    print(json.dumps({"card": card()}), flush=True)
    for curve in a.curves:
        g = Groth16(curve, 0)
        G = GENERATORS[curve]
        m, z, _ = synthetic_r1cs(curve, a.log_n, seed=1)
        g.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=False)
        # g16_check_witness on a device-resident assignment
        dz = torch.from_numpy(z.view(np.int64).reshape(-1)).to("cuda:0")
        torch.cuda.synchronize()
        for _ in range(a.warmup):
            assert g.check_witness(dz.data_ptr(), count=1, flags=_lib.ASSIGNMENT_ON_DEVICE)[0].ok
        ts = []
        for _ in range(a.calls):
            t = time.perf_counter()
            g.check_witness(dz.data_ptr(), count=1, flags=_lib.ASSIGNMENT_ON_DEVICE)
            ts.append(1e3 * (time.perf_counter() - t))
        # pipelined proving with and without the flag, alternated
        r = np.ascontiguousarray(g.codec.fr.enc1(123456789))
        s = np.ascontiguousarray(g.codec.fr.enc1(987654321))
        nout = 4 * g.nq + g.ng2
        want = np.zeros(nout, dtype=np.uint64)
        g.prove_raw(r, s, z.ctypes.data, 0, want)
        for flags in (0, CHECK_WITNESS):   # warm-up of both slots, both ways
            pipelined(g, r, s, z, flags, 4, nout, want)
        rates = {0: [], CHECK_WITNESS: []}
        for _ in range(a.reps):
            for flags in (0, CHECK_WITNESS):
                rates[flags].append(pipelined(g, r, s, z, flags, a.steps, nout, want))
        off, on = float(np.median(rates[0])), float(np.median(rates[CHECK_WITNESS]))
        print(json.dumps({
            "curve": curve, "log_n": a.log_n, "constraints": m.num_constraints,
            "check_ms": {"median": round(float(np.median(ts)), 3), "min": round(min(ts), 3), "max": round(max(ts), 3)},
            "proofs_per_sec": {"without_flag": round(off, 3), "with_flag": round(on, 3),
                               "all_without": [round(x, 3) for x in rates[0]],
                               "all_with": [round(x, 3) for x in rates[CHECK_WITNESS]]},
            "with_over_without": round(on / off, 4),
            "proof_sha": hashlib.sha256(want.tobytes()).hexdigest()[:16],
        }), flush=True)
        del dz
        g.close()


if __name__ == "__main__":
    main()
