#!/usr/bin/env python3
"""BW6-761 proving on one GPU: proofs/s (two proofs in flight, after a warm-up of both proof slots), single-proof latency
and per-stage times of the synthetic circuit at 2^16, 2^18 and 2^20, plus the resident key's bytes (computed from the
shapes and the launch geometry).  Every proof of a size is checked to be the same.  Prints
one JSON line per size and, first, the card it ran on.

  python tools/bench_bw6.py --log-n 16 18 20 --steps 10 --warmup 2 [--ba-g1 R --ba-g2 R]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from groth16_b200 import Groth16  # noqa: E402
from groth16_b200.params import GENERATORS  # noqa: E402
from groth16_b200.workload import synthetic_r1cs  # noqa: E402

TOXIC = (11, 22, 33, 44, 55)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # report, do not guess
        return f"nvidia-smi unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, nargs="+", default=[16, 18, 20])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ba-g1", type=int, default=None)
    ap.add_argument("--ba-g2", type=int, default=None)
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    G = GENERATORS["bw6_761"]
    for L in a.log_n:
        g = Groth16("bw6_761", 0)
        if a.ba_g1 is not None:
            g.set_option("msm_ba", a.ba_g1)
        if a.ba_g2 is not None:
            g.set_option("msm_ba_g2", a.ba_g2)
        m, z, _ = synthetic_r1cs("bw6_761", L, seed=1)
        t = time.time()
        g.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=False)
        t_setup = time.time() - t
        r = np.ascontiguousarray(g.codec.fr.enc1(123456789))
        s = np.ascontiguousarray(g.codec.fr.enc1(987654321))
        nout = 4 * g.nq + g.ng2
        ref_proof = np.zeros(nout, dtype=np.uint64)
        g.prove_raw(r, s, z.ctypes.data, 0, ref_proof)
        # warm-up through both proof slots: slot 1 reserves its work buffers and MSM workspaces on first use, which must not
        # land in the timed pipelined run
        warm = [np.zeros(nout, dtype=np.uint64) for _ in range(2)]
        for _ in range(max(1, a.warmup)):
            g.prove_submit_raw(0, r, s, z.ctypes.data, 0)
            g.prove_submit_raw(1, r, s, z.ctypes.data, 0)
            g.prove_wait_raw(0, warm[0])
            g.prove_wait_raw(1, warm[1])
            assert np.array_equal(warm[0], ref_proof) and np.array_equal(warm[1], ref_proof)
        lat = []
        out = np.zeros(nout, dtype=np.uint64)
        stages = []
        for _ in range(a.steps):
            t = time.perf_counter()
            g.prove_raw(r, s, z.ctypes.data, 0, out)
            lat.append(time.perf_counter() - t)
            assert np.array_equal(out, ref_proof)
            tm = g.timings()
            stages.append([tm["witness_map_ms"]] + [tm["msm_ms"][k] for k in ("h", "l", "a", "b_g1", "b_g2")])
        outs = [np.zeros(nout, dtype=np.uint64) for _ in range(2)]
        t = time.perf_counter()
        g.prove_submit_raw(0, r, s, z.ctypes.data, 0)
        for i in range(1, a.steps):
            g.prove_submit_raw(i & 1, r, s, z.ctypes.data, 0)
            g.prove_wait_raw((i - 1) & 1, outs[(i - 1) & 1])
        g.prove_wait_raw((a.steps - 1) & 1, outs[(a.steps - 1) & 1])
        t_pipe = time.perf_counter() - t
        assert all(np.array_equal(o, ref_proof) for o in outs)
        st = np.median(np.array(stages), axis=0)
        nv = m.num_instance_variables + m.num_witness_variables
        key_bytes = sum(q * (2 * g.nq * 8) for q in (nv, nv, (1 << L) - 1, m.num_witness_variables)) + nv * g.ng2 * 8
        cfg = g.config()
        print(json.dumps({
            "curve": "bw6_761", "log_n": L, "setup_s": round(t_setup, 2),
            "latency_ms": {"median": round(1e3 * float(np.median(lat)), 2), "min": round(1e3 * min(lat), 2),
                           "max": round(1e3 * max(lat), 2)},
            "proofs_per_sec_two_in_flight": round(a.steps / t_pipe, 3),
            "stage_ms_median": dict(zip(("witness_map", "msm_h", "msm_l", "msm_a", "msm_b_g1", "msm_b_g2"),
                                        [round(float(x), 2) for x in st])),
            "config": cfg, "key_bytes_one_copy": int(key_bytes),
            "resident_key_bytes": int(key_bytes * cfg["copies"]),   # every base with its precomputed copies
            "proof_sha": __import__("hashlib").sha256(ref_proof.tobytes()).hexdigest()[:16],
        }), flush=True)
        g.close()


if __name__ == "__main__":
    main()
