#!/usr/bin/env python3
"""tools/sweep.py -- one process, one resident key, many MSM launch geometries (g16_set_option): proofs/s and the
per-MSM accumulation-stage times for each, every proof compared bit for bit with the first.  Writes JSON lines to
gpurun_out/sweep_<tag>.jsonl.  Development tool (not part of the product or the tests).

  python tools/sweep.py --curve bls12_381 --log-n 20 --tag r02a [--set name=spec ...]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEFAULT_GRID = [
    {"msm_ba": 0, "msm_ba_g2": 0},
    {"msm_ba": 2, "msm_ba_g2": 0},
    {"msm_ba": 3, "msm_ba_g2": 0},
    {"msm_ba": 4, "msm_ba_g2": 0},
    {"msm_ba": 5, "msm_ba_g2": 0},
    {"msm_ba": 6, "msm_ba_g2": 0},
    {"msm_ba": 4, "msm_ba_g2": 0, "ba_m": 8},
    {"msm_ba": 4, "msm_ba_g2": 0, "ba_m": 32},
    {"msm_ba": 4, "msm_ba_g2": 0, "ba_g": 16},
    {"msm_ba": 4, "msm_ba_g2": 0, "ba_g": 256},
    {"msm_ba": 4, "msm_ba_g2": 0, "ba_inv_gcd": 0},
    {"msm_ba": 4, "msm_ba_g2": 2},
    {"msm_ba": 4, "msm_ba_g2": 3},
    {"msm_ba": 4, "msm_ba_g2": 4},
    {"msm_ba": 4, "msm_ba_g2": 5},
    {"msm_ba": 4, "msm_ba_g2": 4, "ba_m": 8},
    {"msm_ba": 4, "msm_ba_g2": 0, "acc_k0_g2": 16},
    {"msm_ba": 4, "msm_ba_g2": 0, "acc_k0_g2": 64},
]
BASE = {"msm_ba": 4, "msm_ba_g2": 4, "ba_m": 32, "ba_g": 16, "ba_inv_gcd": 1, "acc_k0_g1": 0, "acc_k0_g2": 0, "acc_block": 128,
        "share_b_sort": 1, "ba_occ_g1": 0, "ba_occ_g2": 0, "ntt_tma": -1,
        "ba_cap_fwd_g1": 0, "ba_cap_bwd_g1": 0, "ba_cap_fwd_g2": 0, "ba_cap_bwd_g2": 0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curve", default="bls12_381")
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--tag", default="sweep")
    ap.add_argument("--grid", default="", help="JSON list of option dicts (default: the built-in grid)")
    a = ap.parse_args()
    import torch
    from bench import TOXIC
    from groth16_b200 import Groth16, _lib
    from groth16_b200.params import GENERATORS
    from groth16_b200.workload import synthetic_r1cs
    m, z_np, pub = synthetic_r1cs(a.curve, a.log_n, seed=1)
    g = Groth16(a.curve, 0)
    G = GENERATORS[g.curve.name]
    g.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=False)
    cd, nq = g.codec, g.nq
    r = np.ascontiguousarray(cd.fr.enc1(123456789))
    s = np.ascontiguousarray(cd.fr.enc1(987654321))
    z_dev = torch.from_numpy(z_np.view(np.int64)).pin_memory().to("cuda:0")
    proof = np.zeros(8 * nq, dtype=np.uint64)
    grid = json.loads(a.grid) if a.grid else DEFAULT_GRID
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    out = open(os.path.join(ROOT, "gpurun_out", f"sweep_{a.tag}.jsonl"), "a")
    first = None
    for opts in grid:
        cfg = dict(BASE)
        cfg.update(opts)
        for k, v in cfg.items():
            g.set_option(k, v)
        ON = _lib.ASSIGNMENT_ON_DEVICE
        for _ in range(3):
            g.prove_raw(r, s, z_dev.data_ptr(), ON, proof)
        if first is None:
            first = proof.copy()
        ok = bool(np.array_equal(first, proof))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.steps):
            g.prove_raw(r, s, z_dev.data_ptr(), ON, proof)
        torch.cuda.synchronize()
        ms = 1e3 * (time.perf_counter() - t0) / a.steps
        acc = {k: [] for k in ("h", "l", "a", "b_g1", "b_g2")}
        msm = {k: [] for k in acc}
        for _ in range(3):
            g.prove_raw(r, s, z_dev.data_ptr(), ON | _lib.SERIAL_MSMS, proof)
            tm = g.timings()
            for k in acc:
                acc[k].append(tm["msm_accum_ms"][k])
                msm[k].append(tm["msm_ms"][k])
        ok = ok and bool(np.array_equal(first, proof))
        line = {"curve": a.curve, "log_n": a.log_n, "opts": opts, "ms_per_proof": ms, "proof_identical": ok,
                "accum_ms": {k: round(statistics.median(v), 3) for k, v in acc.items()},
                "msm_ms_serial": {k: round(statistics.median(v), 3) for k, v in msm.items()},
                "witness_map_ms": round(tm["witness_map_ms"], 3), "launches": tm["launches"], "config": g.config()}
        print(json.dumps(line), flush=True)
        out.write(json.dumps(line) + "\n")
        out.flush()
        if not ok:
            print("PARITY FAILURE for", opts, flush=True)
    out.close()


if __name__ == "__main__":
    main()
