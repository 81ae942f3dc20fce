#!/usr/bin/env python3
"""Cost of deriving a proving key from a powers-of-tau transcript on the synthetic circuit: per curve, reduction and size,

  * g16_setup_from_srs, whole call and by stage (upload and point checks, the four group inverse transforms, the sparse sums,
    the H query; host clock around work that ends in a stream synchronise, read through g16_get_timings);
  * g16_setup_contribute (one delta);
  * g16_setup on the same circuit with the same secrets.
Each is run --warmup times untimed, then --reps times; the median is printed.  Before timing, the derived key after one
contribution must equal the g16_setup key in every exported limb.  Prints the card (name, power limit, max SM clock, read
with nvidia-smi in the same run) and one JSON line per configuration.

  python tools/bench_srs_setup.py [--curves bls12_381 bn254] [--log-n 16 18 20] [--qaps libsnark circom] [--reps 3]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from groth16_b200 import Groth16, _lib  # noqa: E402
from groth16_b200.params import GENERATORS  # noqa: E402
from groth16_b200.workload import synthetic_r1cs  # noqa: E402

TAU, ALPHA, BETA, DELTA = 0x1234567890ABCDEF1234567, 0x2222222222222222222223, 0x3333333333333333333335, 0x4444444444444447


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # report, do not guess
        return f"nvidia-smi unavailable: {e}"


def timed(fn):
    t = time.perf_counter()
    fn()
    return (time.perf_counter() - t) * 1e3   # every timed call ends in a stream synchronise inside the library


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", nargs="+", default=["bls12_381", "bn254"])
    ap.add_argument("--log-n", nargs="+", type=int, default=[16, 18, 20])
    ap.add_argument("--qaps", nargs="+", default=["libsnark", "circom"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    for curve in a.curves:
        G = GENERATORS[curve]
        for qap in a.qaps:
            g = Groth16(curve, 0, qap=qap)
            for log_n in a.log_n:
                m, _, _ = synthetic_r1cs(curve, log_n, seed=400 + log_n)
                g.load_matrices(m)
                n = 1 << g._lib.g16_domain_log(g._ctx)
                srs = g.srs_from_secrets(2 * n - 1, n, TAU, ALPHA, BETA, G["g1"], G["g2"])
                g.generate_parameters_from_srs(None, srs, export=False)
                got = g.contribute_delta(DELTA, export=True)
                want = g.generate_parameters_with_qap(m, ALPHA, BETA, 1, DELTA, TAU, G["g1"], G["g2"], export=True)
                same = all(np.array_equal(getattr(got, k), getattr(want, k)) for k in
                           ("a_query", "b_g1_query", "b_g2_query", "h_query", "l_query", "delta_g1")) and \
                    all(np.array_equal(getattr(got.vk, k), getattr(want.vk, k)) for k in
                        ("alpha_g1", "beta_g2", "gamma_g2", "delta_g2", "gamma_abc_g1"))
                if not same:
                    raise SystemExit(f"{curve} {qap} 2^{log_n}: the derived key differs from g16_setup")
                rows = {k: [] for k in ("from_srs_ms", "upload_check_ms", "transforms_ms", "sparse_sums_ms", "h_query_ms",
                                        "contribute_ms", "setup_ms")}
                for rep in range(a.warmup + a.reps):
                    t_srs = timed(lambda: g.generate_parameters_from_srs(None, srs, export=False))
                    tm = _lib.Timings()
                    g._lib.g16_get_timings(g._ctx, C.byref(tm))
                    t_con = timed(lambda: g.contribute_delta(DELTA, export=False))
                    t_set = timed(lambda: g.generate_parameters_with_qap(m, ALPHA, BETA, 1, DELTA, TAU, G["g1"], G["g2"],
                                                                         export=False))
                    if rep < a.warmup:
                        continue
                    for k, v in (("from_srs_ms", t_srs), ("upload_check_ms", tm.h2d_ms), ("transforms_ms", tm.witness_map_ms),
                                 ("sparse_sums_ms", tm.msm_ms[1]), ("h_query_ms", tm.msm_ms[0]), ("contribute_ms", t_con),
                                 ("setup_ms", t_set)):
                        rows[k].append(v)
                res = dict(curve=curve, qap=qap, log_n=log_n, key_equal=True,
                           **{k: round(statistics.median(v), 1) for k, v in rows.items()})
                print(json.dumps(res), flush=True)
            g.close()


if __name__ == "__main__":
    main()
