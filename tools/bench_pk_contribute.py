#!/usr/bin/env python3
"""Cost of a phase-2 contribution to a key held in host memory (g16_pk_contribute) against the same contribution to the
resident key (g16_setup_contribute), on one key: per curve and circuit size 2^log_n (the synthetic circuit, so h_query holds
n - 1 points and l_query n - 1),

  * the whole g16_pk_contribute call (host clock; it ends in a stream synchronise), with and without validate, the check
    pass's share of it (g16_get_timings h2d_ms), and points per second of the H and L transforms (msm_ms[0], msm_ms[1]);
  * g16_setup_contribute on the resident key g16_setup made (host clock around the call).
Each is run --warmup times untimed, then --reps times; the median is printed.  Before timing, the contributed key must equal
g16_setup of the product delta in every limb.  With --big, BN254 at 2^24 runs once more with automatic chunks and with
chunk_points = 2^22 (its resident keys without precomputed multiples, msm_ne = 0).  Prints the card (name, power limit, max
SM clock, read with nvidia-smi in the same run) and one JSON line per configuration.

  python tools/bench_pk_contribute.py [--curves bn254 bls12_381] [--log-n 16 18 20] [--reps 3] [--warmup 1] [--big]
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

TAU, ALPHA, BETA, GAMMA, DELTA0 = (0x1234567890ABCDEF1234567, 0x2222222222222222222223, 0x3333333333333333333335,
                                   0x6666666666666666666661, 0x4444444444444444444447)
DELTA = 0x7777777777777777777779ABC
CHANGED = ("h_query", "l_query", "delta_g1")


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


def run(g, curve, log_n, reps, warmup, chunk_points=0, context=True):
    G = GENERATORS[curve]
    m, _, _ = synthetic_r1cs(curve, log_n, seed=log_n)
    setup = lambda d, export=True: g.generate_parameters_with_qap(m, ALPHA, BETA, GAMMA, d, TAU, G["g1"], G["g2"], export=export)
    want = setup(DELTA0 * DELTA % g.curve.r)
    pk = setup(DELTA0)
    got = g.contribute_key(pk, DELTA, chunk_points=chunk_points)
    if not (all(np.array_equal(getattr(got, k), getattr(want, k)) for k in CHANGED)
            and np.array_equal(got.vk.delta_g2, want.vk.delta_g2)):
        raise SystemExit(f"{curve} 2^{log_n}: the contributed key differs from g16_setup of the product delta")
    del got, want
    rows = {k: [] for k in ("contribute_ms", "validate_ms", "check_ms", "setup_contribute_ms")}
    rate = {k: [] for k in ("h", "l")}
    for rep in range(warmup + reps):
        t = timed(lambda: g.contribute_key(pk, DELTA, chunk_points=chunk_points))
        tm = _lib.Timings()
        g._lib.g16_get_timings(g._ctx, C.byref(tm))
        tv = timed(lambda: g.contribute_key(pk, DELTA, chunk_points=chunk_points, validate=True)) if context else 0.0
        ts = timed(lambda: g.contribute_delta(DELTA, export=False)) if context else 0.0
        if rep < warmup:
            continue
        rows["contribute_ms"].append(t)
        rows["validate_ms"].append(tv)
        rows["check_ms"].append(tm.h2d_ms)
        rows["setup_contribute_ms"].append(ts)
        rate["h"].append(len(pk.h_query) / (tm.msm_ms[0] * 1e-3))
        rate["l"].append(len(pk.l_query) / (tm.msm_ms[1] * 1e-3))
    med = {k: statistics.median(v) for k, v in rows.items()}
    res = dict(curve=curve, log_n=log_n, chunk_points=chunk_points, h_points=len(pk.h_query), l_points=len(pk.l_query),
               equal=True, contribute_ms=round(med["contribute_ms"], 1), check_share=round(med["check_ms"] / med["contribute_ms"], 3),
               h_pts_per_s=float(f"{statistics.median(rate['h']):.3g}"), l_pts_per_s=float(f"{statistics.median(rate['l']):.3g}"))
    if context:
        res.update(contribute_validate_ms=round(med["validate_ms"], 1), setup_contribute_ms=round(med["setup_contribute_ms"], 1))
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", nargs="+", default=["bls12_381", "bn254", "bls12_377", "bw6_761"])
    ap.add_argument("--log-n", nargs="+", type=int, default=[16, 18, 20])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--big", action="store_true", help="also BN254 at 2^24, automatic chunks and 2^22-point chunks")
    a = ap.parse_args()
    print("card:", card(), flush=True)
    for curve in a.curves:
        g = Groth16(curve, 0)
        for log_n in a.log_n:
            run(g, curve, log_n, a.reps, a.warmup)
        g.close()
    if a.big:
        g = Groth16("bn254", 0)
        g.set_option("msm_ne", 0)   # no precomputed multiples: a 2^24 key with them does not fit next to its copies
        for chunk in (0, 1 << 22):
            run(g, "bn254", 24, 1, 0, chunk_points=chunk, context=False)
        g.close()


if __name__ == "__main__":
    main()
