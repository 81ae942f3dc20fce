#!/usr/bin/env python3
"""Cost of a phase-1 contribution to a powers-of-tau transcript (g16_srs_contribute): per curve and transcript size n
(tau_g1 holds 2n - 1 points, the other vectors n),

  * the whole call (host clock; it ends in a stream synchronise), and the check pass's share of it (g16_get_timings h2d_ms);
  * points per second of each member's transform (msm_ms[0..3]);
  * g16_srs_from_secrets at the same lengths (fixed-base tables), for context.
Each is run --warmup times untimed, then --reps times; the median is printed.  Before timing, the contributed transcript
must equal g16_srs_from_secrets of the product secrets in every limb.  With --big, BN254 at n = 2^24 runs once more with
automatic chunks and with chunk_points = 2^22.  Prints the card (name, power limit, max SM clock, read with nvidia-smi in
the same run) and one JSON line per configuration.

  python tools/bench_srs_contribute.py [--curves bn254 bls12_381] [--log-n 16 18 20] [--reps 3] [--warmup 1] [--big]
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

TAU, ALPHA, BETA = 0x1234567890ABCDEF1234567, 0x2222222222222222222223, 0x3333333333333333333335
TAU2, ALPHA2, BETA2 = 0x7777777777777777777779ABC, 0x6666666666666666666661, 0x5555555555555555555557
VECS = ("tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1")


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
    r = g.curve.r
    n = 1 << log_n
    src = g.srs_from_secrets(2 * n - 1, n, TAU, ALPHA, BETA, G["g1"], G["g2"])
    got = g.contribute_srs(src, TAU2, ALPHA2, BETA2, chunk_points=chunk_points)
    want = g.srs_from_secrets(2 * n - 1, n, TAU * TAU2 % r, ALPHA * ALPHA2 % r, BETA * BETA2 % r, G["g1"], G["g2"])
    if not all(np.array_equal(getattr(got, k), getattr(want, k)) for k in VECS + ("beta_g2",)):
        raise SystemExit(f"{curve} 2^{log_n}: the contributed transcript differs from srs_from_secrets")
    del got, want
    rows = {k: [] for k in ("contribute_ms", "check_ms", "from_secrets_ms")}
    rate = {k: [] for k in VECS}
    for rep in range(warmup + reps):
        t = timed(lambda: g.contribute_srs(src, TAU2, ALPHA2, BETA2, chunk_points=chunk_points))
        tm = _lib.Timings()
        g._lib.g16_get_timings(g._ctx, C.byref(tm))
        t_sec = timed(lambda: g.srs_from_secrets(2 * n - 1, n, TAU, ALPHA, BETA, G["g1"], G["g2"])) if context else 0.0
        if rep < warmup:
            continue
        rows["contribute_ms"].append(t)
        rows["check_ms"].append(tm.h2d_ms)
        rows["from_secrets_ms"].append(t_sec)
        for m, k in enumerate(VECS):
            rate[k].append(getattr(src, k).shape[0] / (tm.msm_ms[m] * 1e-3))
    med = {k: statistics.median(v) for k, v in rows.items()}
    res = dict(curve=curve, log_n=log_n, chunk_points=chunk_points, equal=True, contribute_ms=round(med["contribute_ms"], 1),
               check_share=round(med["check_ms"] / med["contribute_ms"], 3),
               **{f"{k}_pts_per_s": float(f"{statistics.median(v):.3g}") for k, v in rate.items()})
    if context:
        res["from_secrets_ms"] = round(med["from_secrets_ms"], 1)
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", nargs="+", default=["bls12_381", "bn254", "bls12_377", "bw6_761"])
    ap.add_argument("--log-n", nargs="+", type=int, default=[16, 18, 20])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--big", action="store_true", help="also BN254 at n = 2^24, automatic chunks and 2^22-point chunks")
    a = ap.parse_args()
    print("card:", card(), flush=True)
    for curve in a.curves:
        g = Groth16(curve, 0)
        for log_n in a.log_n:
            run(g, curve, log_n, a.reps, a.warmup)
        g.close()
    if a.big:
        g = Groth16("bn254", 0)
        for chunk in (0, 1 << 22):
            run(g, "bn254", 24, 1, 0, chunk_points=chunk, context=False)
        g.close()


if __name__ == "__main__":
    main()
