#!/usr/bin/env python3
"""Cost of checking a powers-of-tau transcript (g16_srs_verify_pairs): per curve, transcript size n (tau_g1 holds 2n - 1
points, the other vectors n) and with the subgroup check on and off (`validate`),

  * the whole call (host clock; it ends in a stream synchronise);
  * points per second of each member's chunk loop -- upload, check, scalars, MSM (g16_get_timings msm_ms[0..3]);
  * the subgroup check's share of the call: 1 - (time without validate) / (time with it), on the validate rows;
  * g16_srs_contribute of the same transcript with the same flag, for context.
Each is run --warmup times untimed, then --reps times; the median is printed.  Before timing, the twenty output points must
equal their closed-form scalars times the generators (the CPU oracle; tests/bw6_ref.py for BW6-761).  With --big, BN254 at
n = 2^24 runs once with automatic chunks, without validate.  Prints the card (name, power limit, max SM clock, read with
nvidia-smi in the same run) and one JSON line per configuration.

  python tools/bench_srs_verify.py [--curves bn254 bls12_381] [--log-n 16 18 20] [--reps 3] [--warmup 1] [--big]
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")]
from groth16_b200 import Groth16, _lib  # noqa: E402
from groth16_b200.params import GENERATORS  # noqa: E402
from srs_verify_ref import closed_exponents  # noqa: E402

TAU, ALPHA, BETA = 0x1234567890ABCDEF1234567, 0x2222222222222222222223, 0x3333333333333333333335
TAU2, ALPHA2, BETA2 = 0x7777777777777777777779ABC, 0x6666666666666666666661, 0x5555555555555555555557
RHO = 0x5EED5EED5EED5EED5EED5EED5EED5EED1
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


def closed(g, p, q):
    curve, cd = g.curve.name, g.codec
    G = GENERATORS[curve]
    if curve == "bw6_761":
        import bw6_ref as B
        return cd.enc_g1([B.mul(k, G["g1"]) for k in p]), cd.enc_g2([B.mul(k, G["g2"]) for k in q])
    import orc
    import pyref as P
    cid = P.CURVES[curve].cid
    g1, g2 = (np.ascontiguousarray(x) for x in (cd.enc_g1([G["g1"]])[0], cd.enc_g2([G["g2"]])[0]))
    return orc.batch_mul_g1(cid, cd.nq, g1, cd.fr.enc(p), 4), orc.batch_mul_g2(cid, cd.nq, g2, cd.fr.enc(q), 4)


def run(g, curve, log_n, reps, warmup, context=True, validates=(True, False)):
    G = GENERATORS[curve]
    n = 1 << log_n
    src = g.srs_from_secrets(2 * n - 1, n, TAU, ALPHA, BETA, G["g1"], G["g2"])
    want = closed(g, *closed_exponents(g.curve.r, (2 * n - 1, n, n, n), TAU, ALPHA, BETA, RHO))
    got = g.srs_verification_pairs(src, RHO)
    if not (np.array_equal(got.g1, want[0]) and np.array_equal(got.g2, want[1])):
        raise SystemExit(f"{curve} 2^{log_n}: the output points differ from the closed form")
    res = {}
    for validate in validates:
        rows = {k: [] for k in ("verify_ms", "contribute_ms")}
        rate = {k: [] for k in VECS}
        for rep in range(warmup + reps):
            t = timed(lambda: g.srs_verification_pairs(src, RHO, validate=validate))
            tm = _lib.Timings()
            g._lib.g16_get_timings(g._ctx, C.byref(tm))
            t_c = timed(lambda: g.contribute_srs(src, TAU2, ALPHA2, BETA2, validate=validate)) if context else 0.0
            if rep < warmup:
                continue
            rows["verify_ms"].append(t)
            rows["contribute_ms"].append(t_c)
            for m, k in enumerate(VECS):
                rate[k].append(getattr(src, k).shape[0] / (tm.msm_ms[m] * 1e-3))
        med = {k: statistics.median(v) for k, v in rows.items()}
        res[validate] = dict(curve=curve, log_n=log_n, validate=validate, equal=True, verify_ms=round(med["verify_ms"], 1),
                             **{f"{k}_pts_per_s": float(f"{statistics.median(v):.3g}") for k, v in rate.items()})
        if context:
            res[validate]["contribute_ms"] = round(med["contribute_ms"], 1)
    if True in res and False in res:
        res[True]["subgroup_share"] = round(1 - res[False]["verify_ms"] / res[True]["verify_ms"], 3)
    for v in validates:
        print(json.dumps(res[v]), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", nargs="+", default=["bn254", "bls12_381", "bls12_377", "bw6_761"])
    ap.add_argument("--log-n", nargs="+", type=int, default=[16, 18, 20])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--big", action="store_true", help="also BN254 at n = 2^24, automatic chunks, without validate")
    a = ap.parse_args()
    print("card:", card(), flush=True)
    for curve in a.curves:
        g = Groth16(curve, 0)
        for log_n in a.log_n:
            run(g, curve, log_n, a.reps, a.warmup)
        g.close()
    if a.big:
        g = Groth16("bn254", 0)
        run(g, "bn254", 24, 1, 0, context=False, validates=(False,))
        g.close()


if __name__ == "__main__":
    main()
