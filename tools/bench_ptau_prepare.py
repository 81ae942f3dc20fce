#!/usr/bin/env python3
"""Cost of preparing a snarkjs .ptau file for phase 2 on the GPU (g16_ptau_prepare): per curve and power, on the unprepared
file of the transcript of known secrets (srs_from_secrets),

  * the whole call, the check pass and each member's transforms (every level 1 .. top; host clock around work that ends in
    a stream synchronise, read through g16_get_timings);
  * one level's transform: G1 level 2^p = alpha_tau_g1's time at power p minus at power p - 1, G2 level 2^p the same for
    tau_g2 (every lower level is the same work in both), so power p - 1 is run too;
  * the size of the prepared file.
Before timing, on the same card: the prepared file must round-trip -- read_ptau at the file's power, then
generate_parameters_from_ptau for the synthetic circuit (the Lagrange path and its check) -- to the key
generate_parameters_from_srs makes, in every exported byte, under both reductions.  Each call is run --warmup times
untimed, then --reps times; the median is printed.  Prints the card (name, power limit, SM clock, read with nvidia-smi in
the same run) and one JSON line per configuration.

  python tools/bench_ptau_prepare.py [--configs bn254:16,18,20 ...] [--reps 2] [--warmup 1]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ptau_ref as T  # noqa: E402
from groth16_b200 import Groth16  # noqa: E402
from groth16_b200.params import GENERATORS  # noqa: E402
from groth16_b200.workload import synthetic_r1cs  # noqa: E402

TAU, ALPHA, BETA = 0x1234567890ABCDEF1234567, 0x2222222222222222222223, 0x3333333333333333333335
RHO = 0x5A5A5A5A5A5A5A5A5A5A5A5A5A5A5A5A5
DEFAULT = ["bn254:16,18,20", "bls12_381:16,18,20", "bls12_377:16", "bw6_761:16"]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # report, do not guess
        return f"nvidia-smi unavailable: {e}"


def ptau_file(g, power):
    G = GENERATORS[g.curve.name]
    n = 1 << power
    srs = g.srs_from_secrets(2 * n - 1, n, TAU, ALPHA, BETA, G["g1"], G["g2"])
    members = {k: getattr(srs, k) for k in T.MEMBERS}
    members["beta_g2"] = srs.beta_g2
    return T.write(g.curve.name, power, members), srs


def round_trip(curve, power, prepared, srs):
    for qap in ("libsnark", "circom"):
        g = Groth16(curve, 0, qap=qap)
        m, _, _ = synthetic_r1cs(curve, power, seed=700 + power)
        g.generate_parameters_from_ptau(m, prepared, rho=RHO, export=False)
        got = g.export_proving_key_bytes(compress=False)
        g.generate_parameters_from_srs(None, srs, export=False)
        if g.export_proving_key_bytes(compress=False) != got:
            raise SystemExit(f"{curve} {qap} 2^{power}: the key from the prepared file differs from generate_parameters_from_srs")
        g.close()


def measure(g, data, reps, warmup):
    rows = {k: [] for k in ("total_ms", "check_ms", "tau_g1_ms", "tau_g2_ms", "alpha_tau_g1_ms", "beta_tau_g1_ms", "call_ms")}
    size = 0
    for rep in range(warmup + reps):
        t = time.perf_counter()
        size = len(g.prepare_ptau(data))
        call = (time.perf_counter() - t) * 1e3
        tm = g.timings()
        if rep < warmup:
            continue
        ms = list(tm["msm_ms"].values())
        for k, v in (("total_ms", tm["total_ms"]), ("check_ms", tm["h2d_ms"]), ("tau_g1_ms", ms[0]), ("tau_g2_ms", ms[1]),
                     ("alpha_tau_g1_ms", ms[2]), ("beta_tau_g1_ms", ms[3]), ("call_ms", call)):
            rows[k].append(v)
    return {k: round(statistics.median(v), 1) for k, v in rows.items()}, size


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=DEFAULT, help="curve:power,power,...")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-round-trip", action="store_true", help="skip the key check (timing runs of a build already checked)")
    a = ap.parse_args()
    print("card:", card(), flush=True)
    for cfg in a.configs:
        curve, powers = cfg.split(":")
        for power in (int(p) for p in powers.split(",")):
            g = Groth16(curve, 0)
            data, srs = ptau_file(g, power)
            prepared = g.prepare_ptau(data)
            g.close()
            if not a.no_round_trip:
                round_trip(curve, power, prepared, srs)
            del prepared
            g = Groth16(curve, 0)
            res, size = measure(g, data, a.reps, a.warmup)
            lower, _ = measure(g, ptau_file(g, power - 1)[0], a.reps, a.warmup)
            g.close()
            print(json.dumps(dict(curve=curve, power=power, round_trip=not a.no_round_trip, in_bytes=len(data), out_bytes=size, **res,
                                  level_g1_ms=round(res["alpha_tau_g1_ms"] - lower["alpha_tau_g1_ms"], 1),
                                  level_g2_ms=round(res["tau_g2_ms"] - lower["tau_g2_ms"], 1))), flush=True)
    print("card after:", card(), flush=True)


if __name__ == "__main__":
    main()
