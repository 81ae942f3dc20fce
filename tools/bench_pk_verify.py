#!/usr/bin/env python3
"""Cost of checking a proving key against its circuit and transcript (g16_pk_verify_pairs), against re-deriving the key
(g16_setup_from_srs) of the same circuit and transcript: per curve, circuit size n (the synthetic circuit of bench.py,
LibsnarkReduction) and with the subgroup check on and off (`validate`),

  * the whole call (host clock; it ends in a stream synchronise) and its stages (g16_get_timings: h2d_ms = upload and
    point checks, witness_map_ms = the field work, msm_ms[0] / msm_ms[1] = the key-side / transcript-side MSMs);
  * g16_setup_from_srs of the same circuit and transcript with the same flag;
  * their ratio.
The check is run --warmup times untimed, then --reps times, the derivation once per flag; medians are printed.  Before
timing, the eight G1 and eight G2 output points must equal their closed form: for BN254, BLS12-381 and BLS12-377
S_X(K) = sum_j rho^j K_j by the CPU oracle's MSM over the exported key, S_X(T) = delta S_X(K) (gamma for gamma_abc_g1),
the single points as exported; for BW6-761 the exponents of tests/pk_verify_ref.py times the generators (tests/bw6_ref.py).
With --big, BN254 at n = 2^22 runs too, once per flag.  Prints the card (name, power limit, max SM clock, read with
nvidia-smi in the same run) and one JSON line per configuration.

  python tools/bench_pk_verify.py [--curves bn254 bls12_381] [--log-n 16 18 20] [--reps 3] [--warmup 1] [--big]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")]
from groth16_b200 import Groth16  # noqa: E402
from groth16_b200.api import key_members  # noqa: E402
from groth16_b200.params import GENERATORS  # noqa: E402
from groth16_b200.workload import synthetic_r1cs  # noqa: E402

TAU, ALPHA, BETA, GAMMA, DELTA = (0x1234567890ABCDEF1234567, 0x2222222222222222222223, 0x3333333333333333333335,
                                  0x6666666666666666666661, 0x4444444444444444444447)
RHO = 0x5EED5EED5EED5EED5EED5EED5EED5EED1


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


def expected(g, m, pk):
    """the eight G1 and eight G2 output points of an honest key, independently of the device"""
    curve, cd, r = g.curve.name, g.codec, g.curve.r
    ni = m.num_instance_variables
    if curve == "bw6_761":
        import bw6_ref as B
        from pk_verify_ref import key_exponents, key_sums, verdict
        rows = []
        for rp, col, val in (m.a, m.b, m.c):
            vals = cd.fr.dec(val)
            rows.append([[(vals[e], int(col[e])) for e in range(int(rp[i]), int(rp[i + 1]))] for i in range(len(rp) - 1)])
        k = key_exponents(r, B.domain_root, rows, ni, m.num_witness_variables, ALPHA, BETA, GAMMA, DELTA, TAU, False)
        ks = key_sums(k, RHO, r, ni)
        ts = dict(ks, h=ks["h"] * DELTA % r, l=ks["l"] * DELTA % r, ic=ks["ic"] * GAMMA % r)
        _, p, q = verdict(k, (TAU, ALPHA, BETA), ts, RHO, r, ni)
        G = GENERATORS[curve]
        return cd.enc_g1([B.mul(x, G["g1"]) for x in p]), cd.enc_g2([B.mul(x, G["g2"]) for x in q])
    import orc
    import pyref as P
    cid, nq = P.CURVES[curve].cid, cd.nq
    cx = P.ctx(P.CURVES[curve])
    km = key_members(pk)
    nv = km["a_query"].shape[0]
    rho = [pow(RHO, j, r) for j in range(max(nv, km["h_query"].shape[0]))]

    def msm(pts, first=0):   # the oracle's projective result (Z = 1, or Z = 0 for the identity) as a pyref point
        xyz = orc.msm_g1(cid, nq, pts, cd.fr.bigint(rho[first:first + len(pts)]), 16)
        return cd.dec_g1(xyz[None, :2 * nq])[0] if xyz[2 * nq:].any() else None

    sh, sl, sic = msm(km["h_query"]), msm(km["l_query"], ni), msm(km["gamma_abc_g1"])
    d1, g1 = cd.dec_g1(km["delta_g1"])[0], GENERATORS[curve]["g1"]
    ps = [d1, g1, sh, cx.G1.mul(sh, DELTA), sl, cx.G1.mul(sl, DELTA), sic, cx.G1.mul(sic, GAMMA)]
    g2, d2, gm2 = GENERATORS[curve]["g2"], cd.dec_g2(km["delta_g2"])[0], cd.dec_g2(km["gamma_g2"])[0]
    qs = [g2, d2, d2, g2, d2, g2, gm2, g2]
    return cd.enc_g1(ps), cd.enc_g2(qs)


def run(g, curve, log_n, reps, warmup):
    G = GENERATORS[curve]
    n = 1 << log_n
    m, _, _ = synthetic_r1cs(curve, log_n, seed=700 + log_n)
    pk = g.generate_parameters_with_qap(m, ALPHA, BETA, GAMMA, DELTA, TAU, G["g1"], G["g2"])
    srs = g.srs_from_secrets(2 * n - 1, n, TAU, ALPHA, BETA, G["g1"], G["g2"])
    got = g.key_verification_pairs(pk, srs, RHO)
    want = expected(g, m, pk)
    if not (np.array_equal(got.g1, want[0]) and np.array_equal(got.g2, want[1])):
        raise SystemExit(f"{curve} 2^{log_n}: the output points differ from the closed form")
    res = {}
    for validate in (True, False):
        rows = {k: [] for k in ("verify_ms", "h2d_ms", "field_ms", "key_msm_ms", "srs_msm_ms")}
        for rep in range(warmup + reps):
            t = timed(lambda: g.key_verification_pairs(pk, srs, RHO, validate=validate))
            tm = g.timings()
            if rep < warmup:
                continue
            for k, v in (("verify_ms", t), ("h2d_ms", tm["h2d_ms"]), ("field_ms", tm["witness_map_ms"]),
                         ("key_msm_ms", tm["msm_ms"]["h"]), ("srs_msm_ms", tm["msm_ms"]["l"])):
                rows[k].append(v)
        t_setup = timed(lambda: g.generate_parameters_from_srs(None, srs, validate=validate, export=False))
        g.generate_parameters_with_qap(m, ALPHA, BETA, GAMMA, DELTA, TAU, G["g1"], G["g2"], export=False)
        med = {k: round(statistics.median(v), 1) for k, v in rows.items()}
        res[validate] = dict(curve=curve, log_n=log_n, validate=validate, equal=True, **med, setup_from_srs_ms=round(t_setup, 1),
                             setup_over_verify=round(t_setup / med["verify_ms"], 2))
    for v in (True, False):
        print(json.dumps(res[v]), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", nargs="+", default=["bn254", "bls12_381", "bls12_377", "bw6_761"])
    ap.add_argument("--log-n", nargs="+", type=int, default=[16, 18, 20])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--big", action="store_true", help="also BN254 at n = 2^22, once per flag")
    a = ap.parse_args()
    print("card:", card(), flush=True)
    for curve in a.curves:
        g = Groth16(curve, 0)
        for log_n in a.log_n:
            run(g, curve, log_n, a.reps, a.warmup)
        g.close()
    if a.big:
        g = Groth16("bn254", 0)
        run(g, "bn254", 22, 1, 0)
        g.close()


if __name__ == "__main__":
    main()
