#!/usr/bin/env python3
"""Cost of loading a snarkjs .zkey (g16_zkey_load: circuit A and B plus the proving key in one call) against loading the same
circuit and key from limbs (g16_circuit_load_qap(CIRCOM) + g16_pk_load), per curve on the synthetic circuit of size 2^log_n.
The key is made with g16_setup under CircomReduction, written as a .zkey by tests/zkey_ref.py, and loaded first to check
that a proof under it equals the limbs path's.  Then, alternated over --reps rounds after --warmup untimed ones:

  * g16_zkey_load without and with validate (host clock around the call; it ends in a stream synchronise), with the
    g16_get_timings split (witness_map_ms = coefficient upload, decode and CSR build; h2d_ms = upload and point checks);
  * g16_circuit_load_qap + g16_pk_load from limbs of the same key (host clock).
Medians and ranges are printed as one JSON line per curve, after the card (name, power limit, max SM clock, read with
nvidia-smi in the same run).

  python tools/bench_zkey.py [--curves bn254 bls12_381] [--log-n 20] [--reps 5] [--warmup 1]
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
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from groth16_b200 import Groth16  # noqa: E402
from groth16_b200.params import GENERATORS  # noqa: E402
from groth16_b200.workload import synthetic_r1cs  # noqa: E402
import zkey_ref as Z  # noqa: E402

TOXIC = (0x2222222222222222222223, 0x3333333333333333333335, 0x6666666666666666666661, 0x4444444444444444444447,
         0x1234567890ABCDEF1234567)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # report, do not guess
        return f"nvidia-smi unavailable: {e}"


def timed(fn):
    t = time.perf_counter()
    fn()
    return (time.perf_counter() - t) * 1e3


def stats(v):
    return dict(median=round(statistics.median(v), 1), min=round(min(v), 1), max=round(max(v), 1))


def run(curve, log_n, reps, warmup):
    m, z, _ = synthetic_r1cs(curve, log_n, seed=log_n)
    z = np.ascontiguousarray(z)
    gl = Groth16(curve, 0, qap="circom")
    G = GENERATORS[curve]
    pk = gl.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=True)
    t = time.perf_counter()
    data = Z.write(curve, m, pk)
    write_s = time.perf_counter() - t
    gz = Groth16(curve, 0, qap="circom")
    _, info = gz.load_zkey(data, validate=False)
    gl.load_matrices(m)
    gl.load_proving_key(pk)
    prove = lambda g, c: np.concatenate([getattr(g.create_proof_with_reduction_and_matrices(
        None, 12345, 67890, None, c.num_instance_variables, c.num_constraints, z), k) for k in ("a", "b", "c")])
    if not np.array_equal(prove(gz, info), prove(gl, m)):
        raise SystemExit(f"{curve} 2^{log_n}: the proof under the .zkey differs from the limbs path")
    rows = {k: [] for k in ("zkey_ms", "zkey_validate_ms", "limbs_ms", "coef_ms", "points_ms", "coef_validate_ms",
                            "points_validate_ms")}
    for rep in range(warmup + reps):
        tz = timed(lambda: gz.load_zkey(data, validate=False))
        t1 = gz.timings()
        tv = timed(lambda: gz.load_zkey(data, validate=True))
        t2 = gz.timings()
        tl = timed(lambda: (gl.load_matrices(m), gl.load_proving_key(pk)))
        if rep < warmup:
            continue
        rows["zkey_ms"].append(tz)
        rows["zkey_validate_ms"].append(tv)
        rows["limbs_ms"].append(tl)
        rows["coef_ms"].append(t1["witness_map_ms"])
        rows["points_ms"].append(t1["h2d_ms"])
        rows["coef_validate_ms"].append(t2["witness_map_ms"])
        rows["points_validate_ms"].append(t2["h2d_ms"])
    res = dict(curve=curve, log_n=log_n, zkey_bytes=len(data), coefficients=int(info.a_nnz + info.b_nnz + info.num_instance_variables),
               proofs_equal=True, write_zkey_python_s=round(write_s, 1), **{k: stats(v) for k, v in rows.items()})
    print(json.dumps(res), flush=True)
    gz.close()
    gl.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", nargs="+", default=list(Z.SNARKJS_CURVES))
    ap.add_argument("--log-n", nargs="+", type=int, default=[20])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    for curve in a.curves:
        for log_n in a.log_n:
            run(curve, log_n, a.reps, a.warmup)


if __name__ == "__main__":
    main()
