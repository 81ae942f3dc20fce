#!/usr/bin/env python3
"""Cost of reading circom files on the GPU, per curve on the synthetic circuit of size 2^log_n under CircomReduction:

  * g16_r1cs_load of the circuit's .r1cs against g16_circuit_load_qap of the same matrices in limbs, with the
    g16_get_timings split (h2d_ms = host walk, witness_map_ms = upload, decode and host copies);
  * g16_zkey_load with G16_ZKEY_KEY_ONLY (the key onto the resident .r1cs circuit) against the full g16_zkey_load
    (BN254 and BLS12-381, the curves snarkjs writes), without validate;
  * g16_wtns_read of the circuit's witness.
The files are written by tests/r1cs_ref.py and tests/zkey_ref.py.  Before timing, a proof after load_r1cs (and after the
key-only load) must equal the proof after load_matrices.  Host clock around each call (every call ends in a synchronise),
alternated over --reps rounds after --warmup untimed ones; medians and ranges are printed as one JSON line per curve, after
the card (name, power limit, max SM clock, read with nvidia-smi in the same run).

  python tools/bench_r1cs.py [--curves bn254 bls12_381 bls12_377 bw6_761] [--log-n 20] [--reps 5] [--warmup 1]
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
import r1cs_ref as R  # noqa: E402
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
    snarkjs = curve in Z.SNARKJS_CURVES
    gl = Groth16(curve, 0, qap="circom")
    G = GENERATORS[curve]
    pk = gl.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=True)
    r1 = R.write(R.Circuit.from_matrices(curve, m))
    wt = R.wtns_from_limbs(curve, z)
    zk = Z.write(curve, m, pk) if snarkjs else None
    gr = Groth16(curve, 0, qap="circom")
    info = gr.load_r1cs(r1)
    gr.load_proving_key(pk)
    gl.load_matrices(m)
    gl.load_proving_key(pk)
    prove = lambda g: np.concatenate([getattr(g.create_proof_with_reduction_and_matrices(
        None, 12345, 67890, None, m.num_instance_variables, m.num_constraints, z), k) for k in ("a", "b", "c")])
    want = prove(gl)
    if not np.array_equal(prove(gr), want):
        raise SystemExit(f"{curve} 2^{log_n}: the proof after load_r1cs differs from the limbs path")
    if snarkjs:
        gr.load_zkey_key(zk, validate=False)
        if not np.array_equal(prove(gr), want):
            raise SystemExit(f"{curve} 2^{log_n}: the proof after load_zkey_key differs from the limbs path")
    if not np.array_equal(gr.read_wtns(wt), z):
        raise SystemExit(f"{curve} 2^{log_n}: read_wtns differs from the assignment")
    gz = Groth16(curve, 0, qap="circom") if snarkjs else None
    rows = {k: [] for k in ("r1cs_ms", "matrices_ms", "r1cs_walk_ms", "r1cs_decode_ms", "wtns_ms")
            + (("zkey_key_only_ms", "zkey_full_ms") if snarkjs else ())}
    for rep in range(warmup + reps):
        tr = timed(lambda: gr.load_r1cs(r1))
        t1 = gr.timings()
        tm = timed(lambda: gl.load_matrices(m))
        tw = timed(lambda: gr.read_wtns(wt))
        if snarkjs:
            tk = timed(lambda: gr.load_zkey_key(zk, validate=False))
            tf = timed(lambda: gz.load_zkey(zk, validate=False))
        if rep < warmup:
            continue
        rows["r1cs_ms"].append(tr)
        rows["matrices_ms"].append(tm)
        rows["r1cs_walk_ms"].append(t1["h2d_ms"])
        rows["r1cs_decode_ms"].append(t1["witness_map_ms"])
        rows["wtns_ms"].append(tw)
        if snarkjs:
            rows["zkey_key_only_ms"].append(tk)
            rows["zkey_full_ms"].append(tf)
    res = dict(curve=curve, log_n=log_n, r1cs_bytes=len(r1), terms=int(info.a_nnz + info.b_nnz + info.c_nnz), wtns_bytes=len(wt),
               proofs_equal=True, **{k: stats(v) for k, v in rows.items()})
    print(json.dumps(res), flush=True)
    for g in (gr, gl, gz):
        if g is not None:
            g.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", nargs="+", default=["bn254", "bls12_381", "bls12_377", "bw6_761"])
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
