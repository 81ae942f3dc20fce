#!/usr/bin/env python3
"""tools/kernel_times.py -- total GPU milliseconds per kernel name over one warm proof with the MSMs run one at a time
(SERIAL_MSMS), from torch.profiler's CUDA activities.  Run it for two builds to compare them kernel by kernel.
Development tool (not part of the product or the tests).

  python tools/kernel_times.py [--curve bls12_381] [--log-n 20] [--root TREE] [--json OUT]

--root imports groth16_b200 (and its built library) from another checkout, e.g. a build of the parent commit.
"""
import argparse
import collections
import json
import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def short_name(name: str) -> str:
    """Kernel name without namespace and argument list: 'ba_backward_kernel<Fp2<BLS381_FqP, 1>, 0>'."""
    name = name.replace("g16::", "").replace("(anonymous namespace)::", "")
    depth = 0
    for i, ch in enumerate(name):   # cut at the '(' of the argument list (outside template brackets)
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            name = name[:i]
            break
    name = re.sub(r"^void ", "", name)
    return re.sub(r"Fp<(\w+)>", r"\1", name)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curve", default="bls12_381")
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--root", default=HERE, help="checkout whose groth16_b200 package and library are measured")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default="", help="also write the result to this file")
    a = ap.parse_args()
    root = os.path.abspath(a.root)
    sys.path.insert(0, root)
    import torch
    from torch.profiler import ProfilerActivity, profile
    from bench import TOXIC
    from groth16_b200 import Groth16, _lib
    from groth16_b200.params import GENERATORS
    from groth16_b200.workload import synthetic_r1cs

    m, z_np, _ = synthetic_r1cs(a.curve, a.log_n, seed=1)
    g = Groth16(a.curve, 0)
    G = GENERATORS[g.curve.name]
    g.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=False)
    cd, nq = g.codec, g.nq
    r = np.ascontiguousarray(cd.fr.enc1(123456789))
    s = np.ascontiguousarray(cd.fr.enc1(987654321))
    z_dev = torch.from_numpy(z_np.view(np.int64)).pin_memory().to("cuda:0")
    flags = _lib.ASSIGNMENT_ON_DEVICE | _lib.SERIAL_MSMS
    proof = np.zeros(8 * nq, dtype=np.uint64)
    for _ in range(a.warmup):
        g.prove_raw(r, s, z_dev.data_ptr(), flags, proof)
    first = proof.copy()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.prove_raw(r, s, z_dev.data_ptr(), flags, proof)
        torch.cuda.synchronize()
    if not np.array_equal(first, proof):
        raise SystemExit("profiled proof differs from the warm-up proof")

    per_kernel = collections.defaultdict(lambda: [0.0, 0])
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA or e.name.startswith(("Memcpy", "Memset")):
            continue
        k = per_kernel[short_name(e.name)]
        k[0] += e.device_time_total / 1e3   # microseconds -> milliseconds
        k[1] += 1
    rows = sorted(per_kernel.items(), key=lambda kv: -kv[1][0])
    total = sum(v[0] for _, v in rows)
    tm = g.timings()
    out = {"curve": a.curve, "log_n": a.log_n, "root": root, "device": torch.cuda.get_device_name(0),
           "kernel_ms_total": round(total, 3), "msm_accum_ms": tm["msm_accum_ms"],
           "kernels": [{"name": n, "ms": round(v[0], 4), "launches": v[1]} for n, v in rows]}
    print(f"{'kernel':80s} {'ms':>9s} {'launches':>8s}")
    for n, (ms, cnt) in rows:
        print(f"{n[:80]:80s} {ms:9.3f} {cnt:8d}")
    print(f"{'total':80s} {total:9.3f}")
    print(json.dumps(out), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
