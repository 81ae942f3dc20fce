"""GPU probe of ONE rank of a `world`-way sharded proof on a single GPU (host-plumbed g16_prove_partial: no communicator
needed): per-phase timings for a few launch geometries, and -- under `ncu --profile-from-start off` -- the launch list of one
partial proof with the MSMs serialised.   python tools/probe_shard.py <curve> <log_n> <world> [tag]"""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from groth16_b200 import Groth16, _lib
from groth16_b200.params import GENERATORS
from groth16_b200.workload import synthetic_r1cs

curve, log_n, world = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
tag = sys.argv[4] if len(sys.argv) > 4 else "probe"
m, z, pub = synthetic_r1cs(curve, log_n, seed=1)
g = Groth16(curve, 0)
G = GENERATORS[g.curve.name]
pk = g.generate_parameters_with_qap(m, 11, 22, 33, 44, 55, G["g1"], G["g2"], export=True)
g.load_proving_key(pk, 0, world)
r = g.codec.fr.enc1(123456789)
out = np.zeros(g.partial_limbs(), dtype=np.uint64)
zd = torch.from_numpy(z.view(np.int64)).to("cuda:0")
ON = _lib.ASSIGNMENT_ON_DEVICE
lines = []
GRID = json.loads(os.environ["G16_PROBE_GRID"]) if os.environ.get("G16_PROBE_GRID") else [{}, {"msm_ba": 0, "msm_ba_g2": 0}]
for opts in GRID:
    base = {"msm_ba": 4, "msm_ba_g2": 4, "ba_m": 32, "ba_g": 16, "ba_min_entries_g1": 1 << 19, "ba_min_entries_g2": 1 << 19, "wm_first": -1}
    base.update(opts)
    for k, v in base.items():
        g.set_option(k, v)
    for i in range(3):
        g.prove_partial_raw(r, zd.data_ptr(), ON, out)
    torch.cuda.synchronize()
    t = time.perf_counter()
    n = 10
    for i in range(n):
        g.prove_partial_raw(r, zd.data_ptr(), ON, out)
    torch.cuda.synchronize()
    wall = 1e3 * (time.perf_counter() - t) / n
    tm = g.timings()
    # two partial proofs in flight (what bench.py's sharded arm does by default): throughput of this rank's share
    out2 = np.zeros_like(out)
    g.prove_partial_submit_raw(0, r, zd.data_ptr(), ON)
    for i in range(1, 4):
        g.prove_partial_submit_raw(i & 1, r, zd.data_ptr(), ON)
        g.prove_partial_wait_raw((i - 1) & 1, out2)
    g.prove_partial_wait_raw(3 & 1, out2)
    torch.cuda.synchronize()
    t = time.perf_counter()
    n2 = 20
    g.prove_partial_submit_raw(0, r, zd.data_ptr(), ON)
    for i in range(1, n2 + 1):
        if i < n2:
            g.prove_partial_submit_raw(i & 1, r, zd.data_ptr(), ON)
        g.prove_partial_wait_raw((i - 1) & 1, out2)
    torch.cuda.synchronize()
    wall2 = 1e3 * (time.perf_counter() - t) / n2
    assert np.array_equal(out, out2), "pipelined partial proof differs"
    g.prove_partial_raw(r, zd.data_ptr(), ON | _lib.SERIAL_MSMS, out)
    ts = g.timings()
    line = {"world": world, "opts": opts, "wall_ms": round(wall, 3), "wall_ms_two_in_flight": round(wall2, 3), "device_ms": round(tm["total_ms"], 3), "wm_ms": round(tm["witness_map_ms"], 3),
            "host_ms": round(tm["host_finish_ms"], 3), "msm_ms_concurrent": {k: round(v, 2) for k, v in tm["msm_ms"].items()},
            "msm_ms_serial": {k: round(v, 2) for k, v in ts["msm_ms"].items()}, "accum_ms_serial": {k: round(v, 2) for k, v in ts["msm_accum_ms"].items()},
            "launches": tm["launches"], "entries": tm["msm_entries"],
            "timeline_begin": {k: round(v, 2) for k, v in tm["msm_begin_ms"].items()}, "timeline_end": {k: round(v, 2) for k, v in tm["msm_end_ms"].items()}}
    print(json.dumps(line), flush=True)
    lines.append(line)
for k, v in {"msm_ba": 4, "msm_ba_g2": 4, "ba_m": 32, "ba_g": 16, "ba_min_entries_g1": 1 << 19, "ba_min_entries_g2": 1 << 19}.items():
    g.set_option(k, v)
g.prove_partial_raw(r, zd.data_ptr(), ON | _lib.SERIAL_MSMS, out)
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStart()
g.prove_partial_raw(r, zd.data_ptr(), ON | _lib.SERIAL_MSMS, out)
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStop()
with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out", f"{tag}_shard{world}.jsonl"), "w") as f:
    for l in lines:
        f.write(json.dumps(l) + "\n")
