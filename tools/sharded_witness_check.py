"""Run under torchrun (one rank per GPU): a sharded proof of an unsatisfied assignment with G16_CHECK_WITNESS through the
in-library NCCL exchange (g16_prove_sharded) must be refused on every rank, pipelined in either slot as well, and the next
satisfied sharded proof on the same communicator must equal the single-GPU proof: the refusal left every collective matched.
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29541 tools/sharded_witness_check.py
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import TOXIC  # noqa: E402
from groth16_b200 import CHECK_WITNESS, Groth16, Unsatisfiable  # noqa: E402
from groth16_b200.dist import ShardedProver  # noqa: E402
from groth16_b200.params import GENERATORS  # noqa: E402
from groth16_b200.workload import synthetic_r1cs  # noqa: E402


def refused(fn, want):
    try:
        fn()
    except Unsatisfiable as e:
        assert want in str(e), str(e)
        return
    raise AssertionError("an unsatisfied sharded proof was not refused")


def main():
    curve, log_n = "bls12_381", 12
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    m, z, _ = synthetic_r1cs(curve, log_n, seed=5)
    g = Groth16(curve, local)
    G = GENERATORS[curve]
    pk = g.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=True)
    cd = g.codec
    flat = lambda pf: np.concatenate([pf.a, pf.b, pf.c])
    r, s = cd.fr.enc1(123456789), cd.fr.enc1(987654321)
    single = flat(g.create_proof_with_reduction_and_matrices(None, r, s, None, m.num_instance_variables, m.num_constraints, z))
    zi = cd.fr.dec(z)
    row = 100
    zi[int(m.c[1][row])] = (zi[int(m.c[1][row])] + 1) % g.curve.r   # breaks constraint `row` first
    bad = np.ascontiguousarray(cd.fr.enc(zi))
    sp = ShardedProver(g, pk, None, rank, world, dev, native=True)
    refused(lambda: sp.prove(r, s, bad.ctypes.data, CHECK_WITNESS), f"constraint {row} unsatisfied")
    assert np.array_equal(flat(sp.prove(r, s, z.ctypes.data, CHECK_WITNESS)), single), "sharded proof after a refusal"
    sp.submit(0, r, bad.ctypes.data, CHECK_WITNESS, s=s)
    sp.submit(1, r, z.ctypes.data, CHECK_WITNESS, s=s)
    refused(lambda: sp.finish(0, r, s), f"constraint {row} unsatisfied")
    assert np.array_equal(flat(sp.finish(1, r, s)), single), "slot 1 beside a refused slot 0"
    assert np.array_equal(flat(sp.prove(r, s, z.ctypes.data, 0)), single), "unflagged sharded proof after the refusals"
    dist.barrier()
    if rank == 0:
        print(f"SHARDED_CHECK_OK world={world} curve={curve} log_n={log_n}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
