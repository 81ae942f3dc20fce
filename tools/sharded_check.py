"""Run under torchrun (one rank per GPU): the sharded proof through the in-library NCCL exchange (g16_prove_sharded), the
host-plumbed exchange (g16_prove_partial -> torch.distributed all_gather -> g16_prove_assemble), the pipelined two-slot form
and the single-GPU proof must all be the same bytes, and equal to the CPU oracle's proof (rank 0).  With qap = circom the
circuit is proved under CircomReduction (witness map spread over the ranks with "wm_split"), and the proofs must equal the
LibsnarkReduction proof under the same toxic waste instead (for a satisfying witness the two reductions give the same proof).
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tools/sharded_check.py [curve] [log_n] [qap]
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from bench import TOXIC  # noqa: E402
from groth16_b200 import Groth16  # noqa: E402
from groth16_b200.dist import ShardedProver  # noqa: E402
from groth16_b200.params import GENERATORS  # noqa: E402
from groth16_b200.workload import synthetic_r1cs  # noqa: E402


def main():
    curve = sys.argv[1] if len(sys.argv) > 1 else "bls12_381"
    log_n = int(sys.argv[2]) if len(sys.argv) > 2 else 14
    qap = sys.argv[3] if len(sys.argv) > 3 else "libsnark"
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    m, z, pub = synthetic_r1cs(curve, log_n, seed=3)
    g = Groth16(curve, local, qap=qap)
    G = GENERATORS[g.curve.name]
    pk = g.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=True)
    cd, nq = g.codec, g.nq
    flat = lambda pf: np.concatenate([pf.a, pf.b, pf.c])
    for r_int, s_int in ((123456789, 987654321), (0, 5)):       # second pair: the r == 0 branch (prover.rs:98)
        r, s = cd.fr.enc1(r_int), cd.fr.enc1(s_int)
        g.load_proving_key(pk, 0, 1)
        single = flat(g.create_proof_with_reduction_and_matrices(None, r, s, None, m.num_instance_variables, m.num_constraints, z))
        sp = ShardedProver(g, pk, None, rank, world, dev, native=True)
        native = flat(sp.prove(r, s, z.ctypes.data, 0))
        sp.submit(0, r, z.ctypes.data, 0, s=s)
        sp.submit(1, r, z.ctypes.data, 0, s=s)
        piped = [flat(sp.finish(0, r, s)), flat(sp.finish(1, r, s))]
        hp = ShardedProver(g, pk, None, rank, world, dev, native=False)
        hosted = flat(hp.prove(r, s, z.ctypes.data, 0))
        assert np.array_equal(single, native), "in-library sharded proof != single-GPU proof"
        assert np.array_equal(single, piped[0]) and np.array_equal(single, piped[1]), "pipelined sharded proof differs"
        assert np.array_equal(single, hosted), "host-plumbed sharded proof != single-GPU proof"
        if rank == 0 and qap == "libsnark":
            import orc
            want, _ = orc.prove(cd.c.cid, nq, pk, m, z, r, s, threads=8)
            assert np.array_equal(single, want), "CUDA proof != CPU oracle proof"
        elif rank == 0:
            gl = Groth16(curve, local)
            gl.generate_parameters_with_qap(m, *TOXIC, G["g1"], G["g2"], export=False)
            want = flat(gl.create_proof_with_reduction_and_matrices(None, r, s, None, m.num_instance_variables, m.num_constraints, z))
            gl.close()
            assert np.array_equal(single, want), "CircomReduction proof != LibsnarkReduction proof"
    dist.barrier()
    if rank == 0:
        print(f"SHARDED_OK world={world} curve={curve} log_n={log_n}" + ("" if qap == "libsnark" else f" qap={qap}"))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
