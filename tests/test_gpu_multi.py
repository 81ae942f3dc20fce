"""Multi-GPU tier (needs >= 2 H100s on the box; skipped otherwise): one process per GPU under torchrun, NCCL inside the
library.  `python -m pytest tests/test_gpu_multi.py -m gpu` on a multi-GPU box runs it; the N > 1 host logic is also
covered on CPU with gloo (tests/test_dist_cpu.py)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.parametrize("curve,log_n", [("bls12_381", 14), ("bn254", 17)])
def test_sharded_proof_over_nccl(curve, log_n):
    n = min(_ngpus(), 4)
    if n < 2:
        pytest.skip("needs at least 2 GPUs (the in-library exchange is an NCCL all-gather between processes)")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29533", os.path.join(ROOT, "tools", "sharded_check.py"), curve, str(log_n)]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and f"SHARDED_OK world={n}" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
