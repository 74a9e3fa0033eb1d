"""all_to_all_single with the output aliasing the input (ucc_b200.ops and the torch.distributed backend) on host tensors over tl/shm:
the call is posted as an in-place alltoall / alltoallv and gives the in-place result."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("n", [2, 3])
def test_aliased_all_to_all_single_host(n):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(29630 + n), os.path.join(ROOT, "tests", "inplace_a2a_worker.py"), "cpu"]
    out = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT, CUDA_VISIBLE_DEVICES=""), capture_output=True, text=True, timeout=600)
    assert "INPLACE_A2A_WORKER_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]
