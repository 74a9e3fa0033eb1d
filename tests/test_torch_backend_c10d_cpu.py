"""The "ucc_b200" torch.distributed backend beyond the basic collectives, on host tensors (tl/shm), one process per rank under
torchrun: gather / scatter with equal and unequal blocks, list all_to_all, gather_object / scatter_object_list,
all_gather_coalesced, _coalescing_manager, torch.bool tensors and the refused operations (worker: tests/pg_c10d_worker.py)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("n", [3, 4])
def test_torch_backend_c10d_host(n):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(29680 + n), os.path.join(ROOT, "tests", "pg_c10d_worker.py"), "cpu"]
    env = dict(os.environ, PYTHONPATH=ROOT, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=150)
    assert "PG_C10D_WORKER_OK" in out.stdout, out.stdout[-4000:] + out.stderr[-3000:]
