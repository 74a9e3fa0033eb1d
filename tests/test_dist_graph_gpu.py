"""The "ucc_b200" torch.distributed backend inside torch.cuda.graph, one process per GPU (worker: tests/dist_graph_worker.py):
allreduce, allgather, reduce_scatter, alltoall, broadcast and isend / irecv captured and replayed exactly."""
import os
import subprocess
import sys

import pytest

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def test_torch_backend_in_cuda_graphs():
    n = min(4, torch.cuda.device_count()) if torch.cuda.is_available() else 0
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29797", os.path.join(ROOT, "tests", "dist_graph_worker.py")]
    out = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=300)
    assert out.stdout.count("DIST_GRAPH_WORKER_OK") == n, out.stdout[-2000:] + out.stderr[-4000:]
