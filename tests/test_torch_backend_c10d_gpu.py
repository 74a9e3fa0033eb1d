"""The "ucc_b200" torch.distributed backend beyond the basic collectives, on CUDA tensors (tl/nvl): the cases of
tests/test_torch_backend_c10d_cpu.py, each call checked to have launched a tl/nvl kernel, plus a gather and a list all_to_all
captured in a CUDA graph inside pg.graphed() and replayed (worker: tests/pg_c10d_worker.py).

One process per rank under torchrun, as the backend is used, with rank r on GPU r % device count, so that the test runs on a
single GPU too: tl/nvl builds a team of processes that share a device (the heap is exported by file descriptor, user buffers
are reached through CUDA IPC).  The processes' kernels then take turns on the device instead of running side by side, which
costs time but not correctness."""
import os
import subprocess
import sys

import pytest

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n", [3, 4])
def test_torch_backend_c10d_cuda(n):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(29780 + n), os.path.join(ROOT, "tests", "pg_c10d_worker.py"), "cuda"]
    out = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=170)
    assert "PG_C10D_WORKER_OK" in out.stdout, out.stdout[-4000:] + out.stderr[-4000:]
