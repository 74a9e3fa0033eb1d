"""In-place alltoall / alltoallv with one process per GPU: the members' buffers are CUDA IPC mappings, swapped pairwise by tl/nvl
(aliased all_to_all_single through ucc_b200.ops and through the torch.distributed backend)."""
import os
import subprocess
import sys

import pytest

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def test_multiproc_inplace_alltoall():
    n = min(2, torch.cuda.device_count()) if torch.cuda.is_available() else 0
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29765", os.path.join(ROOT, "tests", "inplace_a2a_worker.py"), "cuda"]
    out = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=300)
    assert "INPLACE_A2A_WORKER_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]
