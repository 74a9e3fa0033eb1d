"""float8 and complex32 CUDA tensors (tl/nvl) on the "ucc_b200" torch.distributed backend and in ucc_b200.ops / .parallel: the cases
of tests/test_torch_float8_cpu.py, each direct call checked to have launched a tl/nvl kernel, plus a float8 all_gather captured in a
CUDA graph inside pg.graphed() and replayed with new inputs (worker: tests/float8_worker.py).

One process per rank under torchrun, with rank r on GPU r % device count, so that the test runs on a single GPU too (see
tests/test_torch_backend_c10d_gpu.py).  Each part is a test of its own, so that one launch stays well inside the per-test limit."""
import os
import subprocess
import sys

import pytest

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
SECTIONS = {"small": "small,p2p", "big": "big", "stack": "stack", "reduce": "reduce,graph"}


@pytest.mark.parametrize("n", [3, 4])
@pytest.mark.parametrize("part", list(SECTIONS))
def test_torch_float8_cuda(n, part):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    port = 29950 + 10 * list(SECTIONS).index(part) + n
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "float8_worker.py"), "cuda", SECTIONS[part]]
    out = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=170)
    assert "FLOAT8_WORKER_OK" in out.stdout, out.stdout[-4000:] + out.stderr[-4000:]
