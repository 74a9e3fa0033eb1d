"""PyTorch's parallel stack on the "ucc_b200" backend with CUDA tensors (tl/nvl): the cases of tests/test_torch_native_cpu.py, each
direct collective checked to have launched a tl/nvl kernel, plus Work.wait() ordering the caller's stream behind a collective
posted on another stream, below and above the zero-copy threshold (worker: tests/torch_native_worker.py).

One process per rank under torchrun, with rank r on GPU r % device count, so that the test runs on a single GPU too (see
tests/test_torch_backend_c10d_gpu.py).  Each part is a test of its own, so that one launch stays well inside the per-test limit."""
import os
import subprocess
import sys

import pytest

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
SECTIONS = {"collectives": "funcol,uneven,stream,refusals", "dtensor": "dtensor,tp", "fsdp": "fsdp"}


@pytest.mark.parametrize("n", [3, 4])
@pytest.mark.parametrize("part", list(SECTIONS))
def test_torch_native_cuda(n, part):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    port = 29850 + 10 * list(SECTIONS).index(part) + n
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "torch_native_worker.py"), "cuda", SECTIONS[part]]
    out = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=170)
    assert "TORCH_NATIVE_OK" in out.stdout, out.stdout[-4000:] + out.stderr[-4000:]
