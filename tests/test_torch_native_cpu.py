"""PyTorch's parallel stack on the "ucc_b200" backend with host tensors (tl/shm), one process per rank under torchrun: functional
collectives (eager and under torch.compile), DeviceMesh / DTensor, FSDP2, tensor parallel, uneven all_gather / reduce_scatter lists
and the PREMUL_SUM refusal (worker: tests/torch_native_worker.py)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SECTIONS = {"collectives": "funcol,uneven,refusals", "dtensor": "dtensor,tp", "fsdp": "fsdp"}


@pytest.mark.parametrize("n", [2, 4])
@pytest.mark.parametrize("part", list(SECTIONS))
def test_torch_native_host(n, part):
    port = 29810 + 10 * list(SECTIONS).index(part) + n
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "torch_native_worker.py"), "cpu", SECTIONS[part]]
    env = dict(os.environ, PYTHONPATH=ROOT, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="1")
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=170)
    assert "TORCH_NATIVE_OK" in out.stdout, out.stdout[-4000:] + out.stderr[-4000:]
