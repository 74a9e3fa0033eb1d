"""float8 and complex32 host tensors (tl/shm) on the "ucc_b200" torch.distributed backend and in ucc_b200.ops / .parallel, one
process per rank under torchrun: every data-movement operation byte for byte with guard bytes around every output, send / recv,
functional collectives (eager and under torch.compile), DTensor, MoE dispatch / combine, complex32 SUM / AVG, the refusal of every
other reduction of these dtypes, and graphed() requests keyed by dtype (worker: tests/float8_worker.py)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SECTIONS = {"small": "small,p2p", "big": "big", "stack": "stack", "reduce": "reduce,graph"}


@pytest.mark.parametrize("n", [3, 4])
@pytest.mark.parametrize("part", list(SECTIONS))
def test_torch_float8_host(n, part):
    port = 29900 + 10 * list(SECTIONS).index(part) + n
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "float8_worker.py"), "cpu", SECTIONS[part]]
    env = dict(os.environ, PYTHONPATH=ROOT, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="1")
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=170)
    assert "FLOAT8_WORKER_OK" in out.stdout, out.stdout[-4000:] + out.stderr[-4000:]
