"""Complex allreduce with one process per GPU: complex float SUM through the NVSwitch (NVLS variants forced) and complex double PROD
on the default algorithms."""
import os
import subprocess
import sys

import pytest

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dt,op,env", [
    ("c64", "sum", {"UCC_TL_NVL_TUNE": "allreduce:cuda:inf:@nvls", "UCC_TL_NVL_ALLREDUCE_ONESHOT_THRESH": "0"}),
    ("c128", "prod", {}),
])
def test_multiproc_complex_allreduce(dt, op, env):
    n = min(2, torch.cuda.device_count()) if torch.cuda.is_available() else 0
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29760", os.path.join(ROOT, "tests", "dist_complex_worker.py"), dt, op]
    out = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT, **env), capture_output=True, text=True, timeout=150)
    assert "DIST_COMPLEX_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]
