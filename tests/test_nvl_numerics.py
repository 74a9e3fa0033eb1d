"""The numerical contract of the tl/nvl reduction kernels (tests/nvl_numerics.py, tests/README.md) without a GPU: allreduce,
reduce_scatter(v) and reduce on every path, teams of 2..5, on the host-emulated plugin (tests/hostemu_numerics_worker.py)."""
import os
import subprocess
import sys

import pytest

from test_nvl_hostemu import emu_build  # noqa: F401  (module fixture: builds the host-emulated runtime and plugin)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("path", ["oneshot", "twoshot", "zcopy", "ring", "rhd"])
def test_reduction_numerics_host_emulation(emu_build, path):  # noqa: F811
    env = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("UCC_TL_NVL_TUNE", "UCC_MODULE_DIR", "UCC_TLS"):
        env.pop(k, None)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostemu_numerics_worker.py"), path], env=env, capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0 and "HOSTEMU_WORKER_OK" in out.stdout, out.stdout[-2500:] + out.stderr[-2500:]
