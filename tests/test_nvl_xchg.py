"""The byte contract of the tl/nvl data-movement collectives (tests/nvl_xchg.py, tests/README.md) without a GPU: allgather(v),
alltoall(v), bcast, gather(v) and scatter(v) on every path, teams of 2..5 and a team of one, on the host-emulated plugin
(tests/hostemu_xchg_worker.py).  The emulated push_bulk path runs the thread-copy push kernel: the TMA mover is covered by
tests/test_nvl_xchg_gpu.py only."""
import os
import subprocess
import sys

import pytest

from test_nvl_hostemu import emu_build  # noqa: F401  (module fixture: builds the host-emulated runtime and plugin)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("path", ["staged", "zcopy", "push", "push_bulk", "ce", "ring", "self"])
def test_xchg_contract_host_emulation(emu_build, path):  # noqa: F811
    env = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("UCC_TL_NVL_TUNE", "UCC_MODULE_DIR", "UCC_TLS"):
        env.pop(k, None)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostemu_xchg_worker.py"), path], env=env, capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0 and "HOSTEMU_WORKER_OK" in out.stdout, out.stdout[-2500:] + out.stderr[-2500:]
