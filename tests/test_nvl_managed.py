"""tl/nvl on CUDA managed memory without a GPU: the host-emulated plugin (tests/emu/build_hostemu.sh) serves every collective
with buffers, send / recv, persistent and triggered requests, a team of one and the forced push movers on managed and mixed managed / device buffers,
with UCC_TLS=nvl, byte-exact against numpy; no direct (zero-copy) form ever maps a managed buffer; ucc_mem_map still refuses a
managed segment.  Worker: tests/hostemu_managed_worker.py, cases: tests/nvl_managed.py."""
import os
import subprocess
import sys

import pytest

from test_nvl_hostemu import emu_build  # noqa: F401  (session fixture: builds the host-emulated runtime and plugin)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("scenario", ["colls", "persistent", "p2p", "push", "triggered", "self", "mem_map"])
def test_managed_memory(emu_build, scenario):  # noqa: F811
    env = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("UCC_TL_NVL_TUNE", "UCC_MODULE_DIR", "UCC_TLS"):
        env.pop(k, None)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostemu_managed_worker.py"), scenario], env=env,
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "HOSTEMU_WORKER_OK" in out.stdout, out.stdout[-2500:] + out.stderr[-2500:]
