"""UCC_COLL_ARGS_HINT_OPTIMIZE_OVERLAP_GPU on tl/nvl without a GPU: the host-emulated plugin (tests/emu/build_hostemu.sh) serves
every collective the hint reaches on its copy-engine path - reductions bitwise equal to the zero-copy two-shot kernel, in rounds
when the heap is small, data movement byte-exact - and falls back to the ordinary staged kernels on managed buffers and captured
posts.  Worker: tests/hostemu_overlap_worker.py, cases: tests/nvl_overlap.py."""
import os
import subprocess
import sys

import pytest

from test_nvl_hostemu import emu_build  # noqa: F401  (session fixture: builds the host-emulated runtime and plugin)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("scenario", ["numerics2", "numerics3", "numerics4", "rounds", "colls", "persistent", "fallbacks", "captured"])
def test_overlap_hint(emu_build, scenario):  # noqa: F811
    env = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("UCC_TL_NVL_TUNE", "UCC_MODULE_DIR", "UCC_TLS"):
        env.pop(k, None)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostemu_overlap_worker.py"), scenario], env=env,
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "HOSTEMU_WORKER_OK" in out.stdout, out.stdout[-2500:] + out.stderr[-2500:]
