"""Which kernel serves each collective on tl/nvl, without a GPU: tests/launch_paths_worker.py sweeps every algorithm that runs without
a multicast mapping, on teams of 1 to 4, staged and zero-copy, on the host-emulated plugin, and prints the launch note of each case.
The notes must match tests/golden/nvl_launch_paths.txt line for line: a change to how tl/nvl picks a kernel, its grid or its block
shows up here.  Regenerate the golden with `python tests/launch_paths_worker.py` (after tests/emu/build_hostemu.sh) only when a
change of the launch behaviour is intended."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "nvl_launch_paths.txt")


@pytest.fixture(scope="module")
def emu_plugin():
    if not os.path.exists("/usr/local/cuda/include/cuda_fp16.h"):
        pytest.skip("CUDA headers not installed")
    out = subprocess.run(["bash", os.path.join(ROOT, "tests", "emu", "build_hostemu.sh")], capture_output=True, text=True, timeout=900)
    assert "HOSTEMU_BUILD_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]


def test_launch_paths_match_golden(emu_plugin):
    env = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("UCC_TL_NVL_TUNE", "UCC_MODULE_DIR", "UCC_TLS"):
        env.pop(k, None)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "launch_paths_worker.py")], env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "LAUNCH_PATHS_OK" in out.stdout, out.stdout[-2500:] + out.stderr[-2500:]
    got = [ln for ln in out.stdout.splitlines() if " -> " in ln]
    with open(GOLDEN) as f:
        want = [ln for ln in f.read().splitlines() if ln]
    diff = [f"line {i + 1}: golden {w!r}, got {g!r}" for i, (w, g) in enumerate(zip(want, got)) if w != g]
    assert not diff and len(got) == len(want), (len(want), len(got), diff[:20])
