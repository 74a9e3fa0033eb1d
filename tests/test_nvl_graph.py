"""tl/nvl collectives in CUDA graphs without a GPU: the host-emulated plugin with an emulated stream capture
(tests/emu/build_hostemu_graph.sh).  Every collective type, on the one-shot, staged, ring, push / swap and send / recv paths, in
place and not, is captured rank by rank and replayed three times with new inputs; persistent requests whose eager post resolved the zero-copy tables keep the direct form in
the graph; eager and replayed collectives alternate on one stream; a replay that times out is reported by the device-error query.
Worker: tests/hostemu_graph_worker.py."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu_build():
    if not os.path.exists("/usr/local/cuda/include/cuda_fp16.h"):
        pytest.skip("CUDA headers not installed")
    out = subprocess.run(["bash", os.path.join(ROOT, "tests", "emu", "build_hostemu_graph.sh")], capture_output=True, text=True, timeout=900)
    assert "HOSTEMU_GRAPH_BUILD_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]


def test_graph_capture_and_replay(emu_build):
    env = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("UCC_TL_NVL_TUNE", "UCC_MODULE_DIR", "UCC_TLS"):
        env.pop(k, None)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostemu_graph_worker.py"), "graphs"], env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "HOSTEMU_WORKER_OK" in out.stdout, out.stdout[-2500:] + out.stderr[-2500:]
    assert "{TL_NVL}" in out.stdout + out.stderr
