"""tl/nvl collectives in CUDA graphs without a GPU: the host-emulated plugin with an emulated stream capture
(tests/emu/build_hostemu.sh).  Every collective type, on the one-shot, staged, ring, push / swap and send / recv paths, in
place and not, is captured rank by rank and replayed three times with new inputs; persistent requests whose eager post resolved the zero-copy tables keep the direct form in
the graph; eager and replayed collectives alternate on one stream; a replay that times out is reported by the device-error query.
Worker: tests/hostemu_graph_worker.py."""
import os
import subprocess
import sys

from test_nvl_hostemu import emu_build  # noqa: F401  (module fixture: builds the host-emulated runtime and plugin)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_graph_capture_and_replay(emu_build):  # noqa: F811
    env = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("UCC_TL_NVL_TUNE", "UCC_MODULE_DIR", "UCC_TLS"):
        env.pop(k, None)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostemu_graph_worker.py"), "graphs"], env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "HOSTEMU_WORKER_OK" in out.stdout, out.stdout[-2500:] + out.stderr[-2500:]
    assert "{TL_NVL}" in out.stdout + out.stderr
