"""tl/nvl END TO END WITHOUT A GPU: the plugin's host code is built unchanged against an emulated CUDA runtime
(tests/emu/cudart_emu.cpp: streams = worker threads, events, "device" memory registry) and the host-emulated kernels
(tests/emu/nvl_emu_launch.cpp), then driven through the public UCC API with N ranks in one process - team creation with a
pointer-shared heap, score selection / TUNE, launch ordering, the zero-copy exchange board (RAW pointers) with deferred launches,
persistent requests, several teams, multi-round messages, asymmetric memory staging in the core.  Every collective of tl/nvl,
staged and zero-copy, including the push exchange and the one-shot reduce_scatter."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_built = []


@pytest.fixture(scope="module")
def emu_build():
    """the host-emulated runtime and plugin; every module that imports this fixture shares one build per session"""
    if not os.path.exists("/usr/local/cuda/include/cuda_fp16.h"):
        pytest.skip("CUDA headers not installed")
    if _built:
        return
    out = subprocess.run(["bash", os.path.join(ROOT, "tests", "emu", "build_hostemu.sh")], capture_output=True, text=True, timeout=900)
    assert "HOSTEMU_BUILD_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]
    _built.append(True)


@pytest.mark.parametrize("scenario", ["allreduce", "colls_staged", "colls_zcopy", "colls_push", "colls_ce", "colls_ring", "misc", "triggered", "cross_team", "timeout", "p2p", "p2p_fuzz", "coll_fuzz", "memh", "lanes", "defaults", "hier"])
def test_tl_nvl_host_emulation(emu_build, scenario):
    env = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("UCC_TL_NVL_TUNE", "UCC_MODULE_DIR", "UCC_TLS"):
        env.pop(k, None)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostemu_worker.py"), scenario], env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "HOSTEMU_WORKER_OK" in out.stdout, out.stdout[-2500:] + out.stderr[-2500:]
    log = out.stdout + out.stderr
    if scenario == "hier":                                           # node sub-teams are forced to tl/nvl; the leaders sub-team spans fake hosts (host transport)
        assert "CL_HIER {schedule}" in log and "CL_BASIC" not in log
        return
    assert "{TL_NVL}" in log                                         # the collectives really ran on tl/nvl
    # nothing but the (memory-less) barrier may fall back to the host transport
    assert all("coll_init: barrier" in ln for ln in log.splitlines() if "{TL_SHM}" in ln), [ln for ln in log.splitlines() if "{TL_SHM}" in ln][:3]
