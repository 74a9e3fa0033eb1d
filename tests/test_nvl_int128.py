"""INT128 / UINT128 reductions on tl/nvl without a GPU: the plugin's datatype table, the contract of tests/nvl_int128.py on the
host-emulated plugin (tests/hostemu_int128_worker.py) for every path and teams of 2..5, and the kernels' synchronisation under
ThreadSanitizer (tests/emu/nvl_emu_int128.cpp through tools/run_emu_tsan.sh)."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import pytest

import test_nvl_complex as T  # the datatype / operator tables of the older types
from test_nvl_hostemu import emu_build  # noqa: F401  (module fixture: builds the host-emulated runtime and plugin)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = "/usr/local/cuda/include"


def test_int128_datatype_table():
    """every datatype of kernels/nvl_kernels.h: the older ones answer as test_nvl_complex.py pins them, the float128 slot after complex
    double has no kernels (host-only), INT128 / UINT128 after it are 16 bytes with every operator and nothing in the switch
    (multimem.ld_reduce has no 128-bit form), and nothing follows them"""
    so = os.path.join(ROOT, "ucc_b200", "lib", "ucc", "libucc_tl_nvl.so")
    if not os.path.exists(so):
        pytest.skip("tl/nvl plugin not built")
    lib = C.CDLL(so)
    lib.nvl_dt_size.restype = C.c_size_t
    dts = T.DTS + ["F128", "I128", "U128"]
    for d, dt in enumerate(dts):
        new = dt in ("I128", "U128")
        assert lib.nvl_dt_size(d) == (16 if new else T.SIZE.get(dt, 0)), dt
        for o, op in enumerate(T.OPS):
            assert bool(lib.nvl_dt_supports_op(d, o)) == (new or (dt in T.SIZE and T.expected_supports(dt, op))), (dt, op)
            assert bool(lib.nvl_nvls_supports(d, o)) == (dt in T.SIZE and T.expected_nvls(dt, op)), (dt, op)
    assert lib.nvl_dt_size(len(dts)) == 0 and not lib.nvl_dt_supports_op(len(dts), 0)


@pytest.mark.parametrize("path", ["oneshot", "twoshot", "zcopy", "ring", "rhd"])
def test_int128_reductions_host_emulation(emu_build, path):  # noqa: F811
    env = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("UCC_TL_NVL_TUNE", "UCC_MODULE_DIR", "UCC_TLS"):
        env.pop(k, None)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostemu_int128_worker.py"), path], env=env, capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0 and "HOSTEMU_WORKER_OK" in out.stdout, out.stdout[-2500:] + out.stderr[-2500:]


def test_int128_kernels_tsan():
    if not os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h")) or not shutil.which("g++"):
        pytest.skip("CUDA headers or g++ not installed")
    out = subprocess.run(["bash", os.path.join(ROOT, "tools", "run_emu_tsan.sh"), "nvl_emu_int128"], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "int128: tsan reports 0, result ok" in out.stdout, out.stdout[-2500:] + out.stderr[-2500:]
