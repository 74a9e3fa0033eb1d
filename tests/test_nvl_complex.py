"""Complex float / double reductions on tl/nvl without a GPU: the kernels in the host emulation (tests/emu/nvl_emu_complex.cpp), the
plugin's datatype tables, and the public API on the host-emulated plugin (tests/hostemu_complex_worker.py)."""
import ctypes as C
import os
import subprocess
import sys

import pytest

from test_nvl_hostemu import emu_build  # noqa: F401  (module fixture: builds the host-emulated runtime and plugin)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = "/usr/local/cuda/include"

# kernels/nvl_kernels.h
DTS = ["I8", "I16", "I32", "I64", "U8", "U16", "U32", "U64", "F16", "F32", "F64", "BF16", "C64", "C128"]
OPS = ["SUM", "PROD", "MAX", "MIN", "LAND", "LOR", "LXOR", "BAND", "BOR", "BXOR", "AVG"]
SIZE = {"I8": 1, "I16": 2, "I32": 4, "I64": 8, "U8": 1, "U16": 2, "U32": 4, "U64": 8, "F16": 2, "F32": 4, "F64": 8, "BF16": 2, "C64": 8, "C128": 16}


def expected_supports(dt, op):
    if dt in ("F16", "F32", "F64", "BF16"):
        return op in ("SUM", "PROD", "MAX", "MIN", "AVG")
    if dt in ("C64", "C128"):
        return op in ("SUM", "PROD", "AVG")
    return True


def expected_nvls(dt, op):
    if dt in ("F32", "BF16", "F16", "C64"):
        return op in ("SUM", "AVG")
    if dt in ("I32", "U32", "I64", "U64"):
        return op in ("SUM", "MIN", "MAX", "BAND", "BOR", "BXOR")
    return False


def test_datatype_tables():
    """the old (datatype, operator) pairs answer as before; complex types get SUM / PROD / AVG, complex float SUM / AVG in the switch"""
    so = os.path.join(ROOT, "ucc_b200", "lib", "ucc", "libucc_tl_nvl.so")
    if not os.path.exists(so):
        pytest.skip("tl/nvl plugin not built")
    lib = C.CDLL(so)
    lib.nvl_dt_size.restype = C.c_size_t
    for d, dt in enumerate(DTS):
        assert lib.nvl_dt_size(d) == SIZE[dt], dt
        for o, op in enumerate(OPS):
            assert bool(lib.nvl_dt_supports_op(d, o)) == expected_supports(dt, op), (dt, op)
            assert bool(lib.nvl_nvls_supports(d, o)) == expected_nvls(dt, op), (dt, op)
    assert lib.nvl_dt_size(len(DTS)) == 0 and not lib.nvl_dt_supports_op(len(DTS), 0)


def test_complex_kernels_host_emulation(tmp_path):
    if not os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h")):
        pytest.skip("CUDA headers not installed")
    exe = tmp_path / "nvl_emu_complex"
    k = os.path.join(ROOT, "src", "components", "tl", "nvl", "kernels")
    cc = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-pthread", f"-I{CUDA_INC}", f"-I{k}", f"-I{ROOT}/include", f"-I{ROOT}/src",
                         os.path.join(ROOT, "tests", "emu", "nvl_emu_complex.cpp"), "-o", str(exe)], capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-4000:]
    out = subprocess.run([str(exe), "complex"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "NVL_EMU_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-2000:]


def test_complex_collectives_host_emulation(emu_build):  # noqa: F811
    """allreduce / reduce_scatter(v) / reduce on complex float and double, staged and zero-copy, in place and persistent: every rank's
    collective is served by tl/nvl, and a complex MAX never reaches it"""
    env = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("UCC_TL_NVL_TUNE", "UCC_MODULE_DIR", "UCC_TLS"):
        env.pop(k, None)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostemu_complex_worker.py")], env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "HOSTEMU_WORKER_OK" in out.stdout, out.stdout[-2500:] + out.stderr[-2500:]
    inits = [ln for ln in (out.stdout + out.stderr).splitlines() if "coll_init:" in ln and "_complex" in ln]
    served = [ln for ln in inits if " max:" not in ln]
    assert len(served) > 500, len(served)
    assert all("{TL_NVL}" in ln for ln in served), [ln for ln in served if "{TL_NVL}" not in ln][:3]
    assert not any("{TL_NVL}" in ln for ln in inits if " max:" in ln)
