"""In-place alltoall / alltoallv on tl/nvl without a GPU: the swap kernel and the heap-staged fallback in the host emulation
(tests/emu/nvl_emu_swap.cpp), checked byte for byte against a NumPy oracle, and the public API on the host-emulated plugin
(tests/hostemu_swap_worker.py)."""
import glob
import os
import subprocess
import sys

import numpy as np
import pytest

from test_nvl_hostemu import emu_build  # noqa: F401  (module fixture: builds the host-emulated runtime and plugin)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = "/usr/local/cuda/include"


def init_bytes(r, n):
    """what tests/emu/nvl_emu_swap.cpp init_byte(r, i) puts at offset i of rank r's buffer"""
    i = np.arange(n, dtype=np.uint64)
    x = i * np.uint64(0x9E3779B1) + np.uint64(r) * np.uint64(0x85EBCA77)
    return ((x ^ (x >> np.uint64(15))) & np.uint64(0xFF)).astype(np.uint8)


def oracle(N, nbytes, off, ln):
    """rank r's region for p receives the common prefix of p's region for r; own regions, gaps and the rest stay"""
    before = [init_bytes(r, nbytes) for r in range(N)]
    out = [b.copy() for b in before]
    for r in range(N):
        for p in range(N):
            if p != r:
                L = min(ln[r, p], ln[p, r])
                out[r][off[r, p]:off[r, p] + L] = before[p][off[p, r]:off[p, r] + L]
    return out


def test_swap_kernels_host_emulation(tmp_path):
    if not os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h")):
        pytest.skip("CUDA headers not installed")
    exe = tmp_path / "nvl_emu_swap"
    k = os.path.join(ROOT, "src", "components", "tl", "nvl", "kernels")
    cc = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-pthread", f"-I{CUDA_INC}", f"-I{k}", f"-I{ROOT}/include", f"-I{ROOT}/src",
                         os.path.join(ROOT, "tests", "emu", "nvl_emu_swap.cpp"), "-o", str(exe)], capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-4000:]
    dump = tmp_path / "cases"
    dump.mkdir()
    out = subprocess.run([str(exe), "swap", str(dump)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "NVL_EMU_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-2000:]
    files = sorted(glob.glob(str(dump / "case_*.bin")))
    seen = set()
    for f in files:
        raw = np.fromfile(f, dtype=np.uint8)
        N, nbytes, staged, lookup = (int(v) for v in raw[:32].view(np.uint64))
        off = raw[32:32 + 8 * N * N].view(np.uint64).astype(np.int64).reshape(N, N)
        ln = raw[32 + 8 * N * N:32 + 16 * N * N].view(np.uint64).astype(np.int64).reshape(N, N)
        got = raw[32 + 16 * N * N:].reshape(N, nbytes) if nbytes else np.zeros((N, 0), np.uint8)
        exp = oracle(N, nbytes, off, ln)
        for r in range(N):
            assert np.array_equal(got[r], exp[r]), (os.path.basename(f), N, staged, lookup, r)
        seen.add((N, bool(staged), bool(lookup), bool((ln != ln.T).any()), int(ln[0, 1]) if not lookup else -1))
    # every team size, both paths, alltoall at blocks 0 / 1 / 15 / 16 / 4097 / > 1 MB, alltoallv, and the mismatched pair on the swap path
    for N in (2, 3, 4, 8):
        for staged in (False, True):
            blocks = {s[4] for s in seen if s[:3] == (N, staged, False)}
            assert {0, 1, 15, 16, 4097} <= blocks and max(blocks) > (1 << 20), (N, staged, blocks)
            assert (N, staged, True, False, -1) in seen
        assert (N, False, True, True, -1) in seen


@pytest.mark.parametrize("scenario", ["zcopy", "staged", "persistent", "memh", "big_team", "tune"])
def test_inplace_alltoall_host_emulation(emu_build, scenario):  # noqa: F811
    """in-place alltoall / alltoallv through ucc_collective_init: every rank's request is served by tl/nvl, with the swap kernel
    or (UCC_TL_NVL_ZCOPY=n) the staged one"""
    env = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("UCC_TL_NVL_TUNE", "UCC_MODULE_DIR", "UCC_TLS"):
        env.pop(k, None)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostemu_swap_worker.py"), scenario], env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "HOSTEMU_WORKER_OK" in out.stdout, out.stdout[-2500:] + out.stderr[-2500:]
    inits = [ln for ln in (out.stdout + out.stderr).splitlines() if "coll_init: alltoall" in ln and " inplace" in ln]
    assert len(inits) >= 4, len(inits)
    assert all("{TL_NVL}" in ln for ln in inits), [ln for ln in inits if "{TL_NVL}" not in ln][:3]
