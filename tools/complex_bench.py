#!/usr/bin/env python3
"""Per-call time of a complex64 allreduce on tl/nvl and on the route it replaces (UCC_TL_NVL_TUNE=allreduce:0: tl/nvl declines every
allreduce and tl/shm serves it), with N emulated ranks on one GPU (one process, one stream per rank).  The ranks share one GPU's HBM,
so the numbers are not NVLink figures.  Every rank's kernel spins until the others arrive, so all of them must be resident on the one
GPU at once: the grid is capped at 16 CTAs per rank (as in smoke() and the GPU tests) and every rank's stream gets its own hardware
queue.  Prints the card and its power limit, then one JSON line per (route, ranks, size).
    python tools/complex_bench.py [--ranks 4,8] [--bytes 4K,1M,64M]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # (before CUDA starts)
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ucc_b200 import capi as U  # noqa: E402
from ucc_b200.harness import UccJob, coll_args  # noqa: E402

ROUTES = {"tl_nvl": {}, "tl_shm": {"UCC_TL_NVL_TUNE": "allreduce:0"}}


def nbytes(s):
    return int(s[:-1]) << {"K": 10, "M": 20, "G": 30}[s[-1]] if s[-1] in "KMG" else int(s)


def per_call_us(team, n, count, min_time=1.0):
    src = [torch.randn(count, dtype=torch.complex64, device="cuda") for _ in range(n)]
    dst = [torch.empty_like(s) for s in src]
    args = [coll_args("allreduce", dt="float32_complex", mem_type=U.UCC_MEMORY_TYPE_CUDA, src_ptr=src[r].data_ptr(), dst_ptr=dst[r].data_ptr(),
                      count_src=count, count_dst=count, persistent=True) for r in range(n)]
    req = team.coll(args)
    torch.cuda.synchronize()
    for _ in range(3):                       # warm-up: module load, heap first touch
        assert req.run() == U.UCC_OK
    torch.cuda.synchronize()
    iters, t = 0, 0.0
    t0 = time.perf_counter()
    while t < min_time or iters < 5:         # every call ends in a device synchronise: per-call latency, not enqueue rate
        assert req.run() == U.UCC_OK
        torch.cuda.synchronize()
        iters += 1
        t = time.perf_counter() - t0
    req.finalize()
    exp = sum(s.to(torch.complex128) for s in src)
    assert torch.allclose(dst[0].to(torch.complex128), exp, rtol=1e-4, atol=1e-4)
    return t / iters * 1e6, iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", default="4,8")
    ap.add_argument("--bytes", default="4K,1M,64M")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    info = C.CDLL(os.path.join(os.path.dirname(U.LIB_PATH), "ucc", "libucc_tl_nvl.so")).ucc_tl_nvl_last_launch_info
    info.restype = C.c_char_p
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"gpu: {smi}", flush=True)
    for route, env in ROUTES.items():
        for n in (int(x) for x in a.ranks.split(",")):
            with UccJob(n, env=dict(env, UCC_TL_NVL_SYMMETRIC_SIZE="256Mb", UCC_TL_NVL_MAX_BLOCKS="16")) as j:
                team = j.create_team()
                for s in a.bytes.split(","):
                    us, iters = per_call_us(team, n, nbytes(s) // 8)
                    rec = {"route": route, "ranks": n, "bytes": nbytes(s), "us_per_call": round(us, 1), "iters": iters}
                    if route == "tl_nvl":
                        rec["kernel"] = info().decode()
                    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
