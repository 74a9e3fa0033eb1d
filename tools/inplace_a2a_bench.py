#!/usr/bin/env python3
"""Per-call time of an in-place float32 alltoall on tl/nvl (the swap path) and on the route it replaces
(UCC_TL_NVL_TUNE=alltoall:0#alltoallv:0: tl/nvl declines and tl/shm serves it with a scratch copy and a host-driven pairwise program),
with N emulated ranks on one GPU (one process, one stream per rank).  The ranks share one GPU's HBM, so the numbers are not NVLink
figures.  Every rank's kernel spins until the others arrive, so all of them must be resident on the one GPU at once: the grid is capped
at 16 CTAs per rank (as in smoke() and the GPU tests) and every rank's stream gets its own hardware queue.  Each call is a fresh
(non-persistent) request, the way MPI_Alltoall(MPI_IN_PLACE) arrives through a collective component, and ends in a device
synchronise.  Besides the time, every record has the device memory the route allocated and still held after its calls (cudaMemGetInfo
before the first call and after the last; a scratch buffer freed before the call returns does not show).  Prints the card and its
power limit, then one JSON line per (route, ranks, size).
    python tools/inplace_a2a_bench.py [--ranks 4,8] [--bytes 4K,1M,64M]"""
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

ROUTES = {"tl_nvl": {}, "tl_shm": {"UCC_TL_NVL_TUNE": "alltoall:0#alltoallv:0"}}


def nbytes(s):
    return int(s[:-1]) << {"K": 10, "M": 20, "G": 30}[s[-1]] if s[-1] in "KMG" else int(s)


def call(team, bufs, count):
    req = team.coll([coll_args("alltoall", dt="float32", mem_type=U.UCC_MEMORY_TYPE_CUDA, dst_ptr=b.data_ptr(), count_dst=count, inplace=True)
                     for b in bufs])
    assert req.run() == U.UCC_OK
    req.finalize()
    torch.cuda.synchronize()


def measure(team, n, size, min_time=1.0):
    """`size` bytes per rank's buffer; returns (us per call, calls, MB held, result correct)"""
    count = size // 4 // n * n
    blk = count // n
    bufs = [torch.arange(count, dtype=torch.float32, device="cuda") + 1e6 * r for r in range(n)]
    orig = [b.cpu() for b in bufs]           # (the check runs on the host: no device allocation of torch's between the two readings)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    call(team, bufs, count)                  # also the check: one exchange from the known contents
    ok = all(torch.equal(bufs[r].cpu(), torch.cat([orig[p][r * blk:(r + 1) * blk] for p in range(n)])) for r in range(n))
    for _ in range(2):                       # warm-up: module load, heap first touch, IPC mapping cache
        call(team, bufs, count)
    iters, t = 0, 0.0
    t0 = time.perf_counter()
    while t < min_time or iters < 5:
        call(team, bufs, count)
        iters += 1
        t = time.perf_counter() - t0
    held = (free0 - torch.cuda.mem_get_info()[0]) / 2**20
    return t / iters * 1e6, iters, held, ok


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
            with UccJob(n, env=dict(env, UCC_TL_NVL_SYMMETRIC_SIZE="80Mb", UCC_TL_NVL_MAX_BLOCKS="16")) as j:
                team = j.create_team()
                for s in a.bytes.split(","):
                    us, iters, held, ok = measure(team, n, nbytes(s))
                    rec = {"route": route, "ranks": n, "bytes": nbytes(s), "us_per_call": round(us, 1), "iters": iters,
                           "extra_device_mb": round(held, 1), "correct": ok}
                    if route == "tl_nvl":
                        rec["kernel"] = info().decode()
                    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
