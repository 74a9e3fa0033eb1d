#!/usr/bin/env python3
"""Per-call time of allreduce, allgather and alltoall on CUDA managed buffers (cudaMallocManaged, through the library's memory
component), on tl/nvl and on the route managed buffers took before tl/nvl served them (UCC_TL_NVL_TUNE=<coll>:0: tl/nvl declines
and tl/shm serves it through host memory).  N emulated ranks on one GPU (one process, one stream per rank), so the numbers are not
NVLink figures.  Every result is checked against numpy.  Prints the card and its power limit, then one JSON line per
(route, collective, ranks, size); --out also writes them as one JSON list.
    python tools/managed_bench.py [--ranks 4] [--bytes 64K,1M,16M] [--out results.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # (before CUDA starts)
import numpy as np  # noqa: E402
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ucc_b200 import capi as U  # noqa: E402
from ucc_b200.harness import UccJob, coll_args  # noqa: E402

COLLS = ("allreduce", "allgather", "alltoall")
ROUTES = {"tl_nvl": {}, "tl_shm": {"UCC_TL_NVL_TUNE": "#".join(f"{c}:0" for c in COLLS)}}
MANAGED = U.UCC_MEMORY_TYPE_CUDA_MANAGED


def nbytes(s):
    return int(s[:-1]) << {"K": 10, "M": 20, "G": 30}[s[-1]] if s[-1] in "KMG" else int(s)


class Managed:
    def __init__(self, n):
        self.hdr = C.c_void_p()
        assert U.lib.ucc_mc_alloc(C.byref(self.hdr), n * 4, MANAGED) == 0
        self.ptr = C.c_void_p.from_address(self.hdr.value + 8).value
        self.a = np.frombuffer((C.c_char * (n * 4)).from_address(self.ptr), dtype=np.int32)

    def free(self):
        U.lib.ucc_mc_free(self.hdr)


def per_call_us(team, n, coll, count, min_time=1.0):
    """`count`: int32 elements of each rank's destination"""
    blk = count // n
    src_n = blk if coll == "allgather" else count
    src = [Managed(src_n) for _ in range(n)]
    dst = [Managed(count) for _ in range(n)]
    rng = np.random.default_rng(0)
    for s in src:
        s.a[:] = rng.integers(-50, 50, src_n).astype(np.int32)
    args = [coll_args(coll, dt="int32", mem_type=MANAGED, src_ptr=src[r].ptr, dst_ptr=dst[r].ptr, count_src=src_n, count_dst=count,
                      persistent=True) for r in range(n)]
    req = team.coll(args)
    torch.cuda.synchronize()
    for _ in range(3):                       # warm-up: module load, heap first touch, page migration of the inputs
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
    ins = [s.a.copy() for s in src]
    for r in range(n):
        if coll == "allreduce":
            exp = sum(x.astype(np.int64) for x in ins).astype(np.int32)
        elif coll == "allgather":
            exp = np.concatenate(ins)
        else:
            exp = np.concatenate([ins[p][r * blk:(r + 1) * blk] for p in range(n)])
        assert np.array_equal(dst[r].a, exp), (coll, n, count, r)
    for b in src + dst:
        b.free()
    return t / iters * 1e6, iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", default="4")
    ap.add_argument("--bytes", default="64K,1M,16M", help="size of each rank's destination")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    U.lib.ucc_mc_alloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t, C.c_int]
    U.lib.ucc_mc_free.argtypes = [C.c_void_p]
    info = C.CDLL(os.path.join(os.path.dirname(U.LIB_PATH), "ucc", "libucc_tl_nvl.so")).ucc_tl_nvl_last_launch_info
    info.restype = C.c_char_p
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"gpu: {smi}", flush=True)
    recs = []
    for route, env in ROUTES.items():
        for n in (int(x) for x in a.ranks.split(",")):
            with UccJob(n, env=dict(env, UCC_TL_NVL_SYMMETRIC_SIZE="256Mb", UCC_TL_NVL_MAX_BLOCKS="16")) as j:
                team = j.create_team()
                for coll in COLLS:
                    for s in a.bytes.split(","):
                        us, iters = per_call_us(team, n, coll, nbytes(s) // 4)
                        rec = {"gpu": smi, "route": route, "coll": coll, "ranks": n, "bytes": nbytes(s), "us_per_call": round(us, 1), "iters": iters}
                        if route == "tl_nvl":
                            rec["kernel"] = info().decode()
                        print(json.dumps(rec), flush=True)
                        recs.append(rec)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(recs, f, indent=1)


if __name__ == "__main__":
    main()
