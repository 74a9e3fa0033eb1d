#!/usr/bin/env python3
"""Per-call time of tl/nvl allreduces posted eagerly against the same allreduces replayed from CUDA graphs, on one GPU.

    python tools/graph_bench.py [--ranks 1,2,4] [--k 16] [--iters 50] [--out FILE]

For every team size (a team of one, and N emulated ranks sharing cuda:0 in one process) and every size from 1 KB to 16 MB:
  eager:  K allreduces, each one ucc_collective_init + triggered_post on the rank's stream + test until complete + finalize,
          for every rank - the host path of every stream-ordered call
  graph:  the same K allreduces captured once per rank (torch.cuda.graph on the rank's stream), then the graphs of all ranks
          replayed together
Per-call time = host wall time of `iters` rounds, each ending in a device synchronize, over iters * K.  The card's name and power
limit are printed in the same run.  Several processes over several GPUs are not covered here (tests/test_dist_graph_gpu.py
checks the torch backend in graphs there).  Needs a CUDA device: without one the script fails."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

import torch  # noqa: E402

from ucc_b200 import capi as U  # noqa: E402
from ucc_b200.harness import UccJob, coll_args  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: power limit unknown)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", default="1,2,4")
    ap.add_argument("--k", type=int, default=16, help="allreduces per graph")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--sizes", default="1K,16K,256K,1M,4M,16M")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("graph_bench: no CUDA device")
    torch.cuda.set_device(0)
    units = {"K": 1 << 10, "M": 1 << 20}
    sizes = [int(s[:-1]) * units[s[-1]] if s[-1] in units else int(s) for s in a.sizes.split(",")]
    print(f"# card: {card()}", flush=True)
    rows = []
    for n in [int(x) for x in a.ranks.split(",")]:
        with UccJob(n, env={"UCC_TL_NVL_MAX_BLOCKS": "8"}) as job:
            team = job.create_team()
            streams = [torch.cuda.Stream() for _ in range(n)]
            ees = []
            for r in range(n):
                ep = U.ucc_ee_params_t()
                ep.ee_type, ep.ee_context, ep.ee_context_size = U.UCC_EE_CUDA_STREAM, streams[r].cuda_stream, 8
                ee = U.handle()
                U.check(U.ucc_ee_create(team.members[r].team, C.byref(ep), C.byref(ee)), "ee_create")
                ees.append(ee)
            for nbytes in sizes:
                count = nbytes // 4
                bufs = [[(torch.ones(count, device="cuda"), torch.zeros(count, device="cuda")) for _ in range(a.k)] for _ in range(n)]
                args = [[coll_args("allreduce", dt="float32", mem_type=U.UCC_MEMORY_TYPE_CUDA, src_ptr=s.data_ptr(), dst_ptr=d.data_ptr(),
                                   count_src=count, count_dst=count) for s, d in bufs[r]] for r in range(n)]

                def post(r, args_):
                    q = C.POINTER(U.ucc_coll_req_t)()
                    U.check(U.ucc_collective_init(C.byref(args_), C.byref(q), team.members[r].team), "init")
                    ev = U.ucc_ev_t()
                    ev.ev_type, ev.req = U.UCC_EVENT_COMPUTE_COMPLETE, C.cast(q, C.c_void_p)
                    U.check(U.ucc_collective_triggered_post(ees[r], C.byref(ev)), "triggered_post")
                    return q

                def drain(reqs, finalize=True):
                    while any(q.contents.status == U.UCC_INPROGRESS for q in reqs):
                        for r in range(n):
                            U.ucc_context_progress(job.procs[r].ctx)
                            e = C.POINTER(U.ucc_ev_t)()
                            while U.ucc_ee_get_event(ees[r], C.byref(e)) == U.UCC_OK:
                                U.ucc_ee_ack_event(ees[r], e)
                    assert all(q.contents.status == U.UCC_OK for q in reqs)
                    if finalize:
                        for q in reqs:
                            U.ucc_collective_finalize(q)

                def eager_round():
                    for k in range(a.k):
                        drain([post(r, args[r][k]) for r in range(n)])
                    torch.cuda.synchronize()
                for _ in range(3):
                    eager_round()
                t0 = time.perf_counter()
                for _ in range(a.iters):
                    eager_round()
                eager = (time.perf_counter() - t0) / (a.iters * a.k)
                graphs, held = [], []
                torch.cuda.synchronize()
                for r in range(n):
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g, stream=streams[r]):
                        reqs = [post(r, x) for x in args[r]]
                        for q in reqs:
                            while q.contents.status == U.UCC_INPROGRESS:
                                U.ucc_context_progress(job.procs[r].ctx)
                    held += reqs
                    graphs.append(g)

                def replay_round():
                    for r in range(n):
                        with torch.cuda.stream(streams[r]):
                            graphs[r].replay()
                    torch.cuda.synchronize()
                for _ in range(3):
                    replay_round()
                exp = float(n)
                assert all(bool((d == exp).all()) for r in range(n) for _, d in bufs[r]), "graph replay result"
                t0 = time.perf_counter()
                for _ in range(a.iters):
                    replay_round()
                graph = (time.perf_counter() - t0) / (a.iters * a.k)
                for q in held:
                    U.ucc_collective_finalize(q)
                del graphs
                row = {"ranks": n, "bytes": nbytes, "eager_us": round(eager * 1e6, 2), "graph_us": round(graph * 1e6, 2),
                       "speedup": round(eager / graph, 2)}
                rows.append(row)
                print(json.dumps(row), flush=True)
            for ee in ees:
                U.ucc_ee_destroy(ee)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card(), "k": a.k, "iters": a.iters, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
