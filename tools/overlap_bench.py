#!/usr/bin/env python3
"""How much of a GEMM's speed a collective running next to it takes away, with and without UCC_COLL_ARGS_HINT_OPTIMIZE_OVERLAP_GPU.

One GPU, N emulated ranks in this process (--ranks): a bf16 GEMM loop runs on its own torch stream, first alone, then while a
second thread keeps every rank's collectives going on the library's streams - allreduce, reduce_scatter and allgather at 64 MB and
256 MB per rank, each without and with the hint.  The arms alternate and every one runs --reps times.  Reported per arm: the GEMM
loop's time (CUDA events) and its slowdown against the GEMM alone measured in the same repetition, and the per-call time of the
collective (host clock around post + completion, averaged over the calls that ran while the GEMM loop did).  The card's name,
power limit and SM clock are read at the start of the same run.

With emulated ranks on one GPU the copy engines and the kernels move data inside that GPU's HBM: nothing here measures NVLink.
Usage: python tools/overlap_bench.py [--ranks 4] [--reps 3] [--gemm 8192] [--iters 40] [--json out.json]"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

COLLS = ("allreduce", "reduce_scatter", "allgather")
SIZES = (64 << 20, 256 << 20)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [x.strip() for x in out.strip().split(",")]))
    except (OSError, subprocess.SubprocessError) as e:
        return {"error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--gemm", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--json")
    o = ap.parse_args()
    # the emulated ranks share this GPU: one hardware queue per stream, or a copy-engine transfer queued behind one rank's barrier
    # kernel holds up another rank's barrier kernel that shares its queue
    os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    import torch
    from ucc_b200 import capi as U
    from ucc_b200.harness import UccJob, coll_args

    if not torch.cuda.is_available():
        sys.exit("overlap_bench: no CUDA device")
    torch.cuda.set_device(0)
    info = card()
    print(json.dumps({"card": info}), flush=True)
    n = o.ranks
    gs = torch.cuda.Stream()
    a = torch.randn(o.gemm, o.gemm, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(o.gemm, o.gemm, device="cuda", dtype=torch.bfloat16)
    c = torch.empty_like(a)

    def gemm_loop():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(gs):
            e0.record()
            for _ in range(o.iters):
                torch.mm(a, b, out=c)
            e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    # the default heap stages a 256 MB block where a request without the hint needs it.  The kernels of all emulated ranks must be
    # resident together (their CTAs wait for each other), so every rank gets its share of the SMs: 2 CTAs per SM / ranks
    env = {"UCC_TLS": "nvl", "UCC_TL_NVL_MAX_BLOCKS": str(max(1, 2 * torch.cuda.get_device_properties(0).multi_processor_count // (2 * n)))}
    with UccJob(n, env=env) as j:
        team = j.create_team(range(n), team_id=n)
        bufs = {}

        def request(coll, size, hint):
            cnt = size // 4
            if (coll, size) not in bufs:
                src = [torch.randn(cnt, device="cuda") for _ in range(n)]
                dst = [torch.empty(cnt if coll == "allreduce" else (cnt // n if coll == "reduce_scatter" else cnt * n), device="cuda") for _ in range(n)]
                bufs[(coll, size)] = (src, dst)
            src, dst = bufs[(coll, size)]
            args = []
            for r in range(n):
                s_cnt = cnt
                d_cnt = dst[r].numel()
                x = coll_args(coll, dt="float32", mem_type=U.UCC_MEMORY_TYPE_CUDA, src_ptr=src[r].data_ptr(), dst_ptr=dst[r].data_ptr(),
                              count_src=s_cnt, count_dst=d_cnt, persistent=True)
                if hint:
                    x.mask |= U.UCC_COLL_ARGS_FIELD_FLAGS
                    x.flags |= U.UCC_COLL_ARGS_HINT_OPTIMIZE_OVERLAP_GPU
                args.append(x)
            return team.coll(args)

        arms = [(coll, size, hint) for coll in COLLS for size in SIZES for hint in (False, True)]
        reqs = {arm: request(*arm) for arm in arms}
        for arm, q in reqs.items():   # warm-up: resolve the tables, load the modules
            assert q.run() == U.UCC_OK, arm
        torch.cuda.synchronize()
        gemm_loop()
        results = {arm: [] for arm in arms}
        for rep in range(o.reps):
            alone = gemm_loop()
            for arm in (arms if rep % 2 == 0 else arms[::-1]):
                q, stop, calls = reqs[arm], threading.Event(), []

                def coll_loop():
                    while not stop.is_set():
                        t0 = time.perf_counter()
                        assert q.run() == U.UCC_OK
                        calls.append(time.perf_counter() - t0)
                th = threading.Thread(target=coll_loop)
                th.start()
                while not calls:              # the collectives are running before the GEMM loop starts
                    if not th.is_alive():
                        sys.exit(f"overlap_bench: {arm} failed")
                    time.sleep(0.001)
                k0 = len(calls)
                ms = gemm_loop()
                k1 = len(calls)
                stop.set()
                th.join()
                per = sum(calls[k0:k1]) / max(k1 - k0, 1)
                results[arm].append({"gemm_ms": ms, "gemm_alone_ms": alone, "slowdown": ms / alone, "coll_ms": per * 1e3, "coll_calls": k1 - k0})
                line = {"rep": rep, "coll": arm[0], "bytes_per_rank": arm[1], "hint": arm[2], **results[arm][-1]}
                print(json.dumps(line), flush=True)
        for q in reqs.values():
            q.finalize()
    summary = []
    for (coll, size, hint), rs in results.items():
        med = lambda k: sorted(r[k] for r in rs)[len(rs) // 2]  # noqa: E731
        summary.append({"coll": coll, "MB_per_rank": size >> 20, "hint": hint, "gemm_ms": round(med("gemm_ms"), 2),
                        "gemm_alone_ms": round(med("gemm_alone_ms"), 2), "slowdown": round(med("slowdown"), 3), "coll_ms": round(med("coll_ms"), 3)})
    print("SUMMARY (medians of %d repetitions; %d emulated ranks on one GPU: the copies are local HBM traffic, not NVLink)" % (o.reps, n))
    for s in summary:
        print("  %-15s %4d MB  hint=%-5s  gemm %8.2f ms (alone %8.2f, x%.3f)  collective %8.3f ms/call"
              % (s["coll"], s["MB_per_rank"], s["hint"], s["gemm_ms"], s["gemm_alone_ms"], s["slowdown"], s["coll_ms"]))
    if o.json:
        with open(o.json, "w") as f:
            json.dump({"card": info, "ranks": n, "gemm": o.gemm, "iters": o.iters, "summary": summary, "runs": {str(k): v for k, v in results.items()}}, f, indent=1)


if __name__ == "__main__":
    main()
