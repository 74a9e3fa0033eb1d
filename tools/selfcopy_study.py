#!/usr/bin/env python3
"""Study of the team-of-one device copy (the whole 1 GiB allreduce of bench.py --gpus 1): every candidate kernel of
tools/selfcopy_study.cu, the library's thread-copy launcher and cudaMemcpyAsync, timed side by side in one process.

    python tools/selfcopy_study.py [--out DIR] [--rounds R] [--iters K] [--sizes 16M,64M,256M,1G] [--lib prebuilt.so]

Schedule: for every size, R interleaved rounds (A B C ... A B C ...).  In every round a candidate first copies into a
poisoned destination, which is compared bitwise with the source, then runs 2 untimed copies and K copies between two
CUDA events on one stream; the round's figure is the mean of those K.  Reported per candidate: median, min and max over
the rounds, and S/t of the median.  The card's name, power limit and SM clocks (read-only nvidia-smi query) are taken
before and after.  The JSON goes to DIR/selfcopy_study.json."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KB, MB, GB = 1 << 10, 1 << 20, 1 << 30


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="selfcopy_study_out", help="output directory (default: ./selfcopy_study_out)")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--sizes", default="16M,64M,256M,1G")
    ap.add_argument("--lib", default="", help="prebuilt tools/selfcopy_study.cu (default: build it into a temporary directory)")
    return ap.parse_args()


def size_of(s):
    return int(s[:-1]) * {"K": KB, "M": MB, "G": GB}[s[-1]] if s[-1] in "KMG" else int(s)


def gpu_info(dev):
    q = "name,power.limit,power.max_limit,clocks.sm,clocks.max.sm,clocks.mem,temperature.gpu"
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(dev), f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        return dict(zip(q.split(","), (x.strip() for x in r.stdout.strip().split(","))))
    except Exception as e:  # noqa: BLE001 - the record says why it is missing
        return {"unavailable": str(e)}


def build(prebuilt):
    if prebuilt:
        return prebuilt
    so = os.path.join(tempfile.mkdtemp(prefix="selfcopy_study_"), "libselfcopy_study.so")
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    subprocess.check_call([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fPIC",
                           os.path.join(ROOT, "tools", "selfcopy_study.cu"), "-o", so])
    return so


def candidates(exp, nvl, sm):
    """name -> launch(dst, src, nbytes, stream) returning a cudaError_t"""
    P, Z = C.c_void_p, C.c_size_t
    exp.study_tma.argtypes = [P, P, Z, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint, C.c_int, P]
    exp.study_thread.argtypes = [P, P, Z, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, P]
    exp.study_memcpy.argtypes = [P, P, Z, P]
    exp.study_max_blocks_per_sm.argtypes = [C.c_int] * 4
    nvl.nvl_launch_self_copy.argtypes = [P, P, Z, C.c_int, C.c_int, P]
    c = {}
    # what a team of one runs: the library's thread copy below 16 MB, cudaMemcpyAsync from 16 MB on
    c["lib self_copy 256x512"] = lambda d, s, n, st: nvl.nvl_launch_self_copy(d, s, n, 256, 512, st)
    c["cudaMemcpyAsync"] = lambda d, s, n, st: exp.study_memcpy(d, s, n, st)
    # TMA ring: stage KB, stages, loads ahead, CTAs per SM, contiguous span per CTA, L2 evict_first on loads (1) / stores (2)
    hints = {0: "", 1: " ef=ld", 2: " ef=st", 3: " ef=ld+st"}
    for kb, stages, ahead, per_sm, contig, hint in (
            (24, 8, 4, 1, 0, 0),                                             # the former library ring (8 x 24 KB, 4 ahead, 132 CTAs)
            (16, 12, 6, 1, 0, 0), (32, 6, 3, 1, 0, 0), (48, 4, 2, 1, 0, 0),   # stage size at ~192 KB of ring
            (24, 8, 6, 1, 0, 0), (24, 8, 2, 1, 0, 0), (16, 12, 9, 1, 0, 0), (32, 6, 4, 1, 0, 0), (48, 4, 3, 1, 0, 0),   # look-ahead
            (24, 4, 2, 2, 0, 0), (16, 6, 3, 2, 0, 0), (32, 3, 2, 2, 0, 0), (48, 2, 1, 2, 0, 0), (16, 4, 2, 3, 0, 0),      # CTAs per SM
            (24, 8, 4, 1, 1, 0), (32, 6, 3, 1, 1, 0), (24, 4, 2, 2, 1, 0),                                                # contiguous spans
            (24, 8, 4, 1, 0, 1), (24, 8, 4, 1, 0, 2), (24, 8, 4, 1, 0, 3), (32, 6, 3, 1, 0, 3), (24, 4, 2, 2, 0, 3),      # L2 policy
            (32, 6, 3, 1, 1, 3), (24, 4, 2, 2, 1, 3)):
        name = f"tma {kb}K x{stages} a{ahead} {per_sm}/SM {'span' if contig else 'rr'}{hints[hint]}"
        c[name] = (lambda kb, stages, ahead, per_sm, contig, hint: lambda d, s, n, st: exp.study_tma(
            d, s, n, stages, ahead, hint, contig, kb * KB, per_sm * sm, st))(kb, stages, ahead, per_sm, contig, hint)
    # TMA ring, non-persistent: one CTA per span of `per` chunks, the grid sized from the copy
    for kb, stages, ahead, per in ((24, 4, 2, 8), (16, 4, 2, 8), (16, 4, 2, 4), (16, 4, 3, 8), (16, 2, 1, 8), (8, 8, 4, 16), (16, 4, 2, 12), (32, 3, 2, 8)):
        name = f"tma {kb}K x{stages} a{ahead} span {per} chunks/CTA"
        c[name] = (lambda kb, stages, ahead, per: lambda d, s, n, st: exp.study_tma(
            d, s, n, stages, ahead, 0, 1, kb * KB, -(-n // (kb * KB * per)), st))(kb, stages, ahead, per)
    # thread copy, non-persistent: one block per run of nt x U vectors
    exp.study_thread_flat.argtypes = [P, P, Z, C.c_int, C.c_int, C.c_int, C.c_int, P]
    for u, ld, stm, nt in ((1, 0, 0, 1024), (1, 0, 0, 256), (2, 0, 0, 512), (4, 0, 0, 256), (4, 0, 0, 512), (8, 0, 0, 256), (8, 0, 0, 128),
                           (4, 1, 1, 256), (2, 1, 1, 1024), (4, 0, 1, 512), (1, 0, 0, 128), (1, 1, 1, 256), (2, 1, 1, 256), (2, 1, 1, 512), (1, 0, 0, 512), (2, 0, 1, 1024)):
        c[f"thread flat U{u} ld{ld} st{stm} x{nt}"] = (lambda u, ld, stm, nt: lambda d, s, n, st: exp.study_thread_flat(d, s, n, u, ld, stm, nt, st))(u, ld, stm, nt)
    # thread copy: warp tiles of 32 x U vectors; LD 1 = .L2::256B; ST 1 = st.global.cs, 2 = L2 evict_first policy
    for u, ld, stm, per_sm, nt in (
            (8, 0, 0, 2, 512), (8, 1, 0, 2, 512), (8, 1, 1, 2, 512), (8, 1, 2, 2, 512), (8, 0, 1, 2, 512),
            (8, 1, 1, 1, 1024), (8, 1, 1, 3, 512), (8, 1, 1, 4, 256), (8, 1, 1, 6, 256),
            (4, 1, 1, 2, 1024), (4, 1, 1, 4, 512), (4, 1, 1, 2, 512), (4, 0, 0, 4, 512), (4, 1, 2, 4, 512)):
        occ = exp.study_max_blocks_per_sm(u, ld, stm, nt)
        if occ < per_sm:
            print(f"skip thread U{u} ld{ld} st{stm} {per_sm}x{nt}/SM: only {occ} blocks per SM are resident", flush=True)
            continue
        name = f"thread U{u} ld{ld} st{stm} {per_sm * sm}x{nt}"
        c[name] = (lambda u, ld, stm, nb, nt: lambda d, s, n, st: exp.study_thread(d, s, n, u, ld, stm, nb, nt, st))(u, ld, stm, per_sm * sm, nt)
    return c


def main():
    a = parse()
    dev = torch.cuda.current_device()
    info_before = gpu_info(dev)
    sm = torch.cuda.get_device_properties(dev).multi_processor_count
    lib_dir = os.path.join(ROOT, "ucc_b200", "lib")
    C.CDLL(os.path.join(lib_dir, "libucc.so"), mode=C.RTLD_GLOBAL)
    nvl = C.CDLL(os.path.join(lib_dir, "ucc", "libucc_tl_nvl.so"))
    exp = C.CDLL(build(a.lib))
    cands = candidates(exp, nvl, sm)
    sizes = [size_of(s) for s in a.sizes.split(",")]
    st = torch.cuda.Stream()
    g = torch.Generator(device="cuda").manual_seed(7)
    src_all = torch.randint(0, 256, (max(sizes),), dtype=torch.uint8, device="cuda", generator=g)
    dst_all = torch.empty_like(src_all)
    torch.cuda.synchronize()
    res = {"gpu_before": info_before, "sm_count": sm, "rounds": a.rounds, "iters": a.iters, "sizes": {}}
    bad = []
    for n in sizes:
        src, dst = src_all[:n], dst_all[:n]
        times = {k: [] for k in cands}
        ok = {k: True for k in cands}
        with torch.cuda.stream(st):
            for _ in range(a.rounds):
                for name, fn in cands.items():
                    dst.fill_(0xA5)
                    e = fn(dst.data_ptr(), src.data_ptr(), n, st.cuda_stream)
                    if e:
                        raise RuntimeError(f"{name}: cudaError {e}")
                    ok[name] &= bool(torch.equal(dst, src))
                    for _ in range(2):
                        fn(dst.data_ptr(), src.data_ptr(), n, st.cuda_stream)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(st)
                    for _ in range(a.iters):
                        fn(dst.data_ptr(), src.data_ptr(), n, st.cuda_stream)
                    e1.record(st)
                    e1.synchronize()
                    times[name].append(e0.elapsed_time(e1) * 1e3 / a.iters)
        rows = {}
        for name, t in times.items():
            med = statistics.median(t)
            rows[name] = {"median_us": round(med, 2), "min_us": round(min(t), 2), "max_us": round(max(t), 2), "GBps": round(n / med / 1e3, 1),
                          "correct": ok[name], "rounds_us": [round(x, 2) for x in t]}
            if not ok[name]:
                bad.append((n, name))
        res["sizes"][str(n)] = rows
        print(f"\n== {n >> 20} MB", flush=True)
        for name, r in sorted(rows.items(), key=lambda kv: kv[1]["median_us"]):
            print(f"{r['median_us']:10.2f} us  [{r['min_us']:.2f} .. {r['max_us']:.2f}]  {r['GBps']:7.1f} GB/s  {'ok' if r['correct'] else 'WRONG'}  {name}", flush=True)
    res["gpu_after"] = gpu_info(dev)
    res["incorrect"] = [f"{n}: {name}" for n, name in bad]
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "selfcopy_study.json"), "w") as f:
        json.dump(res, f, indent=1)
    print("gpu before:", info_before, "\ngpu after:", res["gpu_after"], flush=True)
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
