"""Worker of tests/test_nvl_launch_paths.py: sweeps the tl/nvl algorithms of every collective on the host-emulated plugin
(tests/emu/build_hostemu.sh) and prints one line per case, `case -> launch note`, where the note (ucc_tl_nvl_last_launch_info) names
the kernel, grid and block of the launch that served the case.  Only tl/nvl is loaded (UCC_TLS=nvl; the teams carry their own ids, as
there is no service team to allocate one), so a case that tl/nvl declines fails at init and is left out.  Barrier,
fanin and fanout are among those: they carry no buffer, the core files them under host memory, and tl/nvl scores CUDA memory only.  Send / recv is left out too: which of its two ranks launches last is not fixed."""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from hostemu_worker import BASE, NOZC, ZC, Dev, U, UccJob, ca, coll_args, last_launch, rnd, rt  # noqa: E402  (loads the emulated runtime)

ENV = {k: v for k, v in BASE.items() if k != "UCC_COLL_TRACE"}
ENV.update(UCC_TLS="nvl", UCC_TL_NVL_MAX_BLOCKS="8")
# one TUNE per job: column i of every row (the algorithm tables of tl_nvl_coll.c, the names that run without a multicast mapping)
ALGS = {"allreduce": ("oneshot", "twoshot", "ring", "rhd"), "reduce_scatter": ("oneshot", "twoshot", "ring", "rhd"),
        "reduce_scatterv": ("oneshot", "twoshot", "ring", "rhd"), "reduce": ("twoshot",) * 4,
        "allgather": ("pull", "ring", "push", "ce"), "allgatherv": ("pull", "ring", "push", "ce"),
        "alltoall": ("pull", "push", "ce", "swap"), "alltoallv": ("pull", "push", "ce", "swap")}
BLKS = (1000, 20000)   # elements of float32 per member: 4 KB and 80 KB


def tune(i):
    return "#".join(f"{c}:cuda:inf:@{a[i]}" for c, a in ALGS.items())


def cases(n, blk):
    """yields (name, per-rank args) of every collective of a team of n, blk elements per member"""
    cnt = [blk + 3 * r for r in range(n)]
    dsp = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(int)
    even = [blk] * n
    edsp = [p * blk for p in range(n)]
    V = lambda c: [Dev(c, fill=rnd(c, r)) for r in range(n)]  # noqa: E731
    s, d = V(blk * n), V(blk * n)
    yield "allreduce", [ca("allreduce", s[r], d[r]) for r in range(n)]
    yield "allreduce inplace", [ca("allreduce", None, d[r], inplace=True) for r in range(n)]
    s, d = V(blk * n), V(blk)
    yield "reduce_scatter", [ca("reduce_scatter", s[r], d[r]) for r in range(n)]
    yield "reduce_scatter inplace", [ca("reduce_scatter", None, s[r], inplace=True) for r in range(n)]
    s, d = V(sum(cnt)), [Dev(cnt[r]) for r in range(n)]
    yield "reduce_scatterv", [ca("reduce_scatterv", s[r], d[r], dst_counts=cnt, dst_displs=dsp) for r in range(n)]
    s, o = V(blk), Dev(blk)
    yield "reduce", [ca("reduce", s[r], o if r == n - 1 else None, root=n - 1, count_dst=blk if r == n - 1 else 0) for r in range(n)]
    s, d = V(blk), V(blk * n)
    yield "allgather", [ca("allgather", s[r], d[r]) for r in range(n)]
    yield "allgather inplace", [ca("allgather", None, d[r], inplace=True) for r in range(n)]
    s, d = [Dev(cnt[r]) for r in range(n)], V(sum(cnt))
    yield "allgatherv", [ca("allgatherv", s[r], d[r], dst_counts=cnt, dst_displs=dsp) for r in range(n)]
    s, d = V(blk * n), V(blk * n)
    yield "alltoall", [ca("alltoall", s[r], d[r]) for r in range(n)]
    yield "alltoall inplace", [ca("alltoall", None, d[r], inplace=True) for r in range(n)]
    yield "alltoallv", [ca("alltoallv", s[r], d[r], src_counts=even, src_displs=edsp, dst_counts=even, dst_displs=edsp) for r in range(n)]
    yield "alltoallv inplace", [ca("alltoallv", None, d[r], inplace=True, dst_counts=even, dst_displs=edsp) for r in range(n)]
    b = V(blk)
    yield "bcast", [ca("bcast", b[r], None, root=1, count_dst=0) for r in range(n)]
    s, g = V(blk), Dev(blk * n)
    yield "gather", [ca("gather", s[r], g if r == 0 else None, root=0, count_dst=blk * n if r == 0 else 0) for r in range(n)]
    s, g = [Dev(cnt[r]) for r in range(n)], Dev(sum(cnt))
    yield "gatherv", [ca("gatherv", s[r], g, root=0, count_src=cnt[r], dst_counts=cnt, dst_displs=dsp) if r == 0
                      else ca("gatherv", s[r], None, root=0, count_src=cnt[r], count_dst=0) for r in range(n)]
    big, d = Dev(blk * n), V(blk)
    yield "scatter", [ca("scatter", big if r == n - 1 else None, d[r], root=n - 1, count_src=blk * n if r == n - 1 else 0) for r in range(n)]
    big, d = Dev(sum(cnt)), [Dev(cnt[r]) for r in range(n)]
    yield "scatterv", [ca("scatterv", big, d[r], root=1, src_counts=cnt, src_displs=dsp, count_dst=cnt[r]) if r == 1
                       else ca("scatterv", None, d[r], root=1, count_dst=cnt[r]) for r in range(n)]
    for c in ("barrier", "fanin", "fanout"):
        yield c, [coll_args(c, root=0) for _ in range(n)]


def sweep(label, team, blks=BLKS):
    n = len(team.members)
    for blk in blks:
        for name, args in cases(n, blk):
            try:
                q = team.coll(args)
            except U.UccError:
                continue                          # not served by tl/nvl
            st = q.run()
            q.finalize()
            assert st == U.UCC_OK, (label, n, blk, name, U.status_str(st))
            rt.cudaDeviceSynchronize()
            print(f"{label} n={n} blk={blk} {name} -> {last_launch()}", flush=True)


def registered(label):
    """twoshot allreduce on ucc_mem_map-registered buffers (the memh scenario of hostemu_worker.py), exchange board off"""
    U.lib.ucc_mem_map.argtypes = [U.handle, C.c_int, C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_void_p)]
    U.lib.ucc_mem_map.restype = C.c_int
    n, count = 4, 40000
    with UccJob(n, env=dict(ENV, UCC_TL_NVL_ZCOPY_THRESH="0", UCC_TL_NVL_TUNE="allreduce:cuda:inf:@twoshot")) as j:
        team = j.create_team(range(n), team_id=1)
        segs = {k: [Dev(2 * count, fill=0) for _ in range(n)] for k in ("src", "dst")}
        blobs, keep, glob = {"src": [], "dst": []}, [], {}
        for k in ("src", "dst"):
            for r in range(n):
                seg = U.ucc_mem_map_t(segs[k][r].ptr, 2 * count * 4)
                params = U.ucc_mem_map_params_t()
                params.segments, params.n_segments = C.pointer(seg), 1
                memh, size = C.c_void_p(), C.c_size_t()
                assert U.lib.ucc_mem_map(j.procs[r].ctx, 0, C.byref(params), C.byref(size), C.byref(memh)) == U.UCC_OK
                blobs[k].append(C.string_at(memh.value, size.value))
            for r in range(n):
                arr = (C.c_void_p * n)()
                for p in range(n):
                    b = C.create_string_buffer(blobs[k][p], len(blobs[k][p]))
                    keep.append(b)
                    h = C.c_void_p(C.addressof(b))
                    assert U.lib.ucc_mem_map(j.procs[r].ctx, 1, None, None, C.byref(h)) == U.UCC_OK
                    arr[p] = h.value
                glob[(k, r)] = arr
        args = []
        for r in range(n):
            a = coll_args("allreduce", dt="float32", mem_type=U.UCC_MEMORY_TYPE_CUDA, src_ptr=segs["src"][r].ptr + count * 4,
                          dst_ptr=segs["dst"][r].ptr + count * 4, count_src=count, count_dst=count)
            a.mask |= U.UCC_COLL_ARGS_FIELD_MEM_MAP_SRC_MEMH | U.UCC_COLL_ARGS_FIELD_MEM_MAP_DST_MEMH | U.UCC_COLL_ARGS_FIELD_FLAGS
            a.flags |= U.UCC_COLL_ARGS_FLAG_SRC_MEMH_GLOBAL | U.UCC_COLL_ARGS_FLAG_DST_MEMH_GLOBAL
            a.src_memh.global_memh = C.cast(glob[("src", r)], C.POINTER(C.c_void_p))
            a.dst_memh.global_memh = C.cast(glob[("dst", r)], C.POINTER(C.c_void_p))
            args.append(a)
        q = team.coll(args)
        assert q.run() == U.UCC_OK
        q.finalize()
        rt.cudaDeviceSynchronize()
        print(f"{label} n={n} count={count} allreduce -> {last_launch()}", flush=True)


def main():
    for mode, extra in (("staged", NOZC), ("zcopy", ZC)):
        for i in range(4):
            with UccJob(4, env=dict(ENV, UCC_TL_NVL_TUNE=tune(i), **extra)) as j:
                for n in (2, 3, 4):
                    sweep(f"{mode} tune={i}", j.create_team(range(n), team_id=n))
    bulk = "#".join(f"{c}:cuda:inf:@push" for c in ("allgather", "allgatherv", "alltoall", "alltoallv"))
    with UccJob(4, env=dict(ENV, UCC_TL_NVL_TUNE=bulk, UCC_TL_NVL_BULK="y", UCC_TL_NVL_BULK_THRESH="0", **ZC)) as j:
        for n in (2, 4):
            sweep("bulk push", j.create_team(range(n), team_id=n), blks=(1000,))
    registered("memh twoshot")
    # team of one: one copy, by the copy kernel below 16 MB and by cudaMemcpyAsync from there
    with UccJob(1, env=dict(ENV), with_ctx_oob=False) as j:
        team = j.create_team(team_id=1)
        for blk in (1000, 5 << 20):
            s, d = Dev(blk, fill=rnd(blk, 1)), Dev(blk)
            for name, args in (("allreduce", [ca("allreduce", s, d)]), ("alltoall", [ca("alltoall", s, d)]),
                               ("allreduce inplace", [ca("allreduce", None, d, inplace=True)]), ("bcast", [ca("bcast", d, None, count_dst=0)]),
                               ("barrier", [coll_args("barrier")])):
                try:
                    q = team.coll(args)
                except U.UccError:
                    continue
                assert q.run() == U.UCC_OK, ("self", blk, name)
                q.finalize()
                rt.cudaDeviceSynchronize()
                print(f"self n=1 blk={blk} {name} -> {last_launch()}", flush=True)


if __name__ == "__main__":
    main()
    print("LAUNCH_PATHS_OK", flush=True)
