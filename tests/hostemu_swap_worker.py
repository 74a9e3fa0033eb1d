"""Worker of tests/test_nvl_swap.py: in-place alltoall / alltoallv through the public UCC API on the tl/nvl plugin built against the
emulated CUDA runtime with the swap kernel (tests/emu/build_hostemu_swap.sh), N ranks in this process.  Every result is compared with
numpy for equality; the launch note names the kernel that served it."""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from hostemu_worker import BASE, NOZC, ZC, Dev, U, UccJob, ca, coll_args, rnd, rt, run  # noqa: E402  (loads the emulated runtime)

# the emulated plugin with the swap kernel (tests/emu/build_hostemu_swap.sh), next to the runtime loaded above; scenario "no_swap_kernel"
# keeps the plugin of tests/emu/build_hostemu.sh, whose launcher set lacks it
if sys.argv[1:] != ["no_swap_kernel"]:
    os.environ["UCC_MODULE_DIR"] = os.path.join(os.path.dirname(os.environ["UCC_MODULE_DIR"]), "ucc_swap")

TRACE = {"UCC_COLL_TRACE": "debug"}   # a coll_init line for every rank, naming the TL that serves the collective
SWAP, STAGED = "exchange_swap", "exchange_pull_staged_inplace"


def last_launch():
    info = C.CDLL(os.path.join(os.environ["UCC_MODULE_DIR"], "libucc_tl_nvl.so")).ucc_tl_nvl_last_launch_info
    info.restype = C.c_char_p
    return info().decode()


def a2a_expect(bufs, n, blk):
    return [np.concatenate([bufs[p][r * blk:(r + 1) * blk] for p in range(n)]) for r in range(n)]


def a2av_layout(n, blk):
    """symmetric skewed counts (rank 0 is hot, one zero-length pair) and displacements with gaps; returns counts[r][p], displs[r][p],
    buffer length"""
    cnt = np.zeros((n, n), dtype=np.int64)
    for r in range(n):
        for p in range(n):
            lo, hi = min(r, p), max(r, p)
            cnt[r, p] = (blk + hi if lo == 0 else blk // 3 + lo * hi) if not (r != p and lo + hi == 3) else 0
    dsp = np.zeros((n, n), dtype=np.int64)
    size = 0
    for r in range(n):
        o = 0
        for p in range(n):
            o += (r + p) % 3          # gaps: unaligned regions
            dsp[r, p] = o
            o += cnt[r, p]
        size = max(size, o + 2)
    return cnt, dsp, size


def a2av_expect(before, cnt, dsp, n):
    out = [b.copy() for b in before]
    for r in range(n):
        for p in range(n):
            if p != r:
                out[r][dsp[r, p]:dsp[r, p] + cnt[r, p]] = before[p][dsp[p, r]:dsp[p, r] + cnt[p, r]]
    return out


def inplace_colls(extra, want):
    """in-place alltoall / alltoallv on teams of 2, 3 and 4, several block sizes, served by `want`"""
    with UccJob(4, env=dict(BASE, **TRACE, **extra)) as j:
        for n in (2, 3, 4):
            team = j.create_team(range(n))
            for blk in (1, 5, 1000, 30011):
                bufs = [Dev(blk * n, fill=rnd(blk * n, 10 * n + r)) for r in range(n)]
                exp = a2a_expect([b.a.copy() for b in bufs], n, blk)
                run(team, [ca("alltoall", None, bufs[r], inplace=True) for r in range(n)])
                assert want in last_launch(), (last_launch(), n, blk)
                for r in range(n):
                    assert np.array_equal(bufs[r].a, exp[r]), ("alltoall inplace", want, n, blk, r)
                cnt, dsp, size = a2av_layout(n, blk)
                bufs = [Dev(size, fill=rnd(size, 20 * n + r)) for r in range(n)]
                exp = a2av_expect([b.a.copy() for b in bufs], cnt, dsp, n)
                run(team, [ca("alltoallv", None, bufs[r], inplace=True, dst_counts=cnt[r], dst_displs=dsp[r]) for r in range(n)])
                assert want in last_launch(), (last_launch(), n, blk)
                for r in range(n):
                    assert np.array_equal(bufs[r].a, exp[r]), ("alltoallv inplace", want, n, blk, r)
    print(f"  in-place alltoall(v) {want} ok", flush=True)


def persistent():
    """a persistent in-place alltoall and alltoallv, each posted three times with new contents: the buffer tables of the first post
    are reused"""
    n, blk = 4, 7001
    with UccJob(n, env=dict(BASE, **TRACE, **ZC)) as j:
        team = j.create_team(range(n))
        bufs = [Dev(blk * n, fill=0) for _ in range(n)]
        q = team.coll([ca("alltoall", None, bufs[r], inplace=True, persistent=True) for r in range(n)])
        for it in range(3):
            for r in range(n):
                bufs[r].a[:] = rnd(blk * n, 100 * it + r)
            exp = a2a_expect([b.a.copy() for b in bufs], n, blk)
            assert q.run() == U.UCC_OK
            rt.cudaDeviceSynchronize()
            assert SWAP in last_launch(), last_launch()
            for r in range(n):
                assert np.array_equal(bufs[r].a, exp[r]), ("persistent alltoall", it, r)
        q.finalize()
        cnt, dsp, size = a2av_layout(n, 999)
        bufs = [Dev(size, fill=0) for _ in range(n)]
        q = team.coll([ca("alltoallv", None, bufs[r], inplace=True, persistent=True, dst_counts=cnt[r], dst_displs=dsp[r]) for r in range(n)])
        for it in range(3):
            for r in range(n):
                bufs[r].a[:] = rnd(size, 200 * it + r)
            exp = a2av_expect([b.a.copy() for b in bufs], cnt, dsp, n)
            assert q.run() == U.UCC_OK
            rt.cudaDeviceSynchronize()
            assert SWAP in last_launch(), last_launch()
            for r in range(n):
                assert np.array_equal(bufs[r].a, exp[r]), ("persistent alltoallv", it, r)
        q.finalize()
    print("  persistent in-place alltoall(v) ok", flush=True)


def registered():
    """in-place alltoall on ucc_mem_map-registered buffers: the swap kernel gets the members' buffers from the registrations"""
    U.lib.ucc_mem_map.argtypes = [U.handle, C.c_int, C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_void_p)]
    U.lib.ucc_mem_map.restype = C.c_int
    n, blk = 4, 5000
    with UccJob(n, env=dict(BASE, **TRACE)) as j:
        team = j.create_team(range(n))
        segs = [Dev(2 * blk * n, fill=0) for _ in range(n)]   # the collective uses the second half of each registered segment
        blobs, keep = [], []
        for r in range(n):
            seg = U.ucc_mem_map_t(segs[r].ptr, 2 * blk * n * 4)
            params = U.ucc_mem_map_params_t()
            params.segments, params.n_segments = C.pointer(seg), 1
            memh, size = C.c_void_p(), C.c_size_t()
            assert U.lib.ucc_mem_map(j.procs[r].ctx, 0, C.byref(params), C.byref(size), C.byref(memh)) == U.UCC_OK
            blobs.append(C.string_at(memh.value, size.value))
            keep.append(memh)
        glob = []
        for r in range(n):
            arr = (C.c_void_p * n)()
            for p in range(n):
                b = C.create_string_buffer(blobs[p], len(blobs[p]))
                keep.append(b)
                h = C.c_void_p(C.addressof(b))
                assert U.lib.ucc_mem_map(j.procs[r].ctx, 1, None, None, C.byref(h)) == U.UCC_OK
                arr[p] = h.value
            glob.append(arr)
        for it in range(2):
            for r in range(n):
                segs[r].a[blk * n:] = rnd(blk * n, 50 * it + r)
            exp = a2a_expect([s.a[blk * n:].copy() for s in segs], n, blk)
            args = []
            for r in range(n):
                a = coll_args("alltoall", dt="float32", mem_type=U.UCC_MEMORY_TYPE_CUDA, dst_ptr=segs[r].ptr + blk * n * 4, count_dst=blk * n, inplace=True)
                a.mask |= U.UCC_COLL_ARGS_FIELD_MEM_MAP_DST_MEMH | U.UCC_COLL_ARGS_FIELD_FLAGS
                a.flags |= U.UCC_COLL_ARGS_FLAG_DST_MEMH_GLOBAL
                a.dst_memh.global_memh = C.cast(glob[r], C.POINTER(C.c_void_p))
                args.append(a)
            run(team, args)
            assert SWAP in last_launch(), last_launch()
            for r in range(n):
                assert np.array_equal(segs[r].a[blk * n:], exp[r]), ("registered alltoall", it, r)
                assert np.all(segs[r].a[:blk * n] == 0)
    print("  registered in-place alltoall ok", flush=True)


def big_team():
    """a team of six with 4.8 and 9.6 MB buffers, inside the alltoall:4M-64M:@push default range of teams of more than four: push
    turns in-place requests down and the score fallback lands on the swap path; out-of-place alltoall keeps the push kernel"""
    n = 6
    with UccJob(n, env=dict(BASE, **TRACE, UCC_TL_NVL_ZCOPY="y", UCC_TL_NVL_SYMMETRIC_SIZE="32Mb")) as j:
        team = j.create_team(range(n))
        for blk in (200000, 400000):
            bufs = [Dev(blk * n, fill=rnd(blk * n, 10 + r)) for r in range(n)]
            exp = a2a_expect([b.a.copy() for b in bufs], n, blk)
            run(team, [ca("alltoall", None, bufs[r], inplace=True) for r in range(n)])
            assert SWAP in last_launch(), (blk, last_launch())
            for r in range(n):
                assert np.array_equal(bufs[r].a, exp[r]), ("big team alltoall inplace", blk, r)
            src = [Dev(blk * n, fill=rnd(blk * n, 30 + r)) for r in range(n)]
            dst = [Dev(blk * n, fill=0) for _ in range(n)]
            run(team, [ca("alltoall", src[r], dst[r]) for r in range(n)])
            assert "exchange_push" in last_launch(), (blk, last_launch())
            assert np.array_equal(dst[3].a, np.concatenate([s.a[3 * blk:4 * blk] for s in src]))
    print("  team of six, 4.8 / 9.6 MB: in-place swap, out-of-place push ok", flush=True)


def tune_swap():
    """UCC_TL_NVL_TUNE=alltoall:@swap selects the swap path for in-place requests; an out-of-place alltoall, which swap turns down,
    still runs on tl/nvl (the pull kernel, through the score fallback)"""
    n, blk = 4, 3001
    with UccJob(n, env=dict(BASE, **TRACE, **ZC, UCC_TL_NVL_TUNE="alltoall:@swap#alltoallv:@swap")) as j:
        team = j.create_team(range(n))
        bufs = [Dev(blk * n, fill=rnd(blk * n, r)) for r in range(n)]
        exp = a2a_expect([b.a.copy() for b in bufs], n, blk)
        run(team, [ca("alltoall", None, bufs[r], inplace=True) for r in range(n)])
        assert SWAP in last_launch(), last_launch()
        for r in range(n):
            assert np.array_equal(bufs[r].a, exp[r]), ("tune swap", r)
        src = [Dev(blk * n, fill=rnd(blk * n, 40 + r)) for r in range(n)]
        dst = [Dev(blk * n, fill=0) for _ in range(n)]
        run(team, [ca("alltoall", src[r], dst[r]) for r in range(n)])
        assert "exchange_pull" in last_launch(), last_launch()
        for r in range(n):
            assert np.array_equal(dst[r].a, np.concatenate([s.a[r * blk:(r + 1) * blk] for s in src])), ("tune swap, out of place", r)
    print("  TUNE alltoall:@swap ok", flush=True)


def no_swap_kernel():
    """a plugin linked without the swap launcher loads and declines in-place alltoall(v) at init: the request goes to the next TL
    (test_nvl_swap.py checks the trace; it is only initialised here), out-of-place alltoall stays on tl/nvl"""
    n, blk = 3, 1001
    with UccJob(n, env=dict(BASE, **TRACE, **ZC)) as j:
        team = j.create_team(range(n))
        bufs = [Dev(blk * n, fill=rnd(blk * n, r)) for r in range(n)]
        for r in range(n):
            a = ca("alltoall", None, bufs[r], inplace=True)
            q = C.POINTER(U.ucc_coll_req_t)()
            assert U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team) == U.UCC_OK
            U.ucc_collective_finalize(q)
        src = [Dev(blk * n, fill=rnd(blk * n, 10 + r)) for r in range(n)]
        dst = [Dev(blk * n, fill=0) for _ in range(n)]
        run(team, [ca("alltoall", src[r], dst[r]) for r in range(n)])
        assert np.array_equal(dst[1].a, np.concatenate([s.a[blk:2 * blk] for s in src]))
    print("  plugin without the swap kernel: in-place alltoall declined ok", flush=True)


SCENARIOS = {
    "zcopy": lambda: inplace_colls(ZC, SWAP),
    "staged": lambda: inplace_colls(NOZC, STAGED),
    "persistent": persistent,
    "memh": registered,
    "big_team": big_team,
    "tune": tune_swap,
    "no_swap_kernel": no_swap_kernel,
}

if __name__ == "__main__":
    SCENARIOS[sys.argv[1]]()
    print("HOSTEMU_WORKER_OK", flush=True)
