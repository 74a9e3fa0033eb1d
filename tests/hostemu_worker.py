"""Worker of tests/test_nvl_hostemu.py: the tl/nvl plugin built against the emulated CUDA runtime (tests/emu/build_hostemu.sh),
N ranks in this process, "device" buffers from the emulated cudaMalloc.  Exercises the HOST side of tl/nvl - team creation with a
shared-pointer heap, score selection / TUNE, launch ordering, the zero-copy exchange board, deferred launches, persistent requests,
asymmetric memory staging in the core - together with the emulated kernels, and checks every result against numpy."""
import ctypes as C
import faulthandler
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ["UCC_MODULE_DIR"] = os.path.join(ROOT, "build-emu", "lib", "ucc")
faulthandler.dump_traceback_later(240, exit=True)
rt = C.CDLL(os.path.join(ROOT, "build-emu", "lib", "libcudart_emu.so"), mode=C.RTLD_GLOBAL)
sys.path.insert(0, ROOT)
from ucc_b200 import capi as U  # noqa: E402
from ucc_b200.harness import UccJob, coll_args  # noqa: E402

CUDA, HOST = U.UCC_MEMORY_TYPE_CUDA, U.UCC_MEMORY_TYPE_HOST
BASE = {"UCC_TL_NVL_MAX_BLOCKS": "2", "UCC_TL_NVL_NTHREADS": "64", "UCC_TL_NVL_TIMEOUT": "30s", "UCC_TL_NVL_SYMMETRIC_SIZE": "1Mb", "UCC_TLS": "nvl,shm,self",
        "UCC_COLL_TRACE": "info"}
ZC = {"UCC_TL_NVL_ZCOPY": "y", "UCC_TL_NVL_ZCOPY_THRESH": "0"}
NOZC = {"UCC_TL_NVL_ZCOPY": "n"}


class Dev:
    """numpy view of a buffer allocated with the emulated cudaMalloc"""

    created = 0     # (buffers are never freed: leak checks subtract this)

    def __init__(self, n, dtype=np.float32, fill=None):
        Dev.created += 1
        p = C.c_void_p()
        nbytes = max(n, 1) * np.dtype(dtype).itemsize
        assert rt.cudaMalloc(C.byref(p), C.c_size_t(nbytes)) == 0
        self.ptr = p.value
        self.a = np.frombuffer((C.c_char * nbytes).from_address(p.value), dtype=dtype)[:n]
        if fill is not None:
            self.a[:] = fill


def ca(coll, src, dst, dt="float32", **kw):
    kw.setdefault("count_src", src.a.size if src is not None else 0)
    kw.setdefault("count_dst", dst.a.size if dst is not None else 0)
    return coll_args(coll, dt=dt, mem_type=CUDA, src_ptr=src.ptr if src is not None else None, dst_ptr=dst.ptr if dst is not None else None, **kw)


def run(team, args):
    q = team.coll(args)
    st = q.run()
    q.finalize()
    assert st == U.UCC_OK, U.status_str(st)
    rt.cudaDeviceSynchronize()


def last_launch():
    """the launch note of the plugin's most recent kernel launch: names the kernel that served it"""
    info = C.CDLL(os.path.join(os.environ["UCC_MODULE_DIR"], "libucc_tl_nvl.so")).ucc_tl_nvl_last_launch_info
    info.restype = C.c_char_p
    return info().decode()


def rnd(n, seed, dtype=np.float32):
    g = np.random.default_rng(seed)
    return g.integers(0, 9, n).astype(dtype)


def allreduce_suite(alg, extra, sizes=(1, 7, 1000, 4097, 70000)):
    env = dict(BASE, UCC_TL_NVL_TUNE=f"allreduce:cuda:inf:@{alg}", UCC_TL_NVL_ALLREDUCE_ONESHOT_THRESH="0" if alg != "oneshot" else "1M", **extra)
    with UccJob(4, env=env) as j:
        teams = {n: j.create_team(range(n)) for n in (2, 3, 4)}
        for n, team in teams.items():
            if alg == "rhd" and n == 3:
                continue
            for count in sizes:
                for inplace in (False, True):
                    src = [Dev(count, fill=rnd(count, 10 * n + r)) for r in range(n)]
                    exp = sum(s.a.copy() for s in src)
                    dst = src if inplace else [Dev(count, fill=0) for _ in range(n)]
                    run(team, [ca("allreduce", None if inplace else src[r], dst[r], inplace=inplace) for r in range(n)])
                    for r in range(n):
                        assert np.allclose(dst[r].a, exp), (alg, extra, n, count, inplace, r)
        # other datatypes / operators through the same path
        team, n = teams[4], 4
        for dt, op in (("float64", "avg"), ("int32", "max"), ("int64", "sum"), ("uint8", "min"), ("float32", "prod")):
            npdt = np.dtype(dt)
            src = [Dev(515, npdt, fill=rnd(515, r + 3, npdt) % 3 + 1) for r in range(n)]
            dst = [Dev(515, npdt, fill=0) for _ in range(n)]
            run(team, [ca("allreduce", src[r], dst[r], dt=dt, op=op) for r in range(n)])
            st = np.stack([s.a.astype(np.float64) for s in src])
            exp = {"avg": st.mean(0), "max": st.max(0), "sum": st.sum(0), "min": st.min(0), "prod": st.prod(0)}[op]
            for r in range(n):
                assert np.allclose(dst[r].a.astype(np.float64), exp), (alg, dt, op, r)
    print(f"  allreduce {alg} {'zcopy' if extra is ZC else 'staged'} ok", flush=True)


def other_colls(extra, tune=""):
    env = dict(BASE, **extra)
    if tune:
        env["UCC_TL_NVL_TUNE"] = tune
    with UccJob(4, env=env) as j:
        for n in (3, 4):
            team = j.create_team(range(n))
            for blk in (5, 1000, 30011):
                # reduce_scatter (+ in place), reduce_scatterv
                src = [Dev(blk * n, fill=rnd(blk * n, r)) for r in range(n)]
                exp = sum(s.a.copy() for s in src)
                dst = [Dev(blk, fill=0) for _ in range(n)]
                run(team, [ca("reduce_scatter", src[r], dst[r]) for r in range(n)])
                for r in range(n):
                    assert np.allclose(dst[r].a, exp[r * blk:(r + 1) * blk]), ("rs", n, blk, r)
                run(team, [ca("reduce_scatter", None, src[r], inplace=True) for r in range(n)])
                for r in range(n):
                    assert np.allclose(src[r].a[r * blk:(r + 1) * blk], exp[r * blk:(r + 1) * blk]), ("rs inplace", n, blk, r)
                counts = [blk + 3 * r for r in range(n)]
                offs = np.concatenate([[0], np.cumsum(counts)[:-1]])
                src = [Dev(sum(counts), fill=rnd(sum(counts), r + 50)) for r in range(n)]
                exp = sum(s.a.copy() for s in src)
                dst = [Dev(counts[r], fill=0) for r in range(n)]
                run(team, [ca("reduce_scatterv", src[r], dst[r], dst_counts=counts, dst_displs=offs) for r in range(n)])
                for r in range(n):
                    assert np.allclose(dst[r].a, exp[offs[r]:offs[r] + counts[r]]), ("rsv", n, blk, r)
                # reduce to a non-zero root
                src = [Dev(blk, fill=rnd(blk, r + 7)) for r in range(n)]
                exp = sum(s.a.copy() for s in src)
                out = Dev(blk, fill=0)
                run(team, [ca("reduce", src[r], out if r == n - 1 else None, root=n - 1, count_dst=blk if r == n - 1 else 0) for r in range(n)])
                assert np.allclose(out.a, exp), ("reduce", n, blk)
                # allgather (+ in place), allgatherv
                src = [Dev(blk, fill=rnd(blk, r + 20)) for r in range(n)]
                exp = np.concatenate([s.a for s in src])
                dst = [Dev(blk * n, fill=0) for _ in range(n)]
                run(team, [ca("allgather", src[r], dst[r]) for r in range(n)])
                for r in range(n):
                    assert np.array_equal(dst[r].a, exp), ("allgather", n, blk, r)
                for r in range(n):
                    dst[r].a[:] = 0
                    dst[r].a[r * blk:(r + 1) * blk] = src[r].a
                run(team, [ca("allgather", None, dst[r], inplace=True) for r in range(n)])
                for r in range(n):
                    assert np.array_equal(dst[r].a, exp), ("allgather inplace", n, blk, r)
                srcv = [Dev(counts[r], fill=rnd(counts[r], r + 30)) for r in range(n)]
                expv = np.concatenate([s.a for s in srcv])
                dstv = [Dev(sum(counts), fill=0) for _ in range(n)]
                run(team, [ca("allgatherv", srcv[r], dstv[r], dst_counts=counts, dst_displs=offs) for r in range(n)])
                for r in range(n):
                    assert np.array_equal(dstv[r].a, expv), ("allgatherv", n, blk, r)
                # alltoall, skewed alltoallv (rank 0 is the hot receiver)
                src = [Dev(blk * n, fill=rnd(blk * n, r + 40)) for r in range(n)]
                dst = [Dev(blk * n, fill=0) for _ in range(n)]
                run(team, [ca("alltoall", src[r], dst[r]) for r in range(n)])
                for r in range(n):
                    assert np.array_equal(dst[r].a, np.concatenate([src[p].a[r * blk:(r + 1) * blk] for p in range(n)])), ("alltoall", n, blk, r)
                m = np.array([[blk * 2 if d == 0 else (0 if s == d else 3 + (s + d) % 4) for d in range(n)] for s in range(n)])
                src = [Dev(int(m[r].sum()), fill=rnd(int(m[r].sum()), r + 60)) for r in range(n)]
                dst = [Dev(int(m[:, r].sum()), fill=0) for r in range(n)]
                sd = [np.concatenate([[0], np.cumsum(m[r])[:-1]]) for r in range(n)]
                rd = [np.concatenate([[0], np.cumsum(m[:, r])[:-1]]) for r in range(n)]
                run(team, [ca("alltoallv", src[r], dst[r], src_counts=m[r], src_displs=sd[r], dst_counts=m[:, r], dst_displs=rd[r]) for r in range(n)])
                for r in range(n):
                    exp = np.concatenate([src[p].a[sd[p][r]:sd[p][r] + m[p][r]] for p in range(n)])
                    assert np.array_equal(dst[r].a, exp), ("alltoallv", n, blk, r)
                # bcast, gather, scatter
                b = [Dev(blk, fill=rnd(blk, 99) if r == 1 else 0) for r in range(n)]
                run(team, [ca("bcast", b[r], None, root=1, count_dst=0) for r in range(n)])
                for r in range(n):
                    assert np.array_equal(b[r].a, rnd(blk, 99)), ("bcast", n, blk, r)
                src = [Dev(blk, fill=rnd(blk, r + 70)) for r in range(n)]
                g = Dev(blk * n, fill=0)
                run(team, [ca("gather", src[r], g if r == 0 else None, root=0, count_dst=blk * n if r == 0 else 0) for r in range(n)])
                assert np.array_equal(g.a, np.concatenate([s.a for s in src])), ("gather", n, blk)
                big = Dev(blk * n, fill=rnd(blk * n, 5))
                outs = [Dev(blk, fill=0) for _ in range(n)]
                run(team, [ca("scatter", big if r == 2 else None, outs[r], root=2, count_src=blk * n if r == 2 else 0) for r in range(n)])
                for r in range(n):
                    assert np.array_equal(outs[r].a, big.a[r * blk:(r + 1) * blk]), ("scatter", n, blk, r)
            run(team, [coll_args("barrier") for _ in range(n)])
    print(f"  collectives {'zcopy' if extra is ZC else 'staged'} {tune or 'default algorithms'} ok", flush=True)


def persistent_and_teams():
    with UccJob(4, env=dict(BASE, **ZC)) as j:
        ta, tb = j.create_team(range(4)), j.create_team([3, 1, 0])
        n, count = 4, 20000
        src = [Dev(count, fill=0) for _ in range(n)]
        dst = [Dev(count, fill=0) for _ in range(n)]
        q = ta.coll([ca("allreduce", src[r], dst[r], persistent=True) for r in range(n)])
        for it in range(4):
            for r in range(n):
                src[r].a[:] = rnd(count, it * 10 + r)
            assert q.run() == U.UCC_OK
            rt.cudaDeviceSynchronize()
            exp = sum(s.a.copy() for s in src)
            for r in range(n):
                assert np.allclose(dst[r].a, exp), ("persistent", it, r)
            # a collective on the second team between the posts (ranks 3,1,0 of the job)
            x = [Dev(333, fill=float(i + 1)) for i in range(3)]
            run(tb, [ca("allreduce", None, x[i], inplace=True) for i in range(3)])
            assert all(np.all(v.a == 6.0) for v in x)
        q.finalize()
        # messages larger than the heap data region: several rounds inside one kernel
        big = 900000
        src = [Dev(big, fill=rnd(big, r)) for r in range(n)]
        dst = [Dev(big, fill=0) for _ in range(n)]
    with UccJob(4, env=dict(BASE, **NOZC)) as j:
        t = j.create_team(range(4))
        run(t, [ca("allreduce", src[r], dst[r]) for r in range(n)])
        exp = sum(s.a.copy() for s in src)
        for r in range(n):
            assert np.allclose(dst[r].a, exp), ("multi-round", r)
    print("  persistent / two teams / multi-round ok", flush=True)


def asymmetric_memory():
    """root's src and dst in different memory types (reference test/gtest/asym_mem): staged by the core around tl/nvl"""
    with UccJob(4, env=dict(BASE)) as j:
        t, n, count = j.create_team(range(4)), 4, 3000
        src = [Dev(count, fill=rnd(count, r)) for r in range(n)]
        host_dst = np.zeros(count, np.float32)
        args = [ca("reduce", src[r], None, root=1, count_dst=0) for r in range(n)]
        args[1] = coll_args("reduce", dt="float32", root=1, src_ptr=src[1].ptr, dst_ptr=host_dst.ctypes.data, count_src=count, count_dst=count, src_mem_type=CUDA, dst_mem_type=HOST)
        run(t, args)
        assert np.allclose(host_dst, sum(s.a for s in src))
        host_src = np.arange(n * 100, dtype=np.float32)
        dst = [Dev(100, fill=0) for _ in range(n)]
        args = [coll_args("scatter", dt="float32", root=0, dst_ptr=dst[r].ptr, count_dst=100, count_src=0, mem_type=CUDA) for r in range(n)]
        args[0] = coll_args("scatter", dt="float32", root=0, src_ptr=host_src.ctypes.data, dst_ptr=dst[0].ptr, count_src=n * 100, count_dst=100, src_mem_type=HOST, dst_mem_type=CUDA)
        run(t, args)
        for r in range(n):
            assert np.array_equal(dst[r].a, host_src[r * 100:(r + 1) * 100])
    print("  asymmetric memory ok", flush=True)


def triggered(extra):
    """stream-ordered posts (ucc_collective_triggered_post, what ProcessGroupUCC uses): the collective must be ordered behind work
    already queued on the user's stream, UCC_EVENT_COLLECTIVE_POST must arrive (after the real launch when it is deferred by the
    zero-copy exchange) and work queued afterwards must see the result"""
    rt.cudaStreamCreate.argtypes = [C.POINTER(C.c_void_p)]
    rt.cudaMemcpyAsync.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]
    rt.cudaStreamSynchronize.argtypes = [C.c_void_p]
    n, count = 4, 50000
    with UccJob(n, env=dict(BASE, **extra)) as j:
        team = j.create_team(range(n))
        streams, ees = [], []
        for r in range(n):
            s = C.c_void_p()
            assert rt.cudaStreamCreate(C.byref(s)) == 0
            ep = U.ucc_ee_params_t()
            ep.ee_type, ep.ee_context, ep.ee_context_size = U.UCC_EE_CUDA_STREAM, s.value, C.sizeof(C.c_void_p)
            ee = U.handle()
            U.check(U.ucc_ee_create(team.members[r].team, C.byref(ep), C.byref(ee)), "ee_create")
            streams.append(s)
            ees.append(ee)
        for it in range(3):
            stage = [Dev(count, fill=rnd(count, 7 * it + r)) for r in range(n)]   # what the stream copies into src BEFORE the collective
            src = [Dev(count, fill=-1) for _ in range(n)]
            dst = [Dev(count, fill=0) for _ in range(n)]
            after = [Dev(count, fill=0) for _ in range(n)]                        # copied from dst by the stream AFTER the collective
            reqs = []
            for r in range(n):
                rt.cudaMemcpyAsync(src[r].ptr, stage[r].ptr, count * 4, 3, streams[r])
                a = ca("allreduce", src[r], dst[r])
                q = C.POINTER(U.ucc_coll_req_t)()
                U.check(U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team), "init")
                ev = U.ucc_ev_t()
                ev.ev_type, ev.req = U.UCC_EVENT_COMPUTE_COMPLETE, C.cast(q, C.c_void_p)
                U.check(U.ucc_collective_triggered_post(ees[r], C.byref(ev)), "triggered_post")
                reqs.append((a, q))
            posted = [False] * n
            import time
            t0 = time.time()
            while not all(posted) or any(q.contents.status == U.UCC_INPROGRESS for _, q in reqs):
                for r in range(n):
                    U.ucc_context_progress(j.procs[r].ctx)
                    e = C.POINTER(U.ucc_ev_t)()
                    while U.ucc_ee_get_event(ees[r], C.byref(e)) == U.UCC_OK:
                        if e.contents.ev_type == U.UCC_EVENT_COLLECTIVE_POST:
                            assert not posted[r]
                            posted[r] = True
                            rt.cudaMemcpyAsync(after[r].ptr, dst[r].ptr, count * 4, 3, streams[r])   # ordered behind the collective
                        U.ucc_ee_ack_event(ees[r], e)
                assert time.time() - t0 < 120, (posted, [q.contents.status for _, q in reqs])
            for r in range(n):
                assert reqs[r][1].contents.status == U.UCC_OK
                rt.cudaStreamSynchronize(streams[r])
                U.ucc_collective_finalize(reqs[r][1])
            exp = sum(s.a.copy() for s in stage)
            for r in range(n):
                assert np.allclose(dst[r].a, exp) and np.allclose(after[r].a, exp), ("triggered", it, r)
        for ee in ees:
            U.ucc_ee_destroy(ee)
    print(f"  triggered posts {'zcopy (deferred launches)' if extra is ZC else 'staged'} ok", flush=True)


def cross_team_order(extra):
    """two teams over the same ranks, collectives posted in opposite team order on odd and even ranks (legal: only the order
    WITHIN a team must agree), several in flight per team; with zero-copy every launch is deferred until the peers published"""
    import time
    n, count, depth = 4, 30000, 3
    with UccJob(n, env=dict(BASE, **extra)) as j:
        ta, tb = j.create_team(range(n)), j.create_team(range(n))
        bufs = {}
        reqs = {r: [] for r in range(n)}
        for r in range(n):
            order = [(ta, "a"), (tb, "b")] if r % 2 == 0 else [(tb, "b"), (ta, "a")]
            for k in range(depth):
                for team, name in order:
                    src = Dev(count, fill=rnd(count, hash((name, k, r)) % 1000))
                    dst = Dev(count, fill=0)
                    bufs[(name, k, r)] = (src, dst)
                    a = ca("allreduce", src, dst)
                    q = C.POINTER(U.ucc_coll_req_t)()
                    U.check(U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team), "init")
                    U.check(U.ucc_collective_post(q), "post")
                    reqs[r].append((a, q))
        t0 = time.time()
        while any(q.contents.status == U.UCC_INPROGRESS for r in range(n) for _, q in reqs[r]):
            for r in range(n):
                U.ucc_context_progress(j.procs[r].ctx)
            assert time.time() - t0 < 120, "cross-team posts did not complete"
        rt.cudaDeviceSynchronize()
        for r in range(n):
            for _, q in reqs[r]:
                assert q.contents.status == U.UCC_OK
                U.ucc_collective_finalize(q)
        for name in "ab":
            for k in range(depth):
                exp = sum(bufs[(name, k, r)][0].a for r in range(n))
                for r in range(n):
                    assert np.allclose(bufs[(name, k, r)][1].a, exp), ("cross team", name, k, r)
    print(f"  cross-team post order {'zcopy' if extra is ZC else 'staged'} ok", flush=True)


def device_timeout():
    """a member that never posts: the kernels of the others give up after UCC_TL_NVL_TIMEOUT (bounded device-side spin) and their
    requests complete with an error instead of hanging the device"""
    import time
    n, count = 3, 1000
    with UccJob(n, env=dict(BASE, UCC_TL_NVL_TIMEOUT="2s", **NOZC)) as j:
        team = j.create_team(range(n))
        reqs = []
        for r in (0, 1):                          # rank 2 stays away
            a = ca("allreduce", Dev(count, fill=1.0), Dev(count, fill=0))
            q = C.POINTER(U.ucc_coll_req_t)()
            U.check(U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team), "init")
            U.check(U.ucc_collective_post(q), "post")
            reqs.append((a, q))
        t0 = time.time()
        while any(q.contents.status == U.UCC_INPROGRESS for _, q in reqs):
            for r in range(n):
                U.ucc_context_progress(j.procs[r].ctx)
            assert time.time() - t0 < 60, "requests still in progress long after the device-side timeout"
        took = time.time() - t0
        for _, q in reqs:
            assert q.contents.status < 0, q.contents.status          # UCC_ERR_TIMED_OUT
            U.ucc_collective_finalize(q)
        assert 1.0 < took < 30, took
        print(f"  device-side timeout ok (statuses {[q.contents.status if q else None for _, q in reqs]}, {took:.1f} s)", flush=True)


def p2p_active_set():
    """two-member active-set bcast on "device" buffers = send / recv (kernels/nvl_p2p.cu): several pairs at once, both directions,
    a message longer than the channel ring (sender and receiver pipeline), repeated (the channel counters persist across launches)
    and next to a collective of the same team.  Run twice: eager ring only (ZCOPY=n), and with the rendezvous protocol for
    messages >= 64 KB (the sender stores into the receiver's published buffer), incl. more large messages in flight between one
    pair than the board has slots and a small message posted behind a large one (sends keep their post order)."""
    import time
    n = 4

    def drive(j, reqs):
        t0 = time.time()
        while any(q.contents.status == U.UCC_INPROGRESS for _, q in reqs):
            for r in range(n):
                U.ucc_context_progress(j.procs[r].ctx)
            assert time.time() - t0 < 120, "p2p did not complete"
        rt.cudaDeviceSynchronize()
        for _, q in reqs:
            assert q.contents.status == U.UCC_OK, q.contents.status
            U.ucc_collective_finalize(q)

    def msg(team, s_, d_, src, dst, tag):
        out = []
        for r, b in ((s_, src), (d_, dst)):
            a = ca("bcast", b, None, root=s_, count_dst=0, active_set=(s_, d_ - s_, 2), tag=tag)
            q = C.POINTER(U.ucc_coll_req_t)()
            U.check(U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team), "init")
            out.append((a, q))
        return out
    for mode, env in (("ring", NOZC), ("rndv", dict(ZC, UCC_TL_NVL_P2P_RNDV_THRESH="64K"))):
        with UccJob(n, env=dict(BASE, **env)) as j:
            team = j.create_team(range(n))
            for count in (1, 1000, 70001, 300007):
                pairs = [(0, 1), (3, 1), (2, 0), (1, 3)]
                for rep in range(2):
                    bufs, reqs = [], []
                    for i, (s_, d_) in enumerate(pairs):
                        src, dst = Dev(count, fill=rnd(count, 100 * rep + i)), Dev(count, fill=0)
                        bufs.append((src, dst))
                        reqs += msg(team, s_, d_, src, dst, 7 + i)
                    for _, q in reqs:
                        U.check(U.ucc_collective_post(q), "post")
                    drive(j, reqs)
                    for i, (src, dst) in enumerate(bufs):
                        assert np.array_equal(src.a, dst.a), ("p2p", mode, count, rep, pairs[i])
                src = [Dev(777, fill=rnd(777, r)) for r in range(n)]
                dst = [Dev(777, fill=0) for _ in range(n)]
                run(team, [ca("allreduce", src[r], dst[r]) for r in range(n)])
                assert np.allclose(dst[1].a, sum(s.a for s in src))
            # seven messages 2 -> 3 back to back, large and small interleaved; all sends are posted before any receive
            counts = [40000, 3, 50000, 60000, 17, 70000, 45000]
            bufs = [(Dev(c, fill=rnd(c, 900 + i)), Dev(c, fill=0)) for i, c in enumerate(counts)]
            pairs_q = [msg(team, 2, 3, s_, d_, 40 + i) for i, (s_, d_) in enumerate(bufs)]
            for snd, _ in pairs_q:
                U.check(U.ucc_collective_post(snd[1]), "post")
            for _ in range(50):
                for r in range(n):
                    U.ucc_context_progress(j.procs[r].ctx)
            time.sleep(0.5)   # let the sender's kernels run as far as they can without the receiver (they fill the ring)
            for _, rcv in pairs_q:
                U.check(U.ucc_collective_post(rcv[1]), "post")
            drive(j, [x for pq in pairs_q for x in pq])
            for i, (s_, d_) in enumerate(bufs):
                assert np.array_equal(s_.a, d_.a), ("p2p burst", mode, i)
            last = last_launch()
            assert ("rndv" in last) == (mode == "rndv"), (mode, last)   # the last message (45000 floats) is above the threshold
            print(f"  active-set p2p [{mode}] ok", flush=True)


def p2p_late_sender():
    """a receive posted seconds before its send: the channel kernels wait without a deadline (TIMEOUT = 1 s here applies to the
    collectives only), the message arrives and the team's later collectives work; with P2P_TIMEOUT = 1 s the same receive fails"""
    import time
    n = 2
    for p2p_to, expect_ok in (("0", True), ("1s", False)):
        with UccJob(n, env=dict(BASE, **dict(NOZC, UCC_TL_NVL_TIMEOUT="1s", UCC_TL_NVL_P2P_TIMEOUT=p2p_to))) as j:
            team = j.create_team(range(n))
            src, dst = Dev(1000, fill=rnd(1000, 5)), Dev(1000, fill=0)
            reqs = []
            for r, b in ((0, src), (1, dst)):
                a = ca("bcast", b, None, root=0, count_dst=0, active_set=(0, 1, 2), tag=1)
                q = C.POINTER(U.ucc_coll_req_t)()
                U.check(U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team), "init")
                reqs.append((a, q))
            U.check(U.ucc_collective_post(reqs[1][1]), "post recv")
            t0 = time.time()
            while time.time() - t0 < 2.5:
                for r in range(n):
                    U.ucc_context_progress(j.procs[r].ctx)
                time.sleep(0.01)
            if expect_ok:
                assert reqs[1][1].contents.status == U.UCC_INPROGRESS
                U.check(U.ucc_collective_post(reqs[0][1]), "post send")
                t0 = time.time()
                while any(q.contents.status == U.UCC_INPROGRESS for _, q in reqs):
                    for r in range(n):
                        U.ucc_context_progress(j.procs[r].ctx)
                    assert time.time() - t0 < 60
                assert all(q.contents.status == U.UCC_OK for _, q in reqs)
                assert np.array_equal(src.a, dst.a)
                s2 = [Dev(100, fill=rnd(100, r)) for r in range(n)]
                d2 = [Dev(100, fill=0) for _ in range(n)]
                run(team, [ca("allreduce", s2[r], d2[r]) for r in range(n)])
                assert np.allclose(d2[0].a, s2[0].a + s2[1].a)
                for _, q in reqs:
                    U.ucc_collective_finalize(q)
            else:
                assert reqs[1][1].contents.status == U.UCC_ERR_TIMED_OUT, reqs[1][1].contents.status
                U.ucc_collective_finalize(reqs[1][1])
                U.ucc_collective_finalize(reqs[0][1])
    print("  p2p late sender ok", flush=True)


def registered_buffers():
    """ucc_mem_map on device buffers + collectives that carry the GLOBAL handles: the zero-copy kernels get the members' buffers
    from the registrations - here with the exchange board switched OFF (UCC_TL_NVL_ZCOPY would normally need it), so a correct
    result through the in-place kernel proves the registration path"""
    U.lib.ucc_mem_map.argtypes = [U.handle, C.c_int, C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_void_p)]
    U.lib.ucc_mem_map.restype = C.c_int
    U.lib.ucc_mem_unmap.argtypes = [C.POINTER(C.c_void_p)]
    n, count = 4, 40000
    with UccJob(n, env=dict(BASE, UCC_TL_NVL_ZCOPY_THRESH="0", UCC_TL_NVL_ALLREDUCE_ONESHOT_THRESH="0")) as j:
        team = j.create_team(range(n))
        seg_src = [Dev(2 * count, fill=0) for _ in range(n)]     # registered segments; the collective uses the second half
        seg_dst = [Dev(2 * count, fill=0) for _ in range(n)]
        blobs = {"src": [], "dst": []}
        keep = []
        for name, segs in (("src", seg_src), ("dst", seg_dst)):
            for r in range(n):
                seg = U.ucc_mem_map_t(segs[r].ptr, 2 * count * 4)
                params = U.ucc_mem_map_params_t()
                params.segments, params.n_segments = C.pointer(seg), 1
                memh, size = C.c_void_p(), C.c_size_t()
                assert U.lib.ucc_mem_map(j.procs[r].ctx, 0, C.byref(params), C.byref(size), C.byref(memh)) == U.UCC_OK
                blobs[name].append(C.string_at(memh.value, size.value))
                keep.append(memh)
        # every rank imports every member's handle (the application would allgather the blobs)
        glob = {}
        for name in ("src", "dst"):
            for r in range(n):
                arr = (C.c_void_p * n)()
                for p in range(n):
                    b = C.create_string_buffer(blobs[name][p], len(blobs[name][p]))
                    keep.append(b)
                    h = C.c_void_p(C.addressof(b))
                    assert U.lib.ucc_mem_map(j.procs[r].ctx, 1, None, None, C.byref(h)) == U.UCC_OK
                    arr[p] = h.value
                glob[(name, r)] = arr
        for it in range(3):
            for r in range(n):
                seg_src[r].a[count:] = rnd(count, 31 * it + r)
            args = []
            for r in range(n):
                a = coll_args("allreduce", dt="float32", mem_type=CUDA, src_ptr=seg_src[r].ptr + count * 4, dst_ptr=seg_dst[r].ptr + count * 4, count_src=count, count_dst=count)
                a.mask |= U.UCC_COLL_ARGS_FIELD_MEM_MAP_SRC_MEMH | U.UCC_COLL_ARGS_FIELD_MEM_MAP_DST_MEMH
                a.flags |= U.UCC_COLL_ARGS_FLAG_SRC_MEMH_GLOBAL | U.UCC_COLL_ARGS_FLAG_DST_MEMH_GLOBAL
                a.mask |= U.UCC_COLL_ARGS_FIELD_FLAGS
                a.src_memh.global_memh = C.cast(glob[("src", r)], C.POINTER(C.c_void_p))
                a.dst_memh.global_memh = C.cast(glob[("dst", r)], C.POINTER(C.c_void_p))
                args.append(a)
            run(team, args)
            assert "zcopy" in last_launch(), last_launch()
            exp = sum(s.a[count:].copy() for s in seg_src)
            for r in range(n):
                assert np.allclose(seg_dst[r].a[count:], exp), ("memh allreduce", it, r)
                assert np.all(seg_dst[r].a[:count] == 0)
    print("  registered buffers (ucc_mem_map -> zero-copy without the exchange board) ok", flush=True)


def hier_on_device_buffers():
    """cl/hier over a synthetic 2-node x 4-GPU placement with "device" buffers: node sub-teams are tl/nvl teams, the cross-node sub-team
    (leaders) cannot be (different fake hosts) and goes to the host TL.  Only the data-movement chain (2step bcast, plain and pipelined)
    runs here: the reductions of rab / split_rail between the nodes need ec/cuda, which has no host emulation (GPU coverage:
    tests/test_nvl_gpu.py::test_cl_hier_on_cuda_buffers, tests/test_dist_gpu.py fake nodes).  The pipelined variant re-targets the
    fragments' sub-collectives between posts (UCC_COLL_TASK_FLAG_ARGS_UPDATED): tl/nvl tasks capture their arguments at init and are
    rebuilt at post (nvl_rebuild) - a stale task would broadcast the first fragment again."""
    n = 8
    for extra in ({}, {"UCC_CL_HIER_BCAST_2STEP_PIPELINE": "thresh=1k:fragsize=16k:nfrags=2:pdepth=2:sequential"},
                  {"UCC_CL_HIER_BCAST_2STEP_PIPELINE": "thresh=1k:fragsize=8k:nfrags=2:pdepth=3:parallel"}):
        # NODE sub-teams may only be tl/nvl teams: were tl/nvl unable to serve them, cl/hier would decline and the trace would show CL_BASIC
        env = dict(BASE, UCC_CLS="hier,basic", UCC_TL_NVL_TIMEOUT="20s", UCC_CL_HIER_NODE_SBGP_TLS="nvl", **NOZC, **extra)
        with UccJob(n, ppn=4, env=env, cls="hier,basic") as j:
            team = j.create_team()
            for count in (16, 5000, 50001):
                for root in (0, 4):
                    b = [Dev(count, fill=rnd(count, 3 + root) if r == root else 0) for r in range(n)]
                    args = [ca("bcast", b[r], None, root=root, count_dst=0, persistent=True) for r in range(n)]
                    q = team.coll(args)
                    for rep in range(2):
                        if rep:
                            for r in range(n):
                                if r != root:
                                    b[r].a[:] = 0
                        assert q.run() == U.UCC_OK
                        rt.cudaDeviceSynchronize()
                        for r in range(n):
                            assert np.array_equal(b[r].a, b[root].a), (extra, count, root, rep, r)
                    q.finalize()
        print(f"  cl/hier 2step bcast on device buffers ok{' (pipelined: ' + list(extra.values())[0] + ')' if extra else ''}", flush=True)


def lanes():
    """UCC_TL_NVL_SLOTS=4: consecutive collectives of one team take consecutive lanes (own control block, one-shot slots, staging space) and,
    posted stream-ordered on different streams, run CONCURRENTLY (emulated streams are worker threads) - two-shot, one-shot and zero-copy
    kernels, three rounds so that every lane is reused"""
    import time
    rt.cudaStreamCreate.argtypes = [C.POINTER(C.c_void_p)]
    n, K = 3, 4
    for alg, extra, count in (("twoshot", NOZC, 30000), ("oneshot", NOZC, 2000), ("twoshot", ZC, 30000)):
        env = dict(BASE, UCC_TL_NVL_SLOTS="4", UCC_TL_NVL_TUNE=f"allreduce:cuda:inf:@{alg}", UCC_TL_NVL_ALLREDUCE_ONESHOT_THRESH="0" if alg != "oneshot" else "1M", **extra)
        with UccJob(n, env=env) as j:
            team = j.create_team(range(n))
            ees = [[None] * K for _ in range(n)]
            for r in range(n):
                for k in range(K):
                    s = C.c_void_p()
                    assert rt.cudaStreamCreate(C.byref(s)) == 0
                    ep = U.ucc_ee_params_t()
                    ep.ee_type, ep.ee_context, ep.ee_context_size = U.UCC_EE_CUDA_STREAM, s.value, C.sizeof(C.c_void_p)
                    ee = U.handle()
                    U.check(U.ucc_ee_create(team.members[r].team, C.byref(ep), C.byref(ee)), "ee_create")
                    ees[r][k] = ee
            for rnd_ in range(3):
                src = [[Dev(count, fill=rnd(count, 100 * rnd_ + 10 * r + k)) for k in range(K)] for r in range(n)]
                dst = [[Dev(count, fill=0) for _ in range(K)] for _ in range(n)]
                reqs = []
                for k in range(K):
                    for r in range(n):
                        a = ca("allreduce", src[r][k], dst[r][k])
                        q = C.POINTER(U.ucc_coll_req_t)()
                        U.check(U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team), "init")
                        ev = U.ucc_ev_t()
                        ev.ev_type, ev.req = U.UCC_EVENT_COMPUTE_COMPLETE, C.cast(q, C.c_void_p)
                        U.check(U.ucc_collective_triggered_post(ees[r][k], C.byref(ev)), "triggered_post")
                        reqs.append((a, q))
                t0 = time.time()
                while any(q.contents.status == U.UCC_INPROGRESS for _, q in reqs):
                    for r in range(n):
                        U.ucc_context_progress(j.procs[r].ctx)
                        for k in range(K):
                            e = C.POINTER(U.ucc_ev_t)()
                            while U.ucc_ee_get_event(ees[r][k], C.byref(e)) == U.UCC_OK:
                                U.ucc_ee_ack_event(ees[r][k], e)
                    assert time.time() - t0 < 120, "lanes: collectives did not complete"
                rt.cudaDeviceSynchronize()
                for _, q in reqs:
                    assert q.contents.status == U.UCC_OK, q.contents.status
                    U.ucc_collective_finalize(q)
                for k in range(K):
                    exp = sum(src[r][k].a for r in range(n))
                    for r in range(n):
                        assert np.allclose(dst[r][k].a, exp), ("lanes", alg, rnd_, k, r)
            for r in range(n):
                for k in range(K):
                    U.ucc_ee_destroy(ees[r][k])
        print(f"  lanes {alg} {'zcopy' if extra is ZC else 'staged'} ok", flush=True)


def int_avg():
    """AVG on integer datatypes = truncated sum / N, on every reduction kernel"""
    n = 3
    for alg, extra in (("oneshot", NOZC), ("twoshot", NOZC), ("twoshot", ZC), ("ring", NOZC)):
        env = dict(BASE, UCC_TL_NVL_TUNE=f"allreduce:cuda:inf:@{alg}", UCC_TL_NVL_ALLREDUCE_ONESHOT_THRESH="0" if alg != "oneshot" else "1M", **extra)
        with UccJob(n, env=env) as j:
            team = j.create_team(range(n))
            for dt in ("int32", "int64"):
                src = [Dev(1001, np.dtype(dt), fill=(rnd(1001, r + 3, np.dtype(dt)) - 4) * 7) for r in range(n)]
                dst = [Dev(1001, np.dtype(dt), fill=0) for _ in range(n)]
                run(team, [ca("allreduce", src[r], dst[r], dt=dt, op="avg") for r in range(n)])
                tot = sum(s.a.astype(np.int64) for s in src)
                exp = np.trunc(tot / n).astype(np.int64)
                for r in range(n):
                    assert np.array_equal(dst[r].a.astype(np.int64), exp), (alg, dt, r, dst[r].a[:8], exp[:8])
    print("  integer AVG ok", flush=True)


def default_selection():
    """score-map defaults of a team of more than four (tl_nvl_coll.c get_scores): allgather / alltoall of 4-64 MB take the zero-copy
    push kernel, everything else (incl. alltoallv, whose sizes are private: no size-based choice) the pull kernel - checked through the launch note"""
    n = 6
    with UccJob(n, env=dict(BASE, UCC_TL_NVL_ZCOPY="y", UCC_TL_NVL_SYMMETRIC_SIZE="32Mb")) as j:
        team = j.create_team(range(n))
        for blk, want_ag, want_a2av in ((1000, "exchange_pull", "exchange_pull"), (200000, "exchange_push", "exchange_pull"), (400000, "exchange_push", "exchange_pull")):
            count = blk * n
            src = [Dev(blk, fill=rnd(blk, r)) for r in range(n)]
            dst = [Dev(count, fill=0) for _ in range(n)]
            run(team, [ca("allgather", src[r], dst[r]) for r in range(n)])
            assert want_ag in last_launch(), (count, last_launch())
            assert np.array_equal(dst[2].a, np.concatenate([s_.a for s_ in src]))
            src = [Dev(count, fill=rnd(count, 10 + r)) for r in range(n)]
            dst = [Dev(count, fill=0) for _ in range(n)]
            run(team, [ca("alltoall", src[r], dst[r]) for r in range(n)])
            assert want_ag in last_launch(), (count, last_launch())
            assert np.array_equal(dst[3].a, np.concatenate([s_.a[3 * blk:4 * blk] for s_ in src]))
            cnt = [blk] * n
            dsp = [i * blk for i in range(n)]
            dst = [Dev(count, fill=0) for _ in range(n)]
            run(team, [ca("alltoallv", src[r], dst[r], src_counts=cnt, src_displs=dsp, dst_counts=cnt, dst_displs=dsp) for r in range(n)])
            assert want_a2av in last_launch(), (count, last_launch())
            assert np.array_equal(dst[1].a, np.concatenate([s_.a[blk:2 * blk] for s_ in src]))
    print("  default selection ok", flush=True)


def mc_lifecycle():
    """memory-component reference counting across lib instances (src/components/mc/ucc_mc.c): CUDA_MANAGED is an alias of the cuda
    component.  One lib created, destroyed and created again in the same process must find the component initialised (a negative
    reference count once made the second ucc_init skip its init: NULL config, SIGSEGV in the first pooled allocation - seen with
    tools/ucc_test_dist.py -M cuda on two GPUs); and with two libs alive, destroying one must not drop the alias of the other."""
    L = U.lib
    hdr = C.c_void_p()
    MANAGED = U.UCC_MEMORY_TYPE_CUDA_MANAGED
    L.ucc_mc_alloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t, C.c_int]
    L.ucc_mc_free.argtypes = [C.c_void_p]
    L.ucc_mc_available.argtypes = [C.c_int]
    for rep in range(3):
        with UccJob(1, env=dict(BASE)) as j:
            assert L.ucc_mc_alloc(C.byref(hdr), 4096, CUDA) == 0, rep
            assert L.ucc_mc_free(hdr) == 0
            assert L.ucc_mc_available(MANAGED) == 0
    with UccJob(1, env=dict(BASE)) as a:
        with UccJob(1, env=dict(BASE)) as b:
            assert L.ucc_mc_available(MANAGED) == 0
        assert L.ucc_mc_available(MANAGED) == 0, "alias dropped while a lib is alive"
        assert L.ucc_mc_alloc(C.byref(hdr), 4096, CUDA) == 0 and L.ucc_mc_free(hdr) == 0
    print("  mc lifecycle ok", flush=True)


def p2p_fuzz():
    """send / recv state machine under random traffic: for several seeds, 30 messages between random ordered pairs of a 4-member team,
    sizes from 1 element to 1.2 MB (once with eager ring and rendezvous mixed - threshold 64 KB, more large messages per pair than
    board slots - and once with everything through the eager ring, larger than the ring included), posted in a random global order that only keeps each pair's sends and each pair's receives in message order, with
    random amounts of progress in between.  Every message must arrive intact and every request must complete."""
    import time
    n = 4
    rt.cudaStreamCreate.argtypes = [C.POINTER(C.c_void_p)]

    def traffic(thresh, seeds):
        with UccJob(n, env=dict(BASE, **dict(ZC, UCC_TL_NVL_P2P_RNDV_THRESH=thresh))) as j:
            team = j.create_team(range(n))
            # stream-ordered posts, one stream per (rank, peer, direction): a kernel of the eager ring may wait for its peer, so - exactly as
            # with NCCL - two operations that must not wait for each other must not share a stream
            ees = {}
            for r in range(n):
                for p_ in range(n):
                    for kind in ("send", "recv"):
                        if p_ == r:
                            continue
                        s_ = C.c_void_p()
                        assert rt.cudaStreamCreate(C.byref(s_)) == 0
                        ep = U.ucc_ee_params_t()
                        ep.ee_type, ep.ee_context, ep.ee_context_size = U.UCC_EE_CUDA_STREAM, s_.value, C.sizeof(C.c_void_p)
                        ee = U.handle()
                        U.check(U.ucc_ee_create(team.members[r].team, C.byref(ep), C.byref(ee)), "ee_create")
                        ees[(r, p_, kind)] = ee

            def drain():
                for ee in ees.values():
                    e = C.POINTER(U.ucc_ev_t)()
                    while U.ucc_ee_get_event(ee, C.byref(e)) == U.UCC_OK:
                        U.ucc_ee_ack_event(ee, e)
            for seed in range(seeds):
                rng = np.random.default_rng(1000 + seed)
                msgs = []
                for i in range(30):
                    s_, d_ = rng.choice(n, 2, replace=False)
                    count = int(rng.choice([1, 7, 300, 5000, 16384, 20000, 70001, 150000, 300007]))
                    src, dst = Dev(count, fill=rnd(count, 50 * seed + i)), Dev(count, fill=0)
                    reqs = {}
                    for r, b, key in ((s_, src, "send"), (d_, dst, "recv")):
                        a = ca("bcast", b, None, root=int(s_), count_dst=0, active_set=(int(s_), int(d_) - int(s_), 2), tag=i)
                        q = C.POINTER(U.ucc_coll_req_t)()
                        U.check(U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team), "init")
                        reqs[key] = (a, q)
                    msgs.append((int(s_), int(d_), src, dst, reqs))
                # global post order: a random interleaving in which, per ordered pair, sends keep their order and receives keep theirs
                events = [(i, "send") for i in range(len(msgs))] + [(i, "recv") for i in range(len(msgs))]
                order = list(rng.permutation(len(events)))
                pending = [events[k] for k in order]
                while pending:
                    progressed = False
                    for k, (i, kind) in enumerate(pending):
                        pair = (msgs[i][0], msgs[i][1], kind)
                        first = min(m for m, (mm, kk) in [(e[0], e) for e in pending] if (msgs[m][0], msgs[m][1], kk) == pair)
                        if i != first:
                            continue
                        ev = U.ucc_ev_t()
                        ev.ev_type, ev.req = U.UCC_EVENT_COMPUTE_COMPLETE, C.cast(msgs[i][4][kind][1], C.c_void_p)
                        me_, peer_ = (msgs[i][0], msgs[i][1]) if kind == "send" else (msgs[i][1], msgs[i][0])
                        U.check(U.ucc_collective_triggered_post(ees[(me_, peer_, kind)], C.byref(ev)), "triggered_post")
                        pending.pop(k)
                        progressed = True
                        break
                    assert progressed
                    for _ in range(int(rng.integers(0, 4))):
                        for r in range(n):
                            U.ucc_context_progress(j.procs[r].ctx)
                    if rng.integers(0, 8) == 0:   # a collective of the same team while messages are in flight (channels and collectives share nothing)
                        cnt = int(rng.choice([5, 3000, 90000]))
                        csrc = [Dev(cnt, fill=rnd(cnt, 7000 + len(pending) + r)) for r in range(n)]
                        cdst = [Dev(cnt, fill=0) for _ in range(n)]
                        cq = team.coll([ca("allreduce", csrc[r], cdst[r]) for r in range(n)])   # (no device-wide sync as in run(): receives may be parked)
                        assert cq.run() == U.UCC_OK
                        cq.finalize()
                        assert np.allclose(cdst[int(rng.integers(0, n))].a, sum(x.a for x in csrc)), ("allreduce next to p2p traffic", thresh, seed)
                t0 = time.time()
                allq = [m[4][k][1] for m in msgs for k in ("send", "recv")]
                while any(q.contents.status == U.UCC_INPROGRESS for q in allq):
                    for r in range(n):
                        U.ucc_context_progress(j.procs[r].ctx)
                    drain()
                    assert time.time() - t0 < 180, ("p2p fuzz did not complete", seed)
                rt.cudaDeviceSynchronize()
                for i, m in enumerate(msgs):
                    for k in ("send", "recv"):
                        assert m[4][k][1].contents.status == U.UCC_OK, (seed, i, k)
                        U.ucc_collective_finalize(m[4][k][1])
                    assert np.array_equal(m[2].a, m[3].a), ("p2p fuzz data", seed, i, m[0], m[1], m[2].a.size)
                drain()
            for ee in ees.values():
                U.ucc_ee_destroy(ee)
    more = int(os.environ.get("B200_FUZZ_SEEDS", "0"))
    traffic("64K", max(6, more))
    traffic("inf", max(3, more // 2))      # everything through the eager ring, incl. messages larger than the ring (1 MB)
    print("  p2p fuzz ok", flush=True)


def coll_fuzz():
    """random programs on the tl/nvl plugin: for several seeds, 40 collectives of random kind / size / datatype / operator / root on a
    4-member team and on a 3-member sub-team, up to three of them outstanding at once (posted back to back in the same order on every
    member, as UCC requires), with the staged kernels, with the zero-copy exchange (deferred launches), and both again on several lanes
    (UCC_TL_NVL_SLOTS: consecutive collectives use consecutive heap images), always with a heap so small that large messages take several
    rounds; every result is checked against numpy."""
    kinds = ["allreduce", "allgather", "alltoall", "reduce_scatter", "bcast", "reduce", "barrier", "gather", "scatter", "allgatherv", "alltoallv", "reduce_scatterv"]
    def random_tune(seed):
        """a random (non-NVLS) algorithm for every collective type; what an algorithm declines goes down the score chain"""
        g = np.random.default_rng(seed)
        pick = lambda *names: names[int(g.integers(0, len(names)))]  # noqa: E731
        return "#".join([f"allreduce:cuda:inf:@{pick('twoshot', 'oneshot', 'ring', 'rhd')}", f"reduce_scatter:cuda:inf:@{pick('twoshot', 'ring', 'rhd', 'oneshot')}",
                         f"reduce_scatterv:cuda:inf:@{pick('twoshot', 'ring', 'oneshot')}", f"allgather:cuda:inf:@{pick('pull', 'ring', 'push', 'ce')}",
                         f"allgatherv:cuda:inf:@{pick('pull', 'ring', 'push', 'ce')}", f"alltoall:cuda:inf:@{pick('pull', 'push', 'ce')}",
                         f"alltoallv:cuda:inf:@{pick('pull', 'push', 'ce')}"])
    for mode, extra in (("staged", NOZC), ("zcopy", dict(ZC, UCC_TL_NVL_ZCOPY_THRESH="64K")), ("staged, 4 lanes", dict(NOZC, UCC_TL_NVL_SLOTS="4")),
                        ("zcopy, 3 lanes", dict(ZC, UCC_TL_NVL_ZCOPY_THRESH="64K", UCC_TL_NVL_SLOTS="3")),
                        ("zcopy, random algorithms A", dict(ZC, UCC_TL_NVL_ZCOPY_THRESH="0", UCC_TL_NVL_TUNE=random_tune(1))),
                        ("zcopy, random algorithms B", dict(ZC, UCC_TL_NVL_ZCOPY_THRESH="64K", UCC_TL_NVL_TUNE=random_tune(int(os.environ.get("B200_FUZZ_TUNE", "2"))))),
                        ("staged, random algorithms C", dict(NOZC, UCC_TL_NVL_TUNE=random_tune(3)))):
        with UccJob(4, env=dict(BASE, **extra)) as j:
            teams = [j.create_team(range(4)), j.create_team([3, 0, 2])]
            for seed in range(int(os.environ.get("B200_FUZZ_SEEDS", "4"))):
                rng = np.random.default_rng(500 + seed)
                window = []

                def retire(k):
                    while len(window) > k:
                        q, check, what = window.pop(0)
                        st = q.wait()
                        assert st == U.UCC_OK, (mode, seed, what, U.status_str(st))
                        q.finalize()
                        check()    # (no device-wide synchronisation here: other collectives are outstanding and a zero-copy one may still need host progress to be launched)
                for step in range(40):
                    team = teams[int(rng.integers(0, 2))]
                    n = len(team.members)
                    kind = kinds[int(rng.integers(0, len(kinds)))]
                    blk = int(rng.choice([1, 3, 100, 4097, 30011, 120001]))
                    if kind not in ("allreduce", "reduce_scatter", "reduce", "reduce_scatterv") and blk > 30011:
                        blk = 30011      # the data-movement kernels stage the whole message in the (here 1 MB) heap; only reductions work in rounds
                    dt = "float32" if rng.integers(0, 2) else "int32"
                    npdt = np.dtype(dt)
                    op = "sum" if rng.integers(0, 3) else "max"
                    root = int(rng.integers(0, n))
                    what = (step, kind, n, blk, dt, op, root)
                    mk = lambda c, sd: Dev(c, npdt, fill=(rnd(c, sd, npdt) if dt == "float32" else (rnd(c, sd, npdt) % 1000)))  # noqa: E731
                    red = (lambda arrs: np.sum(arrs, 0)) if op == "sum" else (lambda arrs: np.max(arrs, 0))
                    if kind in ("allreduce", "allgather", "alltoall") and rng.integers(0, 5) == 0:
                        # persistent request: posted three times with new input each time (zero-copy: the pointer tables are cached after the first post)
                        retire(0)
                        mult = 1 if kind == "allreduce" else n
                        src = [mk(blk * (n if kind == "alltoall" else 1), 10 * step + r) for r in range(n)]
                        dst = [Dev(blk * mult, npdt, fill=0) for _ in range(n)]
                        q = team.coll([ca(kind, src[r], dst[r], dt=dt, op=op, persistent=True) for r in range(n)])
                        for rep in range(3):
                            for r in range(n):
                                src[r].a[:] = rnd(src[r].a.size, 1000 * rep + 10 * step + r, npdt)
                                dst[r].a[:] = 0
                            q.post()
                            assert q.wait() == U.UCC_OK, (mode, seed, what, "persistent", rep)
                            for r in range(n):
                                if kind == "allreduce":
                                    np.testing.assert_allclose(dst[r].a, red([x.a.copy() for x in src]), rtol=1e-5, err_msg=str((what, rep)))
                                elif kind == "allgather":
                                    np.testing.assert_array_equal(dst[r].a, np.concatenate([x.a for x in src]), err_msg=str((what, rep)))
                                else:
                                    np.testing.assert_array_equal(dst[r].a, np.concatenate([src[p_].a[r * blk:(r + 1) * blk] for p_ in range(n)]), err_msg=str((what, rep)))
                        q.finalize()
                        continue
                    inplace = kind in ("allreduce", "allgather", "reduce_scatter") and rng.integers(0, 3) == 0
                    what = what + (("inplace",) if inplace else ())
                    if kind == "allreduce":
                        src = [mk(blk, 10 * step + r) for r in range(n)]; dst = [Dev(blk, npdt, fill=(src[r].a if inplace else 0)) for r in range(n)]
                        args = [ca(kind, None if inplace else src[r], dst[r], dt=dt, op=op, inplace=inplace) for r in range(n)]
                        exp = red([x.a.copy() for x in src])
                        check = lambda dst=dst, exp=exp, what=what: [np.testing.assert_allclose(d.a, exp, rtol=1e-5, err_msg=str(what)) for d in dst]  # noqa: E731
                    elif kind == "allgather":
                        src = [mk(blk, 10 * step + r) for r in range(n)]; dst = [Dev(blk * n, npdt, fill=0) for _ in range(n)]
                        if inplace:
                            for r in range(n):
                                dst[r].a[r * blk:(r + 1) * blk] = src[r].a
                        args = [ca(kind, None if inplace else src[r], dst[r], dt=dt, inplace=inplace) for r in range(n)]
                        exp = np.concatenate([x.a for x in src])
                        check = lambda dst=dst, exp=exp, what=what: [np.testing.assert_array_equal(d.a, exp, err_msg=str(what)) for d in dst]  # noqa: E731
                    elif kind == "alltoall":
                        src = [mk(blk * n, 10 * step + r) for r in range(n)]; dst = [Dev(blk * n, npdt, fill=0) for _ in range(n)]
                        args = [ca(kind, src[r], dst[r], dt=dt) for r in range(n)]
                        check = lambda src=src, dst=dst, n=n, blk=blk, what=what: [np.testing.assert_array_equal(dst[r].a, np.concatenate([src[p].a[r * blk:(r + 1) * blk] for p in range(n)]), err_msg=str(what)) for r in range(n)]  # noqa: E731
                    elif kind == "reduce_scatter":
                        src = [mk(blk * n, 10 * step + r) for r in range(n)]; dst = [Dev(blk, npdt, fill=0) for _ in range(n)]
                        exp = red([x.a.copy() for x in src])
                        if inplace:   # the whole vector is in dst, the result block stays at its offset
                            dst = [Dev(blk * n, npdt, fill=src[r].a) for r in range(n)]
                            args = [ca(kind, None, dst[r], dt=dt, op=op, inplace=True) for r in range(n)]
                            check = lambda dst=dst, exp=exp, blk=blk, n=n, what=what: [np.testing.assert_allclose(dst[r].a[r * blk:(r + 1) * blk], exp[r * blk:(r + 1) * blk], rtol=1e-5, err_msg=str(what)) for r in range(n)]  # noqa: E731
                        else:
                            args = [ca(kind, src[r], dst[r], dt=dt, op=op) for r in range(n)]
                            check = lambda dst=dst, exp=exp, blk=blk, n=n, what=what: [np.testing.assert_allclose(dst[r].a, exp[r * blk:(r + 1) * blk], rtol=1e-5, err_msg=str(what)) for r in range(n)]  # noqa: E731
                    elif kind == "allgatherv":
                        counts = [int(rng.integers(0, blk + 1)) for _ in range(n)]
                        offs = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(int)
                        src = [mk(counts[r], 10 * step + r) for r in range(n)]; dst = [Dev(max(sum(counts), 1), npdt, fill=0) for _ in range(n)]
                        args = [ca(kind, src[r], dst[r], dt=dt, count_src=counts[r], dst_counts=counts, dst_displs=offs) for r in range(n)]
                        exp = np.concatenate([x.a[:counts[r]] for r, x in enumerate(src)])
                        check = lambda dst=dst, exp=exp, tot=sum(counts), what=what: [np.testing.assert_array_equal(d.a[:tot], exp, err_msg=str(what)) for d in dst]  # noqa: E731
                    elif kind == "alltoallv":
                        m = rng.integers(0, min(blk, 20000) + 1, (n, n))
                        sd = [np.concatenate([[0], np.cumsum(m[r])[:-1]]).astype(int) for r in range(n)]
                        rd = [np.concatenate([[0], np.cumsum(m[:, r])[:-1]]).astype(int) for r in range(n)]
                        src = [mk(max(int(m[r].sum()), 1), 10 * step + r) for r in range(n)]
                        dst = [Dev(max(int(m[:, r].sum()), 1), npdt, fill=0) for r in range(n)]
                        args = [ca(kind, src[r], dst[r], dt=dt, src_counts=m[r], src_displs=sd[r], dst_counts=m[:, r], dst_displs=rd[r]) for r in range(n)]
                        check = lambda src=src, dst=dst, m=m, sd=sd, n=n, what=what: [np.testing.assert_array_equal(dst[r].a[:int(m[:, r].sum())], np.concatenate([src[p_].a[sd[p_][r]:sd[p_][r] + m[p_][r]] for p_ in range(n)]), err_msg=str(what)) for r in range(n)]  # noqa: E731
                    elif kind == "reduce_scatterv":
                        counts = [int(rng.integers(0, blk + 1)) for _ in range(n)]
                        offs = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(int)
                        tot = max(sum(counts), 1)
                        src = [mk(tot, 10 * step + r) for r in range(n)]; dst = [Dev(max(counts[r], 1), npdt, fill=0) for r in range(n)]
                        args = [ca(kind, src[r], dst[r], dt=dt, op=op, count_src=sum(counts), dst_counts=counts, dst_displs=offs) for r in range(n)]
                        exp = red([x.a.copy() for x in src])
                        check = lambda dst=dst, exp=exp, counts=counts, offs=offs, n=n, what=what: [np.testing.assert_allclose(dst[r].a[:counts[r]], exp[offs[r]:offs[r] + counts[r]], rtol=1e-5, err_msg=str(what)) for r in range(n)]  # noqa: E731
                    elif kind == "bcast":
                        b = [mk(blk, 10 * step + 7) if r == root else Dev(blk, npdt, fill=0) for r in range(n)]
                        exp = b[root].a.copy()
                        args = [ca(kind, b[r], None, dt=dt, root=root, count_dst=0) for r in range(n)]
                        check = lambda b=b, exp=exp, what=what: [np.testing.assert_array_equal(x.a, exp, err_msg=str(what)) for x in b]  # noqa: E731
                    elif kind == "reduce":
                        src = [mk(blk, 10 * step + r) for r in range(n)]; out = Dev(blk, npdt, fill=0)
                        args = [ca(kind, src[r], out if r == root else None, dt=dt, op=op, root=root, count_dst=blk if r == root else 0) for r in range(n)]
                        exp = red([x.a.copy() for x in src])
                        check = lambda out=out, exp=exp, what=what: np.testing.assert_allclose(out.a, exp, rtol=1e-5, err_msg=str(what))  # noqa: E731
                    elif kind == "gather":
                        src = [mk(blk, 10 * step + r) for r in range(n)]; g = Dev(blk * n, npdt, fill=0)
                        args = [ca(kind, src[r], g if r == root else None, dt=dt, root=root, count_dst=blk * n if r == root else 0) for r in range(n)]
                        exp = np.concatenate([x.a for x in src])
                        check = lambda g=g, exp=exp, what=what: np.testing.assert_array_equal(g.a, exp, err_msg=str(what))  # noqa: E731
                    elif kind == "scatter":
                        big = mk(blk * n, 10 * step + 3); outs = [Dev(blk, npdt, fill=0) for _ in range(n)]
                        args = [ca(kind, big if r == root else None, outs[r], dt=dt, root=root, count_src=blk * n if r == root else 0) for r in range(n)]
                        check = lambda big=big, outs=outs, blk=blk, n=n, what=what: [np.testing.assert_array_equal(outs[r].a, big.a[r * blk:(r + 1) * blk], err_msg=str(what)) for r in range(n)]  # noqa: E731
                    else:
                        args = [coll_args("barrier") for _ in range(n)]
                        check = lambda: None  # noqa: E731
                    q = team.coll(args)
                    q.post()
                    window.append((q, check, what))
                    retire(int(rng.integers(0, 3)))
                retire(0)
        print(f"  collective fuzz [{mode}] ok", flush=True)


def resource_cycles():
    """team / context life cycle of the tl/nvl plugin: jobs and teams (random subsets, zero-copy boards, p2p side streams, EEs) created,
    used and destroyed many times - file descriptors, POSIX segments and emulated device allocations must not accumulate"""
    import glob
    rt.cudaStreamCreate.argtypes = [C.POINTER(C.c_void_p)]

    def nfd():
        return len(os.listdir("/proc/self/fd"))

    def cycle(i):
        rng = np.random.default_rng(i)
        with UccJob(4, env=dict(BASE, **dict(ZC, UCC_TL_NVL_P2P_RNDV_THRESH="64K"))) as j:
            for _ in range(3):
                ranks = sorted(rng.choice(4, size=int(rng.integers(2, 5)), replace=False).tolist())
                team = j.create_team(ranks)
                n = len(ranks)
                src = [Dev(30000, fill=rnd(30000, r)) for r in range(n)]
                dst = [Dev(30000, fill=0) for _ in range(n)]
                run(team, [ca("allreduce", src[r], dst[r]) for r in range(n)])
                assert np.allclose(dst[0].a, sum(x.a for x in src))
                big_s, big_d = Dev(40000, fill=rnd(40000, 9)), Dev(40000, fill=0)      # one rendezvous message: side stream + board entry
                reqs = []
                for r, b in ((0, big_s), (1, big_d)):
                    a = ca("bcast", b, None, root=0, count_dst=0, active_set=(0, 1, 2), tag=1)
                    q = C.POINTER(U.ucc_coll_req_t)()
                    U.check(U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team), "init")
                    U.check(U.ucc_collective_post(q), "post")
                    reqs.append((a, q))
                while any(q.contents.status == U.UCC_INPROGRESS for _, q in reqs):
                    for p_ in j.procs:
                        p_.progress()
                for _, q in reqs:
                    assert q.contents.status == U.UCC_OK
                    U.ucc_collective_finalize(q)
                assert np.array_equal(big_s.a, big_d.a)
                team.destroy()
    rt.emu_live_objects.restype = C.c_long
    live = lambda: tuple(rt.emu_live_objects(k) for k in range(3))   # noqa: E731  streams, events, allocations of the emulated runtime
    for i in range(3):
        cycle(i)
    f0, s0, l0, d0 = nfd(), len(glob.glob(f"/dev/shm/ucc_b200*.{os.getpid()}.*")), live(), Dev.created
    for i in range(3, 15):
        cycle(i)
    f1, s1, l1, d1 = nfd(), len(glob.glob(f"/dev/shm/ucc_b200*.{os.getpid()}.*")), live(), Dev.created
    assert f1 <= f0 + 2, ("file descriptors leak", f0, f1)
    assert s1 <= s0, ("shared-memory segments leak", s0, s1)
    assert l1[0] <= l0[0] and l1[1] <= l0[1], ("CUDA streams / events leak", l0, l1)
    assert l1[2] - l0[2] <= d1 - d0, ("device / pinned allocations leak (beyond the test's own, never freed, buffers)", l0, l1, d1 - d0)
    print(f"  resource cycles ok (fds {f0} -> {f1}, segments {s0} -> {s1}, streams / events / allocations {l0} -> {l1})", flush=True)


SCENARIOS = {
    "defaults": default_selection,
    "allreduce": lambda: [allreduce_suite(a, e) for a, e in (("oneshot", NOZC), ("twoshot", NOZC), ("twoshot", ZC), ("ring", NOZC), ("rhd", NOZC))],
    "colls_staged": lambda: other_colls(NOZC),
    "colls_zcopy": lambda: other_colls(ZC),
    "colls_push": lambda: other_colls(ZC, "allgather:cuda:inf:@push#allgatherv:cuda:inf:@push#alltoall:cuda:inf:@push#alltoallv:cuda:inf:@push#reduce_scatter:cuda:inf:@oneshot#reduce_scatterv:cuda:inf:@oneshot"),
    "colls_ce": lambda: other_colls(ZC, "allgather:cuda:inf:@ce#allgatherv:cuda:inf:@ce#alltoall:cuda:inf:@ce#alltoallv:cuda:inf:@ce"),
    "colls_ring": lambda: other_colls(NOZC, "allgather:cuda:inf:@ring#allgatherv:cuda:inf:@ring#reduce_scatter:cuda:inf:@ring#reduce_scatterv:cuda:inf:@ring"),
    "misc": lambda: [mc_lifecycle(), resource_cycles(), persistent_and_teams(), asymmetric_memory()],
    "triggered": lambda: [triggered(NOZC), triggered(ZC)],
    "timeout": device_timeout,
    "cross_team": lambda: [cross_team_order(NOZC), cross_team_order(ZC)],
    "p2p": lambda: [p2p_active_set(), p2p_late_sender(), int_avg()],
    "p2p_fuzz": p2p_fuzz,
    "coll_fuzz": coll_fuzz,
    "memh": registered_buffers,
    "hier": hier_on_device_buffers,
    "lanes": lanes,
}

if __name__ == "__main__":
    SCENARIOS[sys.argv[1]]()
    print("HOSTEMU_WORKER_OK", flush=True)
