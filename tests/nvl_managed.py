"""Collectives and send / recv of tl/nvl on CUDA managed memory (cudaMallocManaged), shared by the host-emulated worker
(tests/hostemu_managed_worker.py) and the GPU test (tests/test_nvl_managed_gpu.py).

A managed buffer is never mapped by a peer: its owner publishes it as not mappable, so every path that would read or write it in
place on another member runs its staged form instead.  Every case here runs with UCC_TLS=nvl, so a request tl/nvl turned down
fails instead of going to another TL, checks the result byte for byte against numpy on integer data, and checks the launch note:
it must name a tl/nvl kernel, and never a direct (zero-copy) form when a managed buffer sits on a side that form maps.

`h` provides alloc(nelems, managed) -> buffer with .ptr, .write(int32 array), .read() -> int32 array; run(team, args);
last_launch(); and args(coll, src_buf, dst_buf, smt, dmt, **coll_args keywords)."""
import numpy as np

from ucc_b200 import capi as U

CUDA, MANAGED = U.UCC_MEMORY_TYPE_CUDA, U.UCC_MEMORY_TYPE_CUDA_MANAGED
THRESH = 16 << 10                      # UCC_TL_NVL_ZCOPY_THRESH and UCC_TL_NVL_P2P_RNDV_THRESH
ENV = {"UCC_TLS": "nvl", "UCC_TL_NVL_ZCOPY": "y", "UCC_TL_NVL_ZCOPY_THRESH": "16K", "UCC_TL_NVL_P2P_RNDV_THRESH": "16K",
       "UCC_TL_NVL_ALLREDUCE_ONESHOT_THRESH": "0", "UCC_TL_NVL_SYMMETRIC_SIZE": "1Mb"}
SMALL, LARGE = 37, 6000                # int32 elements per block: 148 B, and 24 KB (above both thresholds)
MIXES = (("m", "m"), ("m", "d"), ("d", "m"))   # (src, dst) memory: managed / device
DIRECT = ("(direct)", "zcopy", "exchange_push", "exchange_swap", "rndv")
NVL_NOTES = ("oneshot", "twoshot", "nvls", "ring", "rhd", "allgather_symm", "exchange_", "self_copy", "barrier", "p2p_")
# which buffers the direct form of the path tl/nvl picks for the collective maps on the peers
MAPS = {"allreduce": "sd", "reduce": "sd", "reduce_scatter": "s", "reduce_scatterv": "s", "allgather": "s", "allgatherv": "s",
        "alltoall": "s", "alltoallv": "s", "bcast": "s", "gather": "s", "gatherv": "s", "scatter": "s", "scatterv": "s"}
COLLS = tuple(MAPS)   # (barrier, fanin and fanout carry no buffer: UCC selects them as host collectives whatever memory is in use)


def rnd(n, seed):
    return np.random.default_rng(seed).integers(-50, 50, n).astype(np.int32)


def is_direct(note):
    return any(k in note for k in DIRECT)


def check_note(h, what, mapped_managed):
    note = h.last_launch()
    assert note.startswith(NVL_NOTES), (what, note)
    if mapped_managed:
        assert not is_direct(note), ("a managed buffer was mapped by a peer", what, note)
    return note


class Case:
    """one collective on one team: buffers per rank, the arguments and the expected contents of what it writes"""

    def __init__(self, h, n, coll, blk, mix, inplace, seed, root):
        self.h, self.n, self.coll, self.blk, self.inplace, self.root = h, n, coll, blk, inplace, root
        self.sm, self.dm = (k == "m" for k in mix)
        self.seed = seed
        self.src, self.dst, self.args, self.exp = [None] * n, [None] * n, [None] * n, {}

    def buf(self, nelems, managed, data=None):
        b = self.h.alloc(max(nelems, 1), managed)
        b.write(data if data is not None else np.zeros(max(nelems, 1), np.int32))
        return b

    def build(self):
        n, blk, coll, ip, root, h = self.n, self.blk, self.coll, self.inplace, self.root, self.h
        counts = [blk + 3 * r for r in range(n)]
        displs = [int(x) for x in np.concatenate([[0], np.cumsum(counts)[:-1]])]
        tot = sum(counts)
        smt, dmt = (MANAGED if self.sm else CUDA), (MANAGED if self.dm else CUDA)
        data = [rnd(tot * n + blk * n, self.seed + r) for r in range(n)]
        A = lambda r, s, d, **kw: h.args(coll, s, d, smt, dmt, **kw)   # noqa: E731
        if coll in ("allreduce", "reduce"):
            cnt = blk * n
            ins = [data[r][:cnt] for r in range(n)]
            tot_ = sum(x.astype(np.int64) for x in ins).astype(np.int32)
            for r in range(n):
                has_dst = coll == "allreduce" or r == root
                if ip and has_dst:
                    self.dst[r] = self.buf(cnt, self.dm, ins[r])
                    self.args[r] = A(r, None, self.dst[r], inplace=True, count_src=cnt, count_dst=cnt, root=root)
                else:
                    self.src[r] = self.buf(cnt, self.sm, ins[r])
                    self.dst[r] = self.buf(cnt, self.dm) if has_dst else None
                    self.args[r] = A(r, self.src[r], self.dst[r], count_src=cnt, count_dst=cnt if has_dst else 0, root=root)
                if has_dst:
                    self.exp[r] = tot_
        elif coll in ("reduce_scatter", "reduce_scatterv"):
            v = coll == "reduce_scatterv"
            cs = counts if v else [blk] * n
            ds = displs if v else [blk * r for r in range(n)]
            cnt = sum(cs)
            ins = [data[r][:cnt] for r in range(n)]
            tot_ = sum(x.astype(np.int64) for x in ins).astype(np.int32)
            for r in range(n):
                kw = dict(dst_counts=cs, dst_displs=ds) if v else {}
                if ip:
                    self.dst[r] = self.buf(cnt, self.dm, ins[r])
                    self.args[r] = A(r, None, self.dst[r], inplace=True, count_src=cnt, count_dst=cnt, **kw)
                    self.exp[r] = (ds[r], tot_[ds[r]:ds[r] + cs[r]])
                else:
                    self.src[r] = self.buf(cnt, self.sm, ins[r])
                    self.dst[r] = self.buf(cs[r], self.dm)
                    self.args[r] = A(r, self.src[r], self.dst[r], count_src=cnt, count_dst=cs[r], **kw)
                    self.exp[r] = tot_[ds[r]:ds[r] + cs[r]]
        elif coll in ("allgather", "allgatherv", "gather", "gatherv"):
            v = coll.endswith("v")
            rooted = coll.startswith("gather")
            cs = counts if v else [blk] * n
            ds = displs if v else [blk * r for r in range(n)]
            cnt = sum(cs)
            blocks = [data[r][:cs[r]] for r in range(n)]
            full = np.concatenate(blocks)
            for r in range(n):
                has_dst = not rooted or r == root
                kw = dict(dst_counts=cs, dst_displs=ds) if v and has_dst else {}
                if ip and has_dst:
                    init = np.zeros(cnt, np.int32)
                    init[ds[r]:ds[r] + cs[r]] = blocks[r]
                    self.dst[r] = self.buf(cnt, self.dm, init)
                    self.args[r] = A(r, None, self.dst[r], inplace=True, count_src=cs[r], count_dst=cnt, root=root, **kw)
                else:
                    self.src[r] = self.buf(cs[r], self.sm, blocks[r])
                    self.dst[r] = self.buf(cnt, self.dm) if has_dst else None
                    self.args[r] = A(r, self.src[r], self.dst[r], count_src=cs[r], count_dst=cnt if has_dst else 0, root=root, **kw)
                if has_dst:
                    self.exp[r] = full
        elif coll in ("scatter", "scatterv"):
            v = coll == "scatterv"
            cs = counts if v else [blk] * n
            ds = displs if v else [blk * r for r in range(n)]
            cnt = sum(cs)
            whole = data[root][:cnt]
            for r in range(n):
                kw = dict(src_counts=cs, src_displs=ds) if v and r == root else {}
                if r == root:
                    self.src[r] = self.buf(cnt, self.sm, whole)
                    if ip:
                        self.args[r] = A(r, self.src[r], None, inplace=True, count_src=cnt, count_dst=cs[r], root=root, **kw)
                        self.exp[r] = ("src", whole)
                        continue
                self.dst[r] = self.buf(cs[r], self.dm)
                self.args[r] = A(r, self.src[r], self.dst[r], count_src=cnt if r == root else 0, count_dst=cs[r], root=root, **kw)
                self.exp[r] = whole[ds[r]:ds[r] + cs[r]]
        elif coll == "bcast":
            cnt = blk * n
            for r in range(n):
                self.src[r] = self.buf(cnt, self.sm, data[root][:cnt] if r == root else None)
                self.args[r] = A(r, self.src[r], None, count_src=cnt, count_dst=0, root=root)
                self.exp[r] = ("src", data[root][:cnt])
        elif coll == "alltoall":
            cnt = blk * n
            ins = [data[r][:cnt] for r in range(n)]
            for r in range(n):
                exp = np.concatenate([ins[p][r * blk:(r + 1) * blk] for p in range(n)])
                if ip:
                    self.dst[r] = self.buf(cnt, self.dm, ins[r])
                    self.args[r] = A(r, None, self.dst[r], inplace=True, count_src=cnt, count_dst=cnt)
                else:
                    self.src[r] = self.buf(cnt, self.sm, ins[r])
                    self.dst[r] = self.buf(cnt, self.dm)
                    self.args[r] = A(r, self.src[r], self.dst[r], count_src=cnt, count_dst=cnt)
                self.exp[r] = exp
        elif coll == "alltoallv":
            # m[s][d]: elements member s sends to member d; in place needs m symmetric (one layout describes both directions)
            m = np.array([[blk + (s + d) % 3 if ip else blk + (2 * s + d) % 5 for d in range(n)] for s in range(n)])
            for r in range(n):
                sd = [int(x) for x in np.concatenate([[0], np.cumsum(m[r])[:-1]])]
                rd = [int(x) for x in np.concatenate([[0], np.cumsum(m[:, r])[:-1]])]
                ins = data[r][:int(m[r].sum())]
                self.exp[r] = np.concatenate([data[p][:int(m[p].sum())][int(np.cumsum(np.r_[0, m[p]])[r]):][:m[p][r]] for p in range(n)])
                if ip:
                    self.dst[r] = self.buf(int(m[r].sum()), self.dm, ins)
                    self.args[r] = A(r, None, self.dst[r], inplace=True, dst_counts=m[:, r], dst_displs=rd)
                else:
                    self.src[r] = self.buf(int(m[r].sum()), self.sm, ins)
                    self.dst[r] = self.buf(int(m[:, r].sum()), self.dm)
                    self.args[r] = A(r, self.src[r], self.dst[r], src_counts=m[r], src_displs=sd, dst_counts=m[:, r], dst_displs=rd)
        return self

    def mapped_managed(self):
        """a managed buffer sits on a side that the direct form of this collective's path maps"""
        if self.coll not in MAPS:
            return False
        if self.inplace:
            return self.dm if self.coll != "scatter" and self.coll != "scatterv" else self.sm
        if self.coll in ("scatter", "scatterv"):
            return self.dm      # the core stages the root's source through a buffer of its destination's memory type
        if self.coll in ("reduce", "gather", "gatherv"):
            return self.sm      # ... and the root's destination through one of its source's type
        sides = MAPS[self.coll]
        return ("s" in sides and self.sm) or ("d" in sides and self.dm)

    def check(self):
        for r, e in self.exp.items():
            if isinstance(e, tuple) and e[0] == "src":
                got, want = self.src[r].read(), e[1]
            elif isinstance(e, tuple):
                off, want = e
                got = self.dst[r].read()[off:off + len(want)]
            else:
                got, want = self.dst[r].read()[:len(e)], e
            assert np.array_equal(got[:len(want)], want), (self.coll, self.n, self.blk, "src/dst", self.sm, self.dm, "inplace", self.inplace, "rank", r)


def inplace_ok(coll):
    return coll in ("allreduce", "reduce", "reduce_scatter", "reduce_scatterv", "allgather", "allgatherv", "gather", "gatherv",
                    "scatter", "scatterv", "alltoall", "alltoallv")


def run_colls(h, team, n, seed=0):
    """every collective type, small and large, on managed / mixed buffers, in place where UCC defines it; returns the case count"""
    k = 0
    for coll in COLLS:
        for blk in (SMALL, LARGE):
            for mix, ip in [(mix, False) for mix in MIXES] + ([(("m", "m"), True)] if inplace_ok(coll) else []):
                c = Case(h, n, coll, blk, mix, ip, seed + 1000 * k, root=(k % n)).build()
                h.run(team, c.args)
                check_note(h, (coll, n, blk, mix, ip), c.mapped_managed())
                c.check()
                k += 1
    return k


def run_controls(h, team, n):
    """the decision is per buffer: a device buffer next to a managed one is still mapped where the path maps only that one, and
    device buffers alone take the direct forms (so the note checks above would see a direct form)"""
    c = Case(h, n, "allreduce", LARGE, ("d", "d"), False, 7, 0).build()
    h.run(team, c.args)
    assert "twoshot_zcopy(direct)" in h.last_launch(), h.last_launch()
    c.check()
    c = Case(h, n, "allgather", LARGE, ("d", "m"), False, 8, 0).build()
    h.run(team, c.args)
    assert "exchange_pull_zcopy" in h.last_launch(), h.last_launch()
    c.check()
    c = Case(h, n, "allreduce", LARGE, ("m", "d"), False, 9, 0).build()
    h.run(team, c.args)
    assert h.last_launch().startswith("twoshot_staged"), h.last_launch()
    c.check()


def run_persistent(h, team, n):
    """persistent requests on managed buffers, posted three times with new inputs"""
    for coll, mix in (("allreduce", ("m", "m")), ("alltoall", ("m", "d")), ("allgather", ("d", "m"))):
        c = Case(h, n, coll, LARGE, mix, False, 300, 0).build()
        for a in c.args:
            a.mask |= U.UCC_COLL_ARGS_FIELD_FLAGS
            a.flags |= U.UCC_COLL_ARGS_FLAG_PERSISTENT
        q = team.coll(c.args)
        for it in range(3):
            for r in range(n):      # new inputs into the same buffers
                data = rnd(LARGE * n, 400 + 10 * it + r)
                c.src[r].write(data if coll != "allgather" else data[:LARGE])
            exp = _expect(coll, [c.src[r].read() for r in range(n)], n)
            h.sync()
            assert q.run() == U.UCC_OK
            h.sync()
            check_note(h, (coll, "persistent", it), c.mapped_managed())
            for r in range(n):
                assert np.array_equal(c.dst[r].read(), exp[r]), (coll, "persistent", it, r)
        q.finalize()
    return 9


def _expect(coll, ins, n):
    if coll == "allreduce":
        s = sum(x.astype(np.int64) for x in ins).astype(np.int32)
        return [s] * n
    if coll == "allgather":
        return [np.concatenate(ins)] * n
    blk = len(ins[0]) // n
    return [np.concatenate([ins[p][r * blk:(r + 1) * blk] for p in range(n)]) for r in range(n)]


def run_p2p(h, team, n):
    """send / recv (two-member active-set bcast) between members 0 and n-1 in both directions, below and above the rendezvous
    threshold: a managed receive buffer makes both sides use the ring; a managed send buffer next to a device receive buffer may
    still go zero-copy"""
    k = 0
    for blk in (SMALL, LARGE):
        for mix in MIXES:
            for s_, d_ in ((0, n - 1), (n - 1, 0)):
                cnt = blk * 2
                data = rnd(cnt, 500 + k)
                sb = h.alloc(cnt, mix[0] == "m")
                sb.write(data)
                db = h.alloc(cnt, mix[1] == "m")
                db.write(np.zeros(cnt, np.int32))
                lo, hi = min(s_, d_), max(s_, d_)
                args = [None] * n
                for r, b, mt in ((s_, sb, mix[0]), (d_, db, mix[1])):
                    m = MANAGED if mt == "m" else CUDA
                    args[r] = h.args("bcast", b, None, m, m, root=s_, count_src=cnt, count_dst=0, active_set=(lo, hi - lo, 2), tag=k)
                h.run_p2p(team, {s_: args[s_], d_: args[d_]})
                note = check_note(h, ("p2p", blk, mix, s_), mix[1] == "m")
                if blk == LARGE and mix == ("m", "d"):
                    assert "rndv" in note, note
                if blk == LARGE and mix[1] == "m":
                    assert note.startswith(("p2p_send ", "p2p_recv ")), note
                assert np.array_equal(db.read(), data), ("p2p", blk, mix, s_, d_)
                k += 1
    return k


PUSH_COLLS = ("allgather", "allgatherv", "alltoall", "alltoallv")


def _tune(alg):
    return "#".join(f"{c}:cuda_managed:inf:@{alg}#{c}:cuda:inf:@{alg}" for c in PUSH_COLLS)


# the three movers of the push exchange, forced through UCC_TL_NVL_TUNE, and the launch note of their direct form
MOVERS = {"push": (dict(UCC_TL_NVL_TUNE=_tune("push"), UCC_TL_NVL_BULK="n"), "exchange_push "),
          "push_bulk": (dict(UCC_TL_NVL_TUNE=_tune("push"), UCC_TL_NVL_BULK="y", UCC_TL_NVL_BULK_THRESH="0"), "exchange_push_bulk(tma)"),
          "ce": (dict(UCC_TL_NVL_TUNE=_tune("ce")), "exchange_push_copy_engine")}


def run_push(h, team, n, mover):
    """a push mover forced for managed buffers.  A managed destination is never mapped, so the request runs the staged pull.  A
    managed source next to device destinations keeps the thread push direct (it reads the source with ordinary loads); push_bulk
    and ce, which hand the source to the TMA or copy engines, withdraw and run the staged pull as well.  Device buffers alone take
    the mover's direct form, so the checks would see it."""
    want_direct = MOVERS[mover][1]
    k = 0
    for coll in PUSH_COLLS:
        for mix in MIXES + (("d", "d"),):
            c = Case(h, n, coll, LARGE, mix, False, 700 + k, 0).build()
            h.run(team, c.args)
            note = h.last_launch()
            direct = mix == ("d", "d") or (mix == ("m", "d") and mover == "push")
            assert note.startswith(want_direct if direct else "exchange_pull_staged"), (mover, coll, mix, note)
            c.check()
            k += 1
    return k


def run_triggered(h, team, n):
    """stream-ordered posts (ucc_collective_triggered_post, one execution engine per rank on a stream of its own) on managed and
    mixed buffers: UCC_EVENT_COLLECTIVE_POST arrives on every rank, the results are exact and no managed buffer is mapped"""
    import ctypes as C
    import time
    ees = []
    for r in range(n):
        ep = U.ucc_ee_params_t()
        ep.ee_type, ep.ee_context, ep.ee_context_size = U.UCC_EE_CUDA_STREAM, h.stream(), C.sizeof(C.c_void_p)
        ee = U.handle()
        U.check(U.ucc_ee_create(team.members[r].team, C.byref(ep), C.byref(ee)), "ee_create")
        ees.append(ee)
    k = 0
    for coll, mix in (("allreduce", ("m", "m")), ("allreduce", ("m", "d")), ("alltoall", ("m", "d")), ("allgather", ("d", "m")),
                      ("reduce_scatter", ("m", "m"))):
        for blk in (SMALL, LARGE):
            c = Case(h, n, coll, blk, mix, False, 800 + k, 0).build()
            h.sync()
            reqs = []
            for r in range(n):
                q = C.POINTER(U.ucc_coll_req_t)()
                U.check(U.ucc_collective_init(C.byref(c.args[r]), C.byref(q), team.members[r].team), "init")
                ev = U.ucc_ev_t()
                ev.ev_type, ev.req = U.UCC_EVENT_COMPUTE_COMPLETE, C.cast(q, C.c_void_p)
                U.check(U.ucc_collective_triggered_post(ees[r], C.byref(ev)), "triggered_post")
                reqs.append(q)
            posted = [False] * n
            t0 = time.time()
            while not all(posted) or any(q.contents.status == U.UCC_INPROGRESS for q in reqs):
                for r in range(n):
                    U.ucc_context_progress(team.members[r].proc.ctx)
                    e = C.POINTER(U.ucc_ev_t)()
                    while U.ucc_ee_get_event(ees[r], C.byref(e)) == U.UCC_OK:
                        if e.contents.ev_type == U.UCC_EVENT_COLLECTIVE_POST:
                            posted[r] = True
                        U.ucc_ee_ack_event(ees[r], e)
                assert time.time() - t0 < 120, ("triggered post did not complete", coll, mix, blk, posted)
            h.sync()
            for q in reqs:
                assert q.contents.status == U.UCC_OK, q.contents.status
                U.ucc_collective_finalize(q)
            check_note(h, (coll, "triggered", mix, blk), c.mapped_managed())
            c.check()
            k += 1
    for ee in ees:
        U.ucc_ee_destroy(ee)
    return k


def run_self(h, team):
    """a team of one: every collective type is a local copy (the thread-copy kernel whenever a side is managed)"""
    k = 0
    for coll in COLLS:
        for blk in (SMALL, LARGE):
            for mix, ip in [(mix, False) for mix in MIXES] + ([(("m", "m"), True)] if inplace_ok(coll) else []):
                c = Case(h, 1, coll, blk, mix, ip, 900 + k, 0).build()
                h.run(team, c.args)
                c.check()
                k += 1
    return k


def run_self_large(h, team):
    """a 16 MB team-of-one copy: device buffers take cudaMemcpyAsync, a managed side the thread-copy kernel"""
    cnt = 4 << 20
    for mix, want in ((("m", "m"), "self_copy "), (("m", "d"), "self_copy "), (("d", "m"), "self_copy "), (("d", "d"), "self_copy(cudaMemcpyAsync)")):
        c = Case(h, 1, "allreduce", cnt, mix, False, 950, 0).build()
        h.run(team, c.args)
        assert h.last_launch().startswith(want), (mix, h.last_launch())
        c.check()
    return 4


def mem_map_refused(lib, ctx, dev_buf, man_buf, nbytes):
    """ucc_mem_map of a managed segment carries no tl/nvl registration; a device segment does"""
    import ctypes as C
    lib.ucc_mem_map.argtypes = [U.handle, C.c_int, C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_void_p)]
    lib.ucc_mem_map.restype = C.c_int
    lib.ucc_mem_unmap.argtypes = [C.POINTER(C.c_void_p)]
    blobs = []
    for b in (dev_buf, man_buf):
        seg = U.ucc_mem_map_t(b.ptr, nbytes)
        params = U.ucc_mem_map_params_t()
        params.segments, params.n_segments = C.pointer(seg), 1
        memh, size = C.c_void_p(), C.c_size_t()
        assert lib.ucc_mem_map(ctx, 0, C.byref(params), C.byref(size), C.byref(memh)) == U.UCC_OK
        blobs.append(C.string_at(memh.value, size.value))
        lib.ucc_mem_unmap(C.byref(memh))
    assert b"nvl" in blobs[0], "a device segment must carry a tl/nvl registration"
    assert b"nvl" not in blobs[1] and len(blobs[1]) < len(blobs[0]), "a managed segment must not be registered with tl/nvl"
