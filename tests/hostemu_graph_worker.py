"""Worker of tests/test_nvl_graph.py: tl/nvl collectives captured into CUDA graphs and replayed, on the host-emulated plugin built by
tests/emu/build_hostemu.sh, whose CUDA runtime emulates stream capture: a capturing stream records kernels, copies and
memsets, and a graph launch replays them in order.  Every rank captures its sequence on its own stream, one rank after the other (a
captured post never waits for the peers), then all ranks replay together; every result is checked exactly against numpy."""
import ctypes as C
import faulthandler
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from hostemu_worker import BASE, NOZC, ZC, Dev, U, UccJob, ca, last_launch, rnd, rt  # noqa: E402  (loads the emulated runtime)

faulthandler.dump_traceback_later(900, exit=True)   # the whole graph scenario is one run: more time than hostemu_worker's 240 s

for _f, _a in (("cudaStreamCreate", [C.POINTER(C.c_void_p)]), ("cudaStreamBeginCapture", [C.c_void_p, C.c_int]),
               ("cudaStreamEndCapture", [C.c_void_p, C.POINTER(C.c_void_p)]), ("cudaGraphInstantiate", [C.POINTER(C.c_void_p), C.c_void_p, C.c_ulonglong]),
               ("cudaGraphLaunch", [C.c_void_p, C.c_void_p]), ("cudaGraphExecDestroy", [C.c_void_p]), ("cudaGraphDestroy", [C.c_void_p]),
               ("cudaStreamSynchronize", [C.c_void_p])):
    getattr(rt, _f).argtypes = _a


class Ranks:
    """one stream (and its execution engine) per member of `team`"""

    def __init__(self, job, team, n):
        self.job, self.team, self.n = job, team, n
        self.streams, self.ees = [], []
        for r in range(n):
            s = C.c_void_p()
            assert rt.cudaStreamCreate(C.byref(s)) == 0
            ep = U.ucc_ee_params_t()
            ep.ee_type, ep.ee_context, ep.ee_context_size = U.UCC_EE_CUDA_STREAM, s.value, C.sizeof(C.c_void_p)
            ee = U.handle()
            U.check(U.ucc_ee_create(team.members[r].team, C.byref(ep), C.byref(ee)), "ee_create")
            self.streams.append(s)
            self.ees.append(ee)

    def init(self, r, args):
        q = C.POINTER(U.ucc_coll_req_t)()
        U.check(U.ucc_collective_init(C.byref(args), C.byref(q), self.team.members[r].team), "init")
        return q

    def post(self, r, q):
        ev = U.ucc_ev_t()
        ev.ev_type, ev.req = U.UCC_EVENT_COMPUTE_COMPLETE, C.cast(q, C.c_void_p)
        U.check(U.ucc_collective_triggered_post(self.ees[r], C.byref(ev)), "triggered_post")

    def drive(self, ranks, reqs):
        t0 = time.time()
        while any(q.contents.status == U.UCC_INPROGRESS for q in reqs):
            for r in ranks:
                U.ucc_context_progress(self.job.procs[r].ctx)
                e = C.POINTER(U.ucc_ev_t)()
                while U.ucc_ee_get_event(self.ees[r], C.byref(e)) == U.UCC_OK:
                    U.ucc_ee_ack_event(self.ees[r], e)
            assert time.time() - t0 < 120, [q.contents.status for q in reqs]
        for q in reqs:
            assert q.contents.status == U.UCC_OK, q.contents.status

    def eager(self, reqs_per_rank):
        """post every rank's requests stream-ordered and wait for them"""
        for r in range(self.n):
            for q in reqs_per_rank[r]:
                self.post(r, q)
        self.drive(range(self.n), [q for rq in reqs_per_rank for q in rq])
        self.sync()

    def capture(self, r, reqs):
        """rank r's requests captured on its stream: returns the instantiated graph"""
        s = self.streams[r]
        assert rt.cudaStreamBeginCapture(s, 0) == 0
        for q in reqs:
            self.post(r, q)
        self.drive([r], reqs)                       # a captured post completes at once, without its peers
        g, ge = C.c_void_p(), C.c_void_p()
        assert rt.cudaStreamEndCapture(s, C.byref(g)) == 0, "capture invalidated"
        assert rt.cudaGraphInstantiate(C.byref(ge), g, 0) == 0
        rt.cudaGraphDestroy(g)
        return ge

    def replay(self, graphs, ranks=None):
        for r in (range(self.n) if ranks is None else ranks):
            assert rt.cudaGraphLaunch(graphs[r], self.streams[r]) == 0
        if ranks is None:
            self.sync()

    def sync(self, ranks=None):
        for r in (range(self.n) if ranks is None else ranks):
            rt.cudaStreamSynchronize(self.streams[r])

    def close(self):
        for ee in self.ees:
            U.ucc_ee_destroy(ee)


def sequence(n, blk):
    """(name, per-rank args, fill(it), check(it)) of every collective type, in-place variants included"""
    out = []
    counts = [blk + 3 * r for r in range(n)]
    offs = [int(x) for x in np.concatenate([[0], np.cumsum(counts)[:-1]])]

    def add(name, bufs, args, fill, check):
        out.append((name, bufs, args, fill, check))

    # allreduce f32 / i64, out of place and in place
    for dt in ("float32", "int64"):
        src = [Dev(blk, np.dtype(dt)) for _ in range(n)]
        dst = [Dev(blk, np.dtype(dt)) for _ in range(n)]
        add(f"allreduce {dt}", (src, dst), [ca("allreduce", src[r], dst[r], dt=dt) for r in range(n)],
            lambda it, src=src, dt=dt: [s.a.__setitem__(slice(None), rnd(blk, 100 * it + r, np.dtype(dt))) for r, s in enumerate(src)],
            lambda it, src=src, dst=dst: all(np.array_equal(d.a, sum(s.a for s in src)) for d in dst))
    ip = [Dev(blk) for _ in range(n)]
    ipv = {}

    def fill_ip(it):
        for r in range(n):
            ip[r].a[:] = rnd(blk, 200 * it + r)
        ipv["exp"] = sum(b.a.copy() for b in ip)
    add("allreduce in place", (ip,), [ca("allreduce", None, ip[r], inplace=True) for r in range(n)], fill_ip,
        lambda it: all(np.array_equal(b.a, ipv["exp"]) for b in ip))
    # reduce_scatter, reduce_scatterv
    rs_src = [Dev(blk * n) for _ in range(n)]
    rs_dst = [Dev(blk) for _ in range(n)]
    add("reduce_scatter", (rs_src, rs_dst), [ca("reduce_scatter", rs_src[r], rs_dst[r]) for r in range(n)],
        lambda it: [s.a.__setitem__(slice(None), rnd(blk * n, 300 * it + r)) for r, s in enumerate(rs_src)],
        lambda it: all(np.array_equal(rs_dst[r].a, sum(s.a for s in rs_src)[r * blk:(r + 1) * blk]) for r in range(n)))
    rsv_src = [Dev(sum(counts)) for _ in range(n)]
    rsv_dst = [Dev(counts[r]) for r in range(n)]
    add("reduce_scatterv", (rsv_src, rsv_dst), [ca("reduce_scatterv", rsv_src[r], rsv_dst[r], dst_counts=counts, dst_displs=offs) for r in range(n)],
        lambda it: [s.a.__setitem__(slice(None), rnd(sum(counts), 400 * it + r)) for r, s in enumerate(rsv_src)],
        lambda it: all(np.array_equal(rsv_dst[r].a, sum(s.a for s in rsv_src)[offs[r]:offs[r] + counts[r]]) for r in range(n)))
    # allgather, in place, allgatherv
    ag_src = [Dev(blk) for _ in range(n)]
    ag_dst = [Dev(blk * n) for _ in range(n)]
    add("allgather", (ag_src, ag_dst), [ca("allgather", ag_src[r], ag_dst[r]) for r in range(n)],
        lambda it: [s.a.__setitem__(slice(None), rnd(blk, 500 * it + r)) for r, s in enumerate(ag_src)],
        lambda it: all(np.array_equal(d.a, np.concatenate([s.a for s in ag_src])) for d in ag_dst))
    agi = [Dev(blk * n) for _ in range(n)]
    agv = {}

    def fill_agi(it):
        parts = [rnd(blk, 600 * it + r) for r in range(n)]
        agv["exp"] = np.concatenate(parts)
        for r in range(n):
            agi[r].a[:] = 0
            agi[r].a[r * blk:(r + 1) * blk] = parts[r]
    add("allgather in place", (agi,), [ca("allgather", None, agi[r], inplace=True) for r in range(n)], fill_agi,
        lambda it: all(np.array_equal(d.a, agv["exp"]) for d in agi))
    agv_src = [Dev(counts[r]) for r in range(n)]
    agv_dst = [Dev(sum(counts)) for _ in range(n)]
    add("allgatherv", (agv_src, agv_dst), [ca("allgatherv", agv_src[r], agv_dst[r], dst_counts=counts, dst_displs=offs) for r in range(n)],
        lambda it: [s.a.__setitem__(slice(None), rnd(counts[r], 700 * it + r)) for r, s in enumerate(agv_src)],
        lambda it: all(np.array_equal(d.a, np.concatenate([s.a for s in agv_src])) for d in agv_dst))
    # alltoall, in place, alltoallv
    a2_src = [Dev(blk * n) for _ in range(n)]
    a2_dst = [Dev(blk * n) for _ in range(n)]
    add("alltoall", (a2_src, a2_dst), [ca("alltoall", a2_src[r], a2_dst[r]) for r in range(n)],
        lambda it: [s.a.__setitem__(slice(None), rnd(blk * n, 800 * it + r)) for r, s in enumerate(a2_src)],
        lambda it: all(np.array_equal(a2_dst[r].a, np.concatenate([s.a[r * blk:(r + 1) * blk] for s in a2_src])) for r in range(n)))
    a2i = [Dev(blk * n) for _ in range(n)]
    a2v = {}

    def fill_a2i(it):
        a2v["before"] = [rnd(blk * n, 900 * it + r) for r in range(n)]
        for r in range(n):
            a2i[r].a[:] = a2v["before"][r]
    add("alltoall in place", (a2i,), [ca("alltoall", None, a2i[r], inplace=True) for r in range(n)], fill_a2i,
        lambda it: all(np.array_equal(a2i[r].a, np.concatenate([b[r * blk:(r + 1) * blk] for b in a2v["before"]])) for r in range(n)))
    m = np.array([[blk + (s + 2 * d) % 5 for d in range(n)] for s in range(n)])
    sd = [np.concatenate([[0], np.cumsum(m[r])[:-1]]) for r in range(n)]
    rd = [np.concatenate([[0], np.cumsum(m[:, r])[:-1]]) for r in range(n)]
    v_src = [Dev(int(m[r].sum())) for r in range(n)]
    v_dst = [Dev(int(m[:, r].sum())) for r in range(n)]
    add("alltoallv", (v_src, v_dst), [ca("alltoallv", v_src[r], v_dst[r], src_counts=m[r], src_displs=sd[r], dst_counts=m[:, r], dst_displs=rd[r]) for r in range(n)],
        lambda it: [s.a.__setitem__(slice(None), rnd(s.a.size, 1000 * it + r)) for r, s in enumerate(v_src)],
        lambda it: all(np.array_equal(v_dst[r].a, np.concatenate([v_src[p].a[sd[p][r]:sd[p][r] + m[p][r]] for p in range(n)])) for r in range(n)))
    # bcast from the last rank
    b = [Dev(blk) for _ in range(n)]
    bv = {}

    def fill_b(it):
        bv["exp"] = rnd(blk, 1100 * it)
        for r in range(n):
            b[r].a[:] = bv["exp"] if r == n - 1 else 0
    add("bcast", (b,), [ca("bcast", b[r], None, root=n - 1, count_dst=0) for r in range(n)], fill_b,
        lambda it: all(np.array_equal(x.a, bv["exp"]) for x in b))
    return out


def p2p_pair(n, blk):
    """send 0 -> 1 (and 1 -> 0 on a second tag): an eager-ring message pair; ranks 2.. take no part"""
    s0, d1, s1, d0 = Dev(blk), Dev(blk), Dev(blk), Dev(blk)
    args = {0: [ca("bcast", s0, None, root=0, count_dst=0, active_set=(0, 1, 2), tag=5), ca("bcast", d0, None, root=1, count_dst=0, active_set=(0, 1, 2), tag=6)],
            1: [ca("bcast", d1, None, root=0, count_dst=0, active_set=(0, 1, 2), tag=5), ca("bcast", s1, None, root=1, count_dst=0, active_set=(0, 1, 2), tag=6)]}

    def fill(it):
        s0.a[:] = rnd(blk, 1200 * it)
        s1.a[:] = rnd(blk, 1300 * it)
        d0.a[:] = 0
        d1.a[:] = 0
    return args, fill, lambda it: np.array_equal(d1.a, s0.a) and np.array_equal(d0.a, s1.a)


def captured_sequences(label, env, sizes=(2, 3, 4), blk=1003):
    with UccJob(4, env=dict(BASE, **env)) as j:
        for n in sizes:
            team = j.create_team(range(n))
            R = Ranks(j, team, n)
            seq = sequence(n, blk)
            p2p_args, p2p_fill, p2p_check = p2p_pair(n, blk)
            reqs = [[R.init(r, c[2][r]) for c in seq] + [R.init(r, a) for a in p2p_args.get(r, [])] for r in range(n)]
            graphs = [R.capture(r, reqs[r]) for r in range(n)]
            for it in range(3):                      # new inputs between replays
                for c in seq:
                    c[3](it)
                p2p_fill(it)
                R.replay(graphs)
                for c in seq:
                    assert c[4](it), (label, n, c[0], it)
                assert p2p_check(it), (label, n, "p2p", it)
            for r in range(n):
                rt.cudaGraphExecDestroy(graphs[r])
                for q in reqs[r]:
                    U.ucc_collective_finalize(q)
            R.close()
    print(f"  captured collectives [{label}] replayed exactly", flush=True)


def persistent_direct():
    """a persistent request whose first (eager) post resolved the zero-copy tables keeps the direct form in the graph"""
    tune = "allreduce:cuda:inf:@twoshot#reduce_scatter:cuda:inf:@twoshot"
    with UccJob(4, env=dict(BASE, UCC_TL_NVL_TUNE=tune, UCC_TL_NVL_ALLREDUCE_ONESHOT_THRESH="0", **ZC)) as j:
        for n in (2, 3, 4):
            team = j.create_team(range(n))
            R = Ranks(j, team, n)
            blk = 4096
            cases = []
            src, dst = [Dev(blk) for _ in range(n)], [Dev(blk) for _ in range(n)]
            cases.append(("allreduce", "twoshot_zcopy(direct)", [ca("allreduce", src[r], dst[r], persistent=True) for r in range(n)],
                          lambda it, src=src: [s.a.__setitem__(slice(None), rnd(blk, 10 * it + r)) for r, s in enumerate(src)],
                          lambda it, src=src, dst=dst: all(np.array_equal(d.a, sum(s.a for s in src)) for d in dst)))
            rs, rd_ = [Dev(blk * n) for _ in range(n)], [Dev(blk) for _ in range(n)]
            cases.append(("reduce_scatter", "twoshot_zcopy(direct)", [ca("reduce_scatter", rs[r], rd_[r], persistent=True) for r in range(n)],
                          lambda it: [s.a.__setitem__(slice(None), rnd(blk * n, 20 * it + r)) for r, s in enumerate(rs)],
                          lambda it: all(np.array_equal(rd_[r].a, sum(s.a for s in rs)[r * blk:(r + 1) * blk]) for r in range(n))))
            a2 = [Dev(blk * n) for _ in range(n)]
            before = {}

            def fill_a2(it):
                before["v"] = [rnd(blk * n, 30 * it + r) for r in range(n)]
                for r in range(n):
                    a2[r].a[:] = before["v"][r]
            cases.append(("alltoall in place", "exchange_swap", [ca("alltoall", None, a2[r], inplace=True, persistent=True) for r in range(n)], fill_a2,
                          lambda it: all(np.array_equal(a2[r].a, np.concatenate([b[r * blk:(r + 1) * blk] for b in before["v"]])) for r in range(n))))
            for name, note, args, fill, check in cases:
                reqs = [[R.init(r, args[r])] for r in range(n)]
                fill(0)
                R.eager(reqs)                        # resolves and caches the members' buffers
                assert check(0), (name, n, "eager")
                graphs = []
                for r in range(n):
                    graphs.append(R.capture(r, reqs[r]))
                    assert note in last_launch(), (name, n, r, last_launch())
                for it in range(1, 4):
                    fill(it)
                    R.replay(graphs)
                    assert check(it), (name, n, it)
                for r in range(n):
                    rt.cudaGraphExecDestroy(graphs[r])
                    U.ucc_collective_finalize(reqs[r][0])
            R.close()
    print("  persistent direct forms in graphs ok", flush=True)


def eager_replay_eager():
    """eager -> replay -> eager, all on one stream per rank"""
    n, blk = 3, 5000
    for env in (NOZC, ZC):
        with UccJob(n, env=dict(BASE, **env)) as j:
            team = j.create_team(range(n))
            R = Ranks(j, team, n)
            src, dst = [Dev(blk) for _ in range(n)], [Dev(blk) for _ in range(n)]
            cap = [R.init(r, ca("allreduce", src[r], dst[r])) for r in range(n)]
            graphs = [R.capture(r, [cap[r]]) for r in range(n)]
            for it in range(3):
                for r in range(n):
                    src[r].a[:] = rnd(blk, 40 * it + r)
                eager = [[R.init(r, ca("allreduce", src[r], dst[r]))] for r in range(n)]
                R.eager(eager)
                for q in eager:
                    U.ucc_collective_finalize(q[0])
                assert all(np.array_equal(d.a, sum(s.a for s in src)) for d in dst), ("eager", it)
                for r in range(n):
                    src[r].a[:] = rnd(blk, 50 * it + r)
                    dst[r].a[:] = 0
                R.replay(graphs)
                assert all(np.array_equal(d.a, sum(s.a for s in src)) for d in dst), ("replay", it)
            for r in range(n):
                rt.cudaGraphExecDestroy(graphs[r])
                U.ucc_collective_finalize(cap[r])
            R.close()
    print("  eager -> replay -> eager ok", flush=True)


def replay_device_error():
    """a replay that one member never joins: the others' kernels give up after TL_NVL_TIMEOUT, and the team's device-error
    query reports it once"""
    n, blk = 3, 1000
    with UccJob(n, env=dict(BASE, UCC_TL_NVL_TIMEOUT="2s", **NOZC)) as j:
        team = j.create_team(range(n))
        R = Ranks(j, team, n)
        err = C.CDLL(os.path.join(os.environ["UCC_MODULE_DIR"], "libucc_tl_nvl.so")).ucc_tl_nvl_take_device_error
        err.restype, err.argtypes = C.c_int, [U.handle]
        src, dst = [Dev(blk, fill=1.0) for _ in range(n)], [Dev(blk, fill=0) for _ in range(n)]
        reqs = [R.init(r, ca("allreduce", src[r], dst[r])) for r in range(n)]
        graphs = [R.capture(r, [reqs[r]]) for r in range(n)]
        R.replay(graphs)
        assert all(np.all(d.a == n) for d in dst)
        assert err(team.members[0].team) == 0
        R.replay(graphs, ranks=(0, 1))               # rank 2 stays away
        R.sync((0, 1))
        assert err(team.members[0].team) == 1 and err(team.members[1].team) == 1
        assert err(team.members[0].team) == 0, "the query clears the latch"
        for r in range(n):
            rt.cudaGraphExecDestroy(graphs[r])
            U.ucc_collective_finalize(reqs[r])
        R.close()
    print("  device error of a replay reported ok", flush=True)


def graphs():
    captured_sequences("default", NOZC)
    captured_sequences("twoshot staged, zero-copy board", dict(ZC, UCC_TL_NVL_TUNE="allreduce:cuda:inf:@twoshot#reduce_scatter:cuda:inf:@twoshot#reduce_scatterv:cuda:inf:@twoshot",
                                                               UCC_TL_NVL_ALLREDUCE_ONESHOT_THRESH="0"))
    captured_sequences("ring", dict(NOZC, UCC_TL_NVL_TUNE="allreduce:cuda:inf:@ring#allgather:cuda:inf:@ring#allgatherv:cuda:inf:@ring#reduce_scatter:cuda:inf:@ring#reduce_scatterv:cuda:inf:@ring",
                                    UCC_TL_NVL_ALLREDUCE_ONESHOT_THRESH="0"))
    captured_sequences("push / swap, zero-copy board", dict(ZC, UCC_TL_NVL_TUNE="allgather:cuda:inf:@push#alltoall:cuda:inf:@push#alltoallv:cuda:inf:@push"))
    persistent_direct()
    eager_replay_eager()
    replay_device_error()


SCENARIOS = {"graphs": graphs}

if __name__ == "__main__":
    SCENARIOS[sys.argv[1]]()
    print("HOSTEMU_WORKER_OK", flush=True)
