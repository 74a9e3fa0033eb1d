"""tl/nvl collectives captured into CUDA graphs (torch.cuda.graph) and replayed on one GPU.

N emulated ranks share cuda:0 in one process: every rank captures its sequence of collectives on its own stream, one rank after
the other (a captured post never waits for its peers), then all ranks replay their graphs together, several times, with new
inputs written between replays; results are exact.  Also a team of one through Communicator.graphed(), and two processes on the
one GPU, where the zero-copy tables of a graphed allreduce are CUDA IPC mappings that must survive a full mapping cache."""
import ctypes as C
import os
import subprocess
import sys

import pytest

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from ucc_b200 import capi as U  # noqa: E402
from ucc_b200.harness import UccJob, coll_args  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = U.UCC_MEMORY_TYPE_CUDA
ENV = {"UCC_TL_NVL_MAX_BLOCKS": "4", "UCC_TL_NVL_TIMEOUT": "10s", "UCC_TL_NVL_SYMMETRIC_SIZE": "8Mb", "UCC_TL_NVL_P2P_TIMEOUT": "20s"}
DT = {torch.float32: "float32", torch.bfloat16: "bfloat16", torch.int64: "int64"}


def need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)


def cargs(coll, src, dst, dt="float32", **kw):
    kw.setdefault("count_src", src.numel() if src is not None else 0)
    kw.setdefault("count_dst", dst.numel() if dst is not None else 0)
    return coll_args(coll, dt=dt, mem_type=CUDA, src_ptr=src.data_ptr() if src is not None else None,
                     dst_ptr=dst.data_ptr() if dst is not None else None, **kw)


def ints(n, dtype, gen):
    return torch.randint(0, 9, (n,), generator=gen).to(dtype).cuda()


def sequence(n, blk):
    """[(name, per-rank args, fill(gen), check())]: every collective type, in-place variants and a send / recv pair"""
    dev = "cuda"
    out = []
    for dtype in (torch.float32, torch.bfloat16, torch.int64):
        src = [torch.zeros(blk, dtype=dtype, device=dev) for _ in range(n)]
        dst = [torch.zeros(blk, dtype=dtype, device=dev) for _ in range(n)]
        out.append((f"allreduce {dtype}", [cargs("allreduce", src[r], dst[r], DT[dtype]) for r in range(n)],
                    lambda g, src=src, dtype=dtype: [s.copy_(ints(blk, dtype, g)) for s in src],
                    lambda src=src, dst=dst: all(torch.equal(d, sum(s.double() for s in src).to(d.dtype)) for d in dst)))
    counts = [blk + 3 * r for r in range(n)]
    offs = [sum(counts[:r]) for r in range(n)]
    rs_src = [torch.zeros(blk * n, device=dev) for _ in range(n)]
    rs_dst = [torch.zeros(blk, device=dev) for _ in range(n)]
    out.append(("reduce_scatter", [cargs("reduce_scatter", rs_src[r], rs_dst[r]) for r in range(n)],
                lambda g: [s.copy_(ints(blk * n, torch.float32, g)) for s in rs_src],
                lambda: all(torch.equal(rs_dst[r], sum(rs_src)[r * blk:(r + 1) * blk]) for r in range(n))))
    rsv_src = [torch.zeros(sum(counts), device=dev) for _ in range(n)]
    rsv_dst = [torch.zeros(counts[r], device=dev) for r in range(n)]
    out.append(("reduce_scatterv", [cargs("reduce_scatterv", rsv_src[r], rsv_dst[r], dst_counts=counts, dst_displs=offs) for r in range(n)],
                lambda g: [s.copy_(ints(sum(counts), torch.float32, g)) for s in rsv_src],
                lambda: all(torch.equal(rsv_dst[r], sum(rsv_src)[offs[r]:offs[r] + counts[r]]) for r in range(n))))
    ag_src = [torch.zeros(blk, device=dev) for _ in range(n)]
    ag_dst = [torch.zeros(blk * n, device=dev) for _ in range(n)]
    out.append(("allgather", [cargs("allgather", ag_src[r], ag_dst[r]) for r in range(n)],
                lambda g: [s.copy_(ints(blk, torch.float32, g)) for s in ag_src],
                lambda: all(torch.equal(d, torch.cat(ag_src)) for d in ag_dst)))
    agv_src = [torch.zeros(counts[r], device=dev) for r in range(n)]
    agv_dst = [torch.zeros(sum(counts), device=dev) for _ in range(n)]
    out.append(("allgatherv", [cargs("allgatherv", agv_src[r], agv_dst[r], dst_counts=counts, dst_displs=offs) for r in range(n)],
                lambda g: [s.copy_(ints(s.numel(), torch.float32, g)) for s in agv_src],
                lambda: all(torch.equal(d, torch.cat(agv_src)) for d in agv_dst)))
    a2_src = [torch.zeros(blk * n, device=dev) for _ in range(n)]
    a2_dst = [torch.zeros(blk * n, device=dev) for _ in range(n)]
    out.append(("alltoall", [cargs("alltoall", a2_src[r], a2_dst[r]) for r in range(n)],
                lambda g: [s.copy_(ints(blk * n, torch.float32, g)) for s in a2_src],
                lambda: all(torch.equal(a2_dst[r], torch.cat([s[r * blk:(r + 1) * blk] for s in a2_src])) for r in range(n))))
    a2i = [torch.zeros(blk * n, device=dev) for _ in range(n)]
    before = {}

    def fill_a2i(g):
        before["v"] = [ints(blk * n, torch.float32, g) for _ in range(n)]
        for r in range(n):
            a2i[r].copy_(before["v"][r])
    out.append(("alltoall in place", [cargs("alltoall", None, a2i[r], inplace=True) for r in range(n)], fill_a2i,
                lambda: all(torch.equal(a2i[r], torch.cat([b[r * blk:(r + 1) * blk] for b in before["v"]])) for r in range(n))))
    m = [[blk + (s + 2 * d) % 5 for d in range(n)] for s in range(n)]
    sd = [[sum(m[r][:d]) for d in range(n)] for r in range(n)]
    rd = [[sum(m[p][r] for p in range(q)) for q in range(n)] for r in range(n)]
    v_src = [torch.zeros(sum(m[r]), device=dev) for r in range(n)]
    v_dst = [torch.zeros(sum(m[p][r] for p in range(n)), device=dev) for r in range(n)]
    out.append(("alltoallv", [cargs("alltoallv", v_src[r], v_dst[r], src_counts=m[r], src_displs=sd[r], dst_counts=[m[p][r] for p in range(n)], dst_displs=rd[r])
                              for r in range(n)],
                lambda g: [s.copy_(ints(s.numel(), torch.float32, g)) for s in v_src],
                lambda: all(torch.equal(v_dst[r], torch.cat([v_src[p][sd[p][r]:sd[p][r] + m[p][r]] for p in range(n)])) for r in range(n))))
    b = [torch.zeros(blk, device=dev) for _ in range(n)]
    bv = {}

    def fill_b(g):
        bv["v"] = ints(blk, torch.float32, g)
        for r in range(n):
            b[r].copy_(bv["v"] if r == n - 1 else torch.zeros_like(bv["v"]))
    out.append(("bcast", [cargs("bcast", b[r], None, root=n - 1, count_dst=0) for r in range(n)], fill_b,
                lambda: all(torch.equal(x, bv["v"]) for x in b)))
    # send 0 -> 1 over a heap channel (ranks 2.. take no part)
    s0, d1 = torch.zeros(blk, device=dev), torch.zeros(blk, device=dev)
    p2p = [cargs("bcast", s0, None, root=0, count_dst=0, active_set=(0, 1, 2), tag=3), cargs("bcast", d1, None, root=0, count_dst=0, active_set=(0, 1, 2), tag=3)]
    out.append(("send / recv", p2p + [None] * (n - 2), lambda g: (s0.copy_(ints(blk, torch.float32, g)), d1.zero_()), lambda: torch.equal(s0, d1)))
    return out


@pytest.mark.parametrize("n", [2, 4])
def test_graph_replay_emulated_ranks(n):
    need_cuda()
    blk, K = 4099, 3
    with UccJob(n, env=ENV) as job:
        team = job.create_team()
        streams = [torch.cuda.Stream() for _ in range(n)]
        ees = []
        for r in range(n):
            ep = U.ucc_ee_params_t()
            ep.ee_type, ep.ee_context, ep.ee_context_size = U.UCC_EE_CUDA_STREAM, streams[r].cuda_stream, 8
            ee = U.handle()
            U.check(U.ucc_ee_create(team.members[r].team, C.byref(ep), C.byref(ee)), "ee_create")
            ees.append(ee)
        seq = sequence(n, blk)
        torch.cuda.synchronize()
        graphs, reqs = [], []
        for r in range(n):
            mine = []
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=streams[r]):
                for _, args, _, _ in seq:
                    if args[r] is None:
                        continue
                    q = C.POINTER(U.ucc_coll_req_t)()
                    U.check(U.ucc_collective_init(C.byref(args[r]), C.byref(q), team.members[r].team), "init")
                    ev = U.ucc_ev_t()
                    ev.ev_type, ev.req = U.UCC_EVENT_COMPUTE_COMPLETE, C.cast(q, C.c_void_p)
                    U.check(U.ucc_collective_triggered_post(ees[r], C.byref(ev)), "triggered_post")
                    while q.contents.status == U.UCC_INPROGRESS:   # a captured post completes at once
                        U.ucc_context_progress(job.procs[r].ctx)
                    assert q.contents.status == U.UCC_OK, q.contents.status
                    mine.append(q)
            graphs.append(g)
            reqs.append(mine)
        gen = torch.Generator().manual_seed(7)
        for it in range(K):
            for _, _, fill, _ in seq:
                fill(gen)
            torch.cuda.synchronize()
            for r in range(n):
                with torch.cuda.stream(streams[r]):
                    graphs[r].replay()
            torch.cuda.synchronize()
            for name, _, _, check in seq:
                assert check(), (n, name, it)
        for r in range(n):
            for q in reqs[r]:
                U.ucc_collective_finalize(q)
            U.ucc_ee_destroy(ees[r])
        del graphs


def test_graph_team_of_one():
    need_cuda()
    from ucc_b200 import ops
    from ucc_b200.dist import Communicator
    comm = Communicator(store=torch.distributed.HashStore(), rank=0, size=1)
    try:
        x = torch.zeros(1 << 20, device="cuda")
        ag = torch.zeros(1 << 20, device="cuda")
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with comm.graphed():
            with torch.cuda.stream(side):
                for _ in range(2):
                    ops.all_reduce(x, comm=comm)
                    ops.all_gather_into_tensor(ag, x, comm=comm)
            torch.cuda.current_stream().wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                ops.all_reduce(x, comm=comm)
                ops.all_gather_into_tensor(ag, x, comm=comm)
        for it in range(3):
            v = torch.arange(1 << 20, device="cuda", dtype=torch.float32) * (it + 1)
            x.copy_(v)
            ag.zero_()
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(x, v) and torch.equal(ag, v), it
        assert not comm.take_device_error()
        del g
    finally:
        comm.destroy()


def test_graphed_direct_two_processes_one_gpu(tmp_path):
    """two processes share cuda:0: a graphed allreduce reads the peer's buffer through CUDA IPC; after more than the mapping cache
    holds of other peer allocations went through it, the graph (and its persistent request) still replays exactly"""
    need_cuda()
    env = dict(os.environ, PYTHONPATH=ROOT, PYTORCH_NO_CUDA_MEMORY_CACHING="1", **ENV)
    worker = os.path.join(ROOT, "tests", "graph_ipc_worker.py")
    store = str(tmp_path / "store")
    procs = [subprocess.Popen([sys.executable, worker, store, str(r)], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = []
    for p in procs:
        try:
            outs.append(p.communicate(timeout=300)[0])
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and "GRAPH_IPC_OK" in o, (r, o[-4000:])
