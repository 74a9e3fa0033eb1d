"""In-place alltoall / alltoallv on tl/nvl on a real GPU (N emulated ranks on cuda:0, as in tests/test_nvl_gpu.py): the pairwise swap
kernel when the members' buffers resolve, the heap-staged pull when they cannot (UCC_TL_NVL_ZCOPY=n).  Every result is compared with
torch.equal against the blocks gathered on the host."""
import ctypes as C
import os

import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from test_nvl_gpu import ENV, NOZC, ZC, U, UccJob, cargs, gen, need_cuda, run  # noqa: E402

# the staged fallback stages the whole buffer in the heap: room for the 64 MB buffers below
ENV_A2A = dict(ENV, UCC_TL_NVL_SYMMETRIC_SIZE="72Mb")
KERNEL = {"swap": "exchange_swap", "staged": "exchange_pull_staged_inplace"}


def last_launch():
    info = C.CDLL(os.path.join(os.path.dirname(U.LIB_PATH), "ucc", "libucc_tl_nvl.so")).ucc_tl_nvl_last_launch_info
    info.restype = C.c_char_p
    return info().decode()


def a2a_expect(bufs, n, blk):
    return [torch.cat([bufs[p][r * blk:(r + 1) * blk] for p in range(n)]) for r in range(n)]


def a2av_layout(n, blk):
    """symmetric skewed counts with odd values (rank 0 is hot, pairs whose ranks add up to 3 exchange nothing), unaligned gaps"""
    cnt = [[0 if (r != p and r + p == 3) else (blk + 2 * max(r, p) + 1 if 0 in (r, p) else blk // 7 + r * p + 1) for p in range(n)] for r in range(n)]
    dsp, size = [], 0
    for r in range(n):
        o, row = 0, []
        for p in range(n):
            o += (r + p) % 3
            row.append(o)
            o += cnt[r][p]
        dsp.append(row)
        size = max(size, o + 1)
    return cnt, dsp, size


def a2av_expect(bufs, cnt, dsp, n):
    out = [b.clone() for b in bufs]
    for r in range(n):
        for p in range(n):
            if p != r:
                out[r][dsp[r][p]:dsp[r][p] + cnt[r][p]] = bufs[p][dsp[p][r]:dsp[p][r] + cnt[p][r]]
    return out


def post_a2a(team, bufs, dt, **kw):
    torch.cuda.synchronize()   # the inputs were filled on torch's stream; the team streams do not wait for it
    run(team, [cargs("alltoall", None, bufs[r], dt, inplace=True, **kw) for r in range(len(bufs))])


@pytest.fixture(scope="module", params=["swap", "staged"])
def a2a_job(request):
    need_cuda()
    j = UccJob(8, env=dict(ENV_A2A, **(ZC if request.param == "swap" else NOZC)))
    teams = {n: j.create_team(range(n)) for n in (2, 3, 4, 8)}
    yield request.param, teams
    j.cleanup()


@pytest.mark.parametrize("n", [2, 3, 4, 8])
@pytest.mark.parametrize("dt", ["float32", "bfloat16"])
def test_inplace_alltoall(a2a_job, n, dt):
    path, teams = a2a_job
    esz = 4 if dt == "float32" else 2
    for blk in (1, 1237, 65536, (64 << 20) // esz // n + 3):   # the last one: a buffer of just over 64 MB per rank
        bufs = [gen(dt, blk * n, 10 * r + blk % 1000) for r in range(n)]
        exp = a2a_expect([b.clone() for b in bufs], n, blk)
        post_a2a(teams[n], bufs, dt)
        assert KERNEL[path] in last_launch(), (last_launch(), n, blk)
        for r in range(n):
            assert torch.equal(bufs[r], exp[r]), (path, dt, n, blk, r)


@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_inplace_alltoallv_skewed(a2a_job, n):
    path, teams = a2a_job
    for blk in (5, 300001):
        cnt, dsp, size = a2av_layout(n, blk)
        bufs = [gen("float32", size, 7 * r + blk) for r in range(n)]
        exp = a2av_expect([b.clone() for b in bufs], cnt, dsp, n)
        torch.cuda.synchronize()
        run(teams[n], [cargs("alltoallv", None, bufs[r], "float32", inplace=True, dst_counts=cnt[r], dst_displs=dsp[r]) for r in range(n)])
        assert KERNEL[path] in last_launch(), (last_launch(), n, blk)
        for r in range(n):
            assert torch.equal(bufs[r], exp[r]), (path, n, blk, r)


def test_inplace_alltoall_persistent(a2a_job):
    """one persistent in-place request posted three times with new contents"""
    path, teams = a2a_job
    n, blk = 4, 100003
    bufs = [torch.zeros(blk * n, device="cuda") for _ in range(n)]
    req = teams[n].coll([cargs("alltoall", None, bufs[r], "float32", inplace=True, persistent=True) for r in range(n)])
    for it in range(3):
        for r in range(n):
            bufs[r].copy_(gen("float32", blk * n, 100 * it + r))
        exp = a2a_expect([b.clone() for b in bufs], n, blk)
        torch.cuda.synchronize()
        assert req.run() == U.UCC_OK
        torch.cuda.synchronize()
        assert KERNEL[path] in last_launch(), last_launch()
        for r in range(n):
            assert torch.equal(bufs[r], exp[r]), (path, it, r)
    req.finalize()


def test_inplace_alltoall_stream_triggered(a2a_job):
    """stream-ordered post (ucc_collective_triggered_post): the collective runs behind the copy that fills the buffer on the user's
    stream, and a copy queued after UCC_EVENT_COLLECTIVE_POST sees the result"""
    import time
    path, teams = a2a_job
    n, blk = 4, 200001
    team = teams[n]
    streams = [torch.cuda.Stream() for _ in range(n)]
    ees = []
    for r in range(n):
        ep = U.ucc_ee_params_t()
        ep.ee_type, ep.ee_context, ep.ee_context_size = U.UCC_EE_CUDA_STREAM, streams[r].cuda_stream, C.sizeof(C.c_void_p)
        ee = U.handle()
        U.check(U.ucc_ee_create(team.members[r].team, C.byref(ep), C.byref(ee)), "ee_create")
        ees.append(ee)
    stage = [gen("float32", blk * n, 40 + r) for r in range(n)]
    bufs = [torch.zeros(blk * n, device="cuda") for _ in range(n)]
    after = [torch.zeros(blk * n, device="cuda") for _ in range(n)]
    torch.cuda.synchronize()
    reqs = []
    for r in range(n):
        with torch.cuda.stream(streams[r]):
            bufs[r].copy_(stage[r], non_blocking=True)
        a = cargs("alltoall", None, bufs[r], "float32", inplace=True)
        q = C.POINTER(U.ucc_coll_req_t)()
        U.check(U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team), "init")
        ev = U.ucc_ev_t()
        ev.ev_type, ev.req = U.UCC_EVENT_COMPUTE_COMPLETE, C.cast(q, C.c_void_p)
        U.check(U.ucc_collective_triggered_post(ees[r], C.byref(ev)), "triggered_post")
        reqs.append((a, q))
    posted = [False] * n
    t0 = time.perf_counter()
    while not all(posted) or any(q.contents.status == U.UCC_INPROGRESS for _, q in reqs):
        team.job.progress()
        for r in range(n):
            e = C.POINTER(U.ucc_ev_t)()
            while U.ucc_ee_get_event(ees[r], C.byref(e)) == U.UCC_OK:
                if e.contents.ev_type == U.UCC_EVENT_COLLECTIVE_POST:
                    posted[r] = True
                    with torch.cuda.stream(streams[r]):
                        after[r].copy_(bufs[r], non_blocking=True)
                U.ucc_ee_ack_event(ees[r], e)
        assert time.perf_counter() - t0 < 60, posted
    torch.cuda.synchronize()
    exp = a2a_expect(stage, n, blk)
    for r in range(n):
        assert reqs[r][1].contents.status == U.UCC_OK
        U.ucc_collective_finalize(reqs[r][1])
        assert torch.equal(bufs[r], exp[r]) and torch.equal(after[r], exp[r]), (path, r)
    assert KERNEL[path] in last_launch(), last_launch()
    for ee in ees:
        U.ucc_ee_destroy(ee)


def test_inplace_alltoall_tune_swap():
    """UCC_TL_NVL_TUNE=alltoall:@swap selects the swap path for in-place requests; an out-of-place alltoall on the same team, which
    swap turns down, still runs (on the pull kernel)"""
    need_cuda()
    n, blk = 4, 300007
    with UccJob(n, env=dict(ENV_A2A, UCC_TL_NVL_TUNE="alltoall:@swap#alltoallv:@swap", UCC_TL_NVL_ZCOPY="y")) as j:
        team = j.create_team()
        bufs = [gen("bfloat16", blk * n, 60 + r) for r in range(n)]
        exp = a2a_expect([b.clone() for b in bufs], n, blk)
        post_a2a(team, bufs, "bfloat16")
        assert "exchange_swap" in last_launch(), last_launch()
        for r in range(n):
            assert torch.equal(bufs[r], exp[r]), r
        src = [gen("float32", blk * n, 70 + r) for r in range(n)]
        dst = [torch.zeros(blk * n, device="cuda") for _ in range(n)]
        torch.cuda.synchronize()
        run(team, [cargs("alltoall", src[r], dst[r], "float32") for r in range(n)])
        assert "exchange_swap" not in last_launch(), last_launch()
        for r in range(n):
            assert torch.equal(dst[r], torch.cat([src[p][r * blk:(r + 1) * blk] for p in range(n)])), r
