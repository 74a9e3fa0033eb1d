"""tl/nvl kernels on a real GPU.  N emulated ranks share cuda:0 (one process, one stream per
rank), so every kernel protocol (flags, epochs, slices, rounds) is exercised without needing
several GPUs; the multi-GPU / multi-process path is covered by tests/test_dist_gpu.py.
Numerics are compared against a plain PyTorch fp32/fp64 reference of the same op."""
import os

import numpy as np
import pytest

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from ucc_b200 import capi as U  # noqa: E402
from ucc_b200.harness import UccJob, coll_args  # noqa: E402

CUDA = U.UCC_MEMORY_TYPE_CUDA
TDT = {"float32": torch.float32, "float64": torch.float64, "float16": torch.float16, "bfloat16": torch.bfloat16,
       "int32": torch.int32, "int64": torch.int64, "int8": torch.int8, "uint8": torch.uint8, "int16": torch.int16}
# zero-copy kernels (members' user buffers used in place) forced for every size / never used
ZC = {"UCC_TL_NVL_ZCOPY": "y", "UCC_TL_NVL_ZCOPY_THRESH": "0"}
NOZC = {"UCC_TL_NVL_ZCOPY": "n"}
ENV = {"UCC_TL_NVL_MAX_BLOCKS": "4", "UCC_TL_NVL_TIMEOUT": "5s", "UCC_TL_NVL_SYMMETRIC_SIZE": "8Mb",
       "UCC_TL_NVL_P2P_TIMEOUT": "20s"}   # (send / recv kernels wait without a deadline by default: keep a hang from eating the whole run)


def need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)


def cargs(coll, src, dst, dt, **kw):
    kw.setdefault("count_src", src.numel() if src is not None else 0)
    kw.setdefault("count_dst", dst.numel() if dst is not None else 0)
    return coll_args(coll, dt=dt, mem_type=CUDA, src_ptr=src.data_ptr() if src is not None else None,
                     dst_ptr=dst.data_ptr() if dst is not None else None, **kw)


def run(team, args):
    req = team.coll(args)
    st = req.run()
    req.finalize()
    assert st == U.UCC_OK, U.status_str(st)
    torch.cuda.synchronize()


def gen(dt, n, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    if TDT[dt].is_floating_point:
        return (torch.rand(n, generator=g) + 0.5).to(TDT[dt]).cuda()
    return torch.randint(1, 5, (n,), generator=g).to(TDT[dt]).cuda()


def ref_reduce(op, xs):
    a = torch.stack([x.double() if x.dtype.is_floating_point else x.long() for x in xs])
    if op == "sum":
        return a.sum(0)
    if op == "avg":   # integers: truncated sum / N
        return a.sum(0) / len(xs) if a.dtype.is_floating_point else torch.div(a.sum(0), len(xs), rounding_mode="trunc")
    if op == "prod":
        return a.prod(0)
    if op == "max":
        return a.max(0).values
    if op == "min":
        return a.min(0).values
    raise ValueError(op)


def assert_close(got, exp, dt):
    if dt in ("bfloat16", "float16"):
        assert torch.allclose(got.double(), exp.double(), rtol=2e-2, atol=2e-2)
    elif TDT[dt].is_floating_point:
        assert torch.allclose(got.double(), exp.double(), rtol=1e-5, atol=1e-6)
    else:
        assert torch.equal(got.long(), exp.long())


@pytest.fixture(scope="module", params=["oneshot", "twoshot", "twoshot-zcopy"])
def alg_job(request):
    need_cuda()
    env = dict(ENV)
    env["UCC_TL_NVL_TUNE"] = f"allreduce:cuda:inf:@{request.param.split('-')[0]}"
    env.update(ZC if request.param.endswith("zcopy") else NOZC)
    job = UccJob(8, env=env)
    teams = {n: job.create_team(range(n)) for n in (2, 3, 4, 8)}
    yield request.param, teams
    job.cleanup()


@pytest.mark.parametrize("n", [2, 3, 4, 8])
@pytest.mark.parametrize("count", [1, 7, 1024, 4097, 16384])
def test_allreduce_f32(alg_job, n, count):
    alg, teams = alg_job
    team = teams[n]
    src = [gen("float32", count, r) for r in range(n)]
    dst = [torch.zeros(count, device="cuda") for _ in range(n)]
    run(team, [cargs("allreduce", src[r], dst[r], "float32") for r in range(n)])
    exp = ref_reduce("sum", src)
    for r in range(n):
        assert_close(dst[r], exp, "float32")


@pytest.mark.parametrize("dt,op", [("float32", "avg"), ("float64", "sum"), ("float16", "sum"), ("bfloat16", "sum"), ("bfloat16", "max"),
                                   ("int32", "sum"), ("int64", "max"), ("int8", "min"), ("uint8", "sum"), ("int16", "prod"), ("int32", "avg"), ("int64", "avg")])
def test_allreduce_dt_op(alg_job, dt, op):
    alg, teams = alg_job
    n, count = 4, 1000
    team = teams[n]
    src = [gen(dt, count, r + 11) for r in range(n)]
    dst = [torch.zeros(count, dtype=TDT[dt], device="cuda") for _ in range(n)]
    run(team, [cargs("allreduce", src[r], dst[r], dt, op=op) for r in range(n)])
    exp = ref_reduce(op, src)
    for r in range(n):
        assert_close(dst[r], exp, dt)


def test_allreduce_inplace_persistent_unaligned(alg_job):
    alg, teams = alg_job
    n, count = 4, 3001
    team = teams[n]
    base = [torch.zeros(count + 1, device="cuda") for _ in range(n)]
    bufs = [b[1:] for b in base]  # 4-byte aligned only
    req = team.coll([cargs("allreduce", None, bufs[r], "float32", inplace=True, persistent=True) for r in range(n)])
    for it in range(3):
        src = [gen("float32", count, 10 * it + r) for r in range(n)]
        for r in range(n):
            bufs[r].copy_(src[r])
        torch.cuda.synchronize()
        assert req.run() == U.UCC_OK
        torch.cuda.synchronize()
        exp = ref_reduce("sum", src)
        for r in range(n):
            assert_close(bufs[r], exp, "float32")
    req.finalize()


@pytest.fixture(scope="module", params=["staged", "zcopy"])
def job(request):
    need_cuda()
    j = UccJob(8, env=dict(ENV, **(ZC if request.param == "zcopy" else NOZC)))
    teams = {n: j.create_team(range(n)) for n in (2, 3, 4, 8)}
    yield teams
    j.cleanup()


@pytest.mark.parametrize("n", [2, 4, 8])
def test_allreduce_multi_round(job, n):
    # 8 MB heap / n ranks => several rounds inside one kernel
    team = job[n]
    count = 5 * 1024 * 1024 + 13
    src = [gen("float32", count, r) for r in range(n)]
    dst = [torch.zeros(count, device="cuda") for _ in range(n)]
    run(team, [cargs("allreduce", src[r], dst[r], "float32") for r in range(n)])
    exp = ref_reduce("sum", src)
    for r in range(n):
        assert_close(dst[r], exp, "float32")


@pytest.mark.parametrize("n", [2, 4])
def test_allreduce_multi_round_short_last_round(job, n):
    """several heap rounds with a SHORTER last round, repeated: the per-block vector ranges must not move between rounds
    (cross-block race found in the host emulation, tests/emu/nvl_emu.cpp `soak`; blocks of one rank are not synchronised)"""
    team = job[n]
    cap = (8 * 1024 * 1024 // n // 16) * 4          # elements of one slice per round (8 MB heap, float32)
    count = n * (2 * cap + cap // 5 + 3)            # two full rounds + a short, ragged third one
    for it in range(4):
        src = [gen("float32", count, 10 * it + r) for r in range(n)]
        dst = [torch.zeros(count, device="cuda") for _ in range(n)]
        run(team, [cargs("allreduce", src[r], dst[r], "float32") for r in range(n)])
        exp = ref_reduce("sum", src)
        for r in range(n):
            assert_close(dst[r], exp, "float32")


@pytest.mark.parametrize("n", [2, 3, 8])
@pytest.mark.parametrize("inplace", [False, True])
def test_reduce_scatter(job, n, inplace):
    team = job[n]
    blk = 1237
    src = [gen("float32", blk * n, r) for r in range(n)]
    exp = ref_reduce("sum", src)
    if inplace:
        bufs = [s.clone() for s in src]
        run(team, [cargs("reduce_scatter", None, bufs[r], "float32", inplace=True) for r in range(n)])
        for r in range(n):
            assert_close(bufs[r][r * blk:(r + 1) * blk], exp[r * blk:(r + 1) * blk], "float32")
    else:
        dst = [torch.zeros(blk, device="cuda") for _ in range(n)]
        run(team, [cargs("reduce_scatter", src[r], dst[r], "float32") for r in range(n)])
        for r in range(n):
            assert_close(dst[r], exp[r * blk:(r + 1) * blk], "float32")


@pytest.mark.parametrize("n", [2, 3, 8])
def test_reduce_scatter_oneshot_mixed_with_allreduce(n):
    """one-shot reduce_scatter(v) (push every block to its owner's latency slot, one flag exchange) interleaved with one-shot allreduces
    of different grid sizes: both share the slot parity / team-wide sequence (kernels/nvl_oneshot_rs.cuh)"""
    need_cuda()
    env = dict(ENV, UCC_TL_NVL_TUNE="reduce_scatter:cuda:0-inf:@oneshot#reduce_scatterv:cuda:0-inf:@oneshot", **NOZC)
    with UccJob(n, env=env) as j:
        team = j.create_team()
        for it, blk in enumerate((5, 1237, 40001, 3, 20000)):
            for dt, op in (("float32", "sum"), ("bfloat16", "max"), ("int32", "avg")):
                src = [gen(dt, blk * n, 10 * it + r) for r in range(n)]
                dst = [torch.zeros(blk, dtype=TDT[dt], device="cuda") for _ in range(n)]
                run(team, [cargs("reduce_scatter", src[r], dst[r], dt, op=op) for r in range(n)])
                exp = ref_reduce(op, src)
                for r in range(n):
                    assert_close(dst[r], exp[r * blk:(r + 1) * blk], dt)
            # an allreduce with another grid size in between (the bug the team-wide sequence fixed: per-block parities diverged)
            cnt = 4096 * (it + 1) + 7
            a = [gen("float32", cnt, 77 + r) for r in range(n)]
            b = [torch.zeros(cnt, device="cuda") for _ in range(n)]
            run(team, [cargs("allreduce", a[r], b[r], "float32") for r in range(n)])
            for r in range(n):
                assert_close(b[r], ref_reduce("sum", a), "float32")
        counts = [100 + 33 * r for r in range(n)]
        offs = np.concatenate([[0], np.cumsum(counts)[:-1]])
        src = [gen("float32", sum(counts), r) for r in range(n)]
        dst = [torch.zeros(counts[r], device="cuda") for r in range(n)]
        run(team, [cargs("reduce_scatterv", src[r], dst[r], "float32", dst_counts=counts, dst_displs=offs) for r in range(n)])
        exp = ref_reduce("sum", src)
        for r in range(n):
            assert_close(dst[r], exp[offs[r]:offs[r] + counts[r]], "float32")


@pytest.mark.parametrize("n", [2, 4])
def test_reduce_scatterv(job, n):
    team = job[n]
    counts = [100 + 33 * r for r in range(n)]
    offs = np.concatenate([[0], np.cumsum(counts)[:-1]])
    src = [gen("int32", sum(counts), r) for r in range(n)]
    dst = [torch.zeros(counts[r], dtype=torch.int32, device="cuda") for r in range(n)]
    run(team, [cargs("reduce_scatterv", src[r], dst[r], "int32", dst_counts=counts, dst_displs=offs) for r in range(n)])
    exp = ref_reduce("sum", src)
    for r in range(n):
        assert_close(dst[r], exp[offs[r]:offs[r] + counts[r]], "int32")


@pytest.mark.parametrize("n", [2, 4, 8])
def test_reduce(job, n):
    team = job[n]
    count = 5000
    for root in {0, n - 1}:
        src = [gen("float32", count, r) for r in range(n)]
        dst = torch.zeros(count, device="cuda")
        run(team, [cargs("reduce", src[r], dst if r == root else None, "float32", root=root, count_dst=count) for r in range(n)])
        assert_close(dst, ref_reduce("sum", src), "float32")


@pytest.mark.parametrize("n", [2, 3, 8])
@pytest.mark.parametrize("count", [1, 1000, 100001])
def test_allgather(job, n, count):
    team = job[n]
    src = [gen("int32", count, r) for r in range(n)]
    dst = [torch.zeros(count * n, dtype=torch.int32, device="cuda") for _ in range(n)]
    run(team, [cargs("allgather", src[r], dst[r], "int32") for r in range(n)])
    exp = torch.cat(src)
    for r in range(n):
        assert torch.equal(dst[r], exp)


@pytest.mark.parametrize("n", [2, 4])
def test_allgatherv(job, n):
    team = job[n]
    counts = [5 + 1000 * r for r in range(n)]
    displs = np.concatenate([[0], np.cumsum(counts)[:-1]])
    src = [gen("float32", counts[r], r) for r in range(n)]
    dst = [torch.zeros(sum(counts), device="cuda") for _ in range(n)]
    run(team, [cargs("allgatherv", src[r], dst[r], "float32", dst_counts=counts, dst_displs=displs) for r in range(n)])
    for r in range(n):
        assert torch.equal(dst[r], torch.cat(src))


@pytest.mark.parametrize("n", [2, 3, 8])
@pytest.mark.parametrize("count", [1, 333, 20000])
def test_alltoall(job, n, count):
    team = job[n]
    src = [gen("float32", count * n, r) for r in range(n)]
    dst = [torch.zeros(count * n, device="cuda") for _ in range(n)]
    run(team, [cargs("alltoall", src[r], dst[r], "float32") for r in range(n)])
    for r in range(n):
        exp = torch.cat([src[p][r * count:(r + 1) * count] for p in range(n)])
        assert torch.equal(dst[r], exp)


@pytest.mark.parametrize("n", [2, 4, 8])
def test_alltoallv_moe_skew(job, n):
    team = job[n]
    rng = np.random.default_rng(n)
    # token-routing style skew: a few hot experts
    m = rng.integers(0, 50, size=(n, n))
    m[:, 0] += 400
    sc = [list(m[r]) for r in range(n)]
    rc = [list(m[:, r]) for r in range(n)]
    sd = [np.concatenate([[0], np.cumsum(c)[:-1]]) for c in sc]
    rd = [np.concatenate([[0], np.cumsum(c)[:-1]]) for c in rc]
    src = [gen("bfloat16", int(sum(sc[r])), r) for r in range(n)]
    dst = [torch.zeros(int(sum(rc[r])), dtype=torch.bfloat16, device="cuda") for r in range(n)]
    run(team, [cargs("alltoallv", src[r], dst[r], "bfloat16", src_counts=sc[r], src_displs=sd[r], dst_counts=rc[r], dst_displs=rd[r]) for r in range(n)])
    for r in range(n):
        exp = torch.cat([src[p][sd[p][r]:sd[p][r] + sc[p][r]] for p in range(n)])
        assert torch.equal(dst[r], exp)


@pytest.mark.parametrize("n", [2, 4, 8])
def test_bcast_gather_scatter_barrier(job, n):
    team = job[n]
    count = 7777
    for root in {0, n - 1}:
        bufs = [gen("float32", count, r) if r == root else torch.zeros(count, device="cuda") for r in range(n)]
        exp = bufs[root].clone()
        run(team, [cargs("bcast", bufs[r], None, "float32", root=root) for r in range(n)])
        for r in range(n):
            assert torch.equal(bufs[r], exp)
        src = [gen("int32", 100, r) for r in range(n)]
        dst = torch.zeros(100 * n, dtype=torch.int32, device="cuda")
        run(team, [cargs("gather", src[r], dst if r == root else None, "int32", root=root, count_dst=100 * n) for r in range(n)])
        assert torch.equal(dst, torch.cat(src))
        big = gen("int32", 100 * n, 5)
        out = [torch.zeros(100, dtype=torch.int32, device="cuda") for _ in range(n)]
        run(team, [cargs("scatter", big if r == root else None, out[r], "int32", root=root, count_src=100 * n) for r in range(n)])
        for r in range(n):
            assert torch.equal(out[r], big[r * 100:(r + 1) * 100])
    run(team, [coll_args("barrier") for _ in range(n)])


# ---------------------------------------------------------------- zero-copy push exchange: thread copies, TMA bulk copies, copy engines
@pytest.mark.parametrize("mover", ["push", "push_bulk", "ce"])
@pytest.mark.parametrize("n", [2, 4, 8])
def test_push_exchange_movers(mover, n):
    """allgather(v) / alltoall / skewed alltoallv through the members' mapped destinations.  push_bulk: the TMA engine moves the
    blocks (cp.async.bulk through shared memory, one elected thread per CTA; unaligned blocks fall back to thread copies inside
    the same kernel); ce: cudaMemcpyAsync between two barrier kernels (reference ALLTOALL_USE_COPY_ENGINE)."""
    need_cuda()
    alg = "ce" if mover == "ce" else "push"
    env = dict(ENV, UCC_TL_NVL_TUNE=f"allgather:cuda:inf:@{alg}#allgatherv:cuda:inf:@{alg}#alltoall:cuda:inf:@{alg}#alltoallv:cuda:inf:@{alg}",
               UCC_TL_NVL_BULK="y" if mover == "push_bulk" else "n", UCC_TL_NVL_BULK_THRESH="0", UCC_TL_NVL_BULK_CTAS="3", **ZC)
    with UccJob(n, env=env) as j:
        team = j.create_team()
        for blk in (4, 1000, 50000):               # 50000 floats = 200000 B: several 24 KB TMA stages per block and a short tail
            src = [gen("float32", blk, 3 * r + blk) for r in range(n)]
            dst = [torch.zeros(blk * n, device="cuda") for _ in range(n)]
            run(team, [cargs("allgather", src[r], dst[r], "float32") for r in range(n)])
            exp = torch.cat(src)
            for r in range(n):
                assert torch.equal(dst[r], exp), ("allgather", mover, n, blk, r)
            src = [gen("float32", blk * n, 7 * r + 1) for r in range(n)]
            dst = [torch.zeros(blk * n, device="cuda") for _ in range(n)]
            run(team, [cargs("alltoall", src[r], dst[r], "float32") for r in range(n)])
            for r in range(n):
                exp = torch.cat([src[p][r * blk:(r + 1) * blk] for p in range(n)])
                assert torch.equal(dst[r], exp), ("alltoall", mover, n, blk, r)
        # skewed alltoallv with odd (unaligned) counts: rank 0 is the hot receiver
        sc = [[(5003 if d == 0 else 17 + 3 * d + s) for d in range(n)] for s in range(n)]      # sc[s][d]: elements s sends to d
        src = [gen("float32", sum(sc[s]), 11 * s) for s in range(n)]
        rc = [[sc[s][d] for s in range(n)] for d in range(n)]
        dst = [torch.zeros(sum(rc[d]), device="cuda") for d in range(n)]
        args = []
        for r in range(n):
            sd = [sum(sc[r][:i]) for i in range(n)]
            rd = [sum(rc[r][:i]) for i in range(n)]
            args.append(cargs("alltoallv", src[r], dst[r], "float32", src_counts=sc[r], src_displs=sd, dst_counts=rc[r], dst_displs=rd))
        run(team, args)
        for d in range(n):
            exp = torch.cat([src[s][sum(sc[s][:d]):sum(sc[s][:d]) + sc[s][d]] for s in range(n)])
            assert torch.equal(dst[d], exp), ("alltoallv", mover, n, d)
        info = __import__("ctypes").CDLL(os.path.join(os.path.dirname(U.LIB_PATH), "ucc", "libucc_tl_nvl.so")).ucc_tl_nvl_last_launch_info
        info.restype = __import__("ctypes").c_char_p
        want = {"push": b"exchange_push ", "push_bulk": b"bulk", "ce": b"copy_engine"}[mover]
        assert want in info() + b" ", info()


# ---------------------------------------------------------------- step-structured algorithms (ring, recursive halving/doubling)
@pytest.fixture(scope="module", params=["ring", "rhd"])
def steps_job(request):
    need_cuda()
    alg = request.param
    tune = f"allreduce:cuda:inf:@{alg}#reduce_scatter:cuda:inf:@{alg}#reduce_scatterv:cuda:inf:@{alg}#allgather:cuda:inf:@ring#allgatherv:cuda:inf:@ring"
    j = UccJob(8, env=dict(ENV, UCC_TL_NVL_TUNE=tune, **NOZC))
    teams = {n: j.create_team(range(n)) for n in (2, 3, 4, 8)}
    yield alg, teams
    j.cleanup()


@pytest.mark.parametrize("n", [2, 3, 4, 8])
@pytest.mark.parametrize("count", [1, 7, 4097, 100003])
def test_steps_allreduce(steps_job, n, count):
    alg, teams = steps_job
    team = teams[n]
    for dt, op in (("float32", "sum"), ("bfloat16", "avg"), ("int32", "max")):
        src = [gen(dt, count, 31 * r + 1) for r in range(n)]
        dst = [torch.zeros(count, dtype=TDT[dt], device="cuda") for _ in range(n)]
        run(team, [cargs("allreduce", src[r], dst[r], dt, op=op) for r in range(n)])
        exp = ref_reduce(op, src)
        for r in range(n):
            assert_close(dst[r], exp, dt)
    # in place
    bufs = [gen("float32", count, r) for r in range(n)]
    exp = ref_reduce("sum", bufs)
    run(team, [cargs("allreduce", None, bufs[r], "float32", inplace=True) for r in range(n)])
    for r in range(n):
        assert_close(bufs[r], exp, "float32")


@pytest.mark.parametrize("n", [2, 4, 8, 3])
def test_steps_reduce_scatter(steps_job, n):
    alg, teams = steps_job
    team = teams[n]
    blk = 1001
    src = [gen("float32", blk * n, r) for r in range(n)]
    dst = [torch.zeros(blk, device="cuda") for _ in range(n)]
    run(team, [cargs("reduce_scatter", src[r], dst[r], "float32") for r in range(n)])
    exp = ref_reduce("sum", src)
    for r in range(n):
        assert_close(dst[r], exp[r * blk:(r + 1) * blk], "float32")
    counts = [100 + 33 * r for r in range(n)]
    tot = sum(counts)
    src = [gen("float32", tot, 5 + r) for r in range(n)]
    dst = [torch.zeros(counts[r], device="cuda") for r in range(n)]
    offs = np.concatenate([[0], np.cumsum(counts)[:-1]])
    run(team, [cargs("reduce_scatterv", src[r], dst[r], "float32", dst_counts=counts, dst_displs=offs) for r in range(n)])
    exp = ref_reduce("sum", src)
    off = 0
    for r in range(n):
        assert_close(dst[r], exp[off:off + counts[r]], "float32")
        off += counts[r]


@pytest.mark.parametrize("n", [2, 3, 8])
@pytest.mark.parametrize("count", [1, 1000, 100001])
def test_ring_allgather(steps_job, n, count):
    alg, teams = steps_job
    team = teams[n]
    for dt in ("float32", "int8"):
        src = [gen(dt, count, 11 * r) for r in range(n)]
        dst = [torch.zeros(count * n, dtype=TDT[dt], device="cuda") for _ in range(n)]
        run(team, [cargs("allgather", src[r], dst[r], dt) for r in range(n)])
        exp = torch.cat(src)
        for r in range(n):
            assert torch.equal(dst[r], exp), (dt, r)
    counts = [count + 3 * r for r in range(n)]
    displs = np.concatenate([[0], np.cumsum(counts)[:-1]])
    src = [gen("int32", counts[r], r) for r in range(n)]
    dst = [torch.zeros(sum(counts), dtype=torch.int32, device="cuda") for _ in range(n)]
    run(team, [cargs("allgatherv", src[r], dst[r], "int32", dst_counts=counts, dst_displs=displs) for r in range(n)])
    for r in range(n):
        assert torch.equal(dst[r], torch.cat(src)), r


def test_single_rank_team_copy_kernel():
    """team of one on CUDA buffers: served by tl/nvl's stream-ordered copy kernel (score above tl/self)."""
    need_cuda()
    with UccJob(1, env=dict(ENV), with_ctx_oob=False) as j:
        team = j.create_team()
        for count in (1, 1000, 1 << 20):
            src = [gen("float32", count, 3)]
            dst = [torch.zeros(count, device="cuda")]
            run(team, [cargs("allreduce", src[0], dst[0], "float32", op="avg")])
            assert torch.equal(dst[0], src[0])
            run(team, [cargs("allgather", src[0], dst[0].zero_(), "float32")])
            assert torch.equal(dst[0], src[0])
            buf = [gen("float32", count, 4)]
            keep = buf[0].clone()
            run(team, [cargs("allreduce", None, buf[0], "float32", inplace=True)])
            assert torch.equal(buf[0], keep)
        run(team, [coll_args("barrier")])


def _p2p_round(j, team, msgs):
    """msgs: list of (src_rank, dst_rank, tensor_src, tensor_dst, tag): init + post everything, progress until done"""
    import ctypes as C
    import time
    reqs = []
    torch.cuda.synchronize()   # the tensors were filled on torch's stream; the (non-blocking) team streams do not wait for it
    for s_, d_, ts, td, tag in msgs:
        for r, buf in ((s_, ts), (d_, td)):
            a = cargs("bcast", buf, None, "float32", root=s_, count_dst=0, active_set=(s_, d_ - s_, 2), tag=tag)
            q = C.POINTER(U.ucc_coll_req_t)()
            st = U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team)
            assert st == U.UCC_OK, U.status_str(st)
            reqs.append((q, a))
    for q, _ in reqs:
        assert U.ucc_collective_post(q) == U.UCC_OK
    t0 = time.time()
    while any(q.contents.status == U.UCC_INPROGRESS for q, _ in reqs) and time.time() - t0 < 20:
        j.progress()
    for q, _ in reqs:
        assert q.contents.status == U.UCC_OK, U.status_str(q.contents.status)
        U.ucc_collective_finalize(q)
    torch.cuda.synchronize()


@pytest.mark.parametrize("thresh", ["inf", "64K"])
@pytest.mark.parametrize("count", [1, 1000, 65536 + 3, 700001])
def test_active_set_p2p(count, thresh):
    """reference test/gtest/active_set/test_active_set.cc:165-184: two-member active-set bcast = send / recv, here on CUDA buffers
    through the tl/nvl channel kernel (700001 floats > the 1 MB ring: sender and receiver pipeline through the slots) and, with
    P2P_RNDV_THRESH=64K, through the rendezvous kernels (the sender stores into the receiver's buffer)"""
    need_cuda()
    n = 4
    # (ZCOPY is set explicitly: module-scoped fixtures of this file keep their own environment alive while other tests run)
    with UccJob(n, env=dict(ENV, UCC_TL_NVL_P2P_RNDV_THRESH=thresh, UCC_TL_NVL_ZCOPY="y")) as j:
        team = j.create_team()
        pairs = [(0, 1), (3, 1), (2, 0), (1, 3)]
        srcs = [gen("float32", count, 10 + i) for i in range(len(pairs))]
        dsts = [torch.zeros(count, device="cuda") for _ in pairs]
        # several messages, two of them to the same receiver, one pair used in both directions; then again (counters persist)
        for rep in range(2):
            for d in dsts:
                d.zero_()
            _p2p_round(j, team, [(s_, d_, srcs[i], dsts[i], 3 + i) for i, (s_, d_) in enumerate(pairs)])
            for i in range(len(pairs)):
                assert torch.equal(dsts[i], srcs[i]), (rep, pairs[i])
        # the team's collectives still work next to the channels
        src = [gen("float32", 5000, r) for r in range(n)]
        dst = [torch.zeros(5000, device="cuda") for _ in range(n)]
        run(team, [cargs("allreduce", src[r], dst[r], "float32") for r in range(n)])
        assert_close(dst[2], ref_reduce("sum", src), "float32")
        import ctypes as C
        info = C.CDLL(os.path.join(os.path.dirname(U.LIB_PATH), "ucc", "libucc_tl_nvl.so")).ucc_tl_nvl_last_launch_info
        info.restype = C.c_char_p
        if count == 700001:
            # burst 2 -> 3: more large messages than board slots, small ones in between, every send posted before any receive
            counts = [40000, 3, 50000, 60000, 17, 70000, 45000]
            bs = [gen("float32", c, 70 + i) for i, c in enumerate(counts)]
            bd = [torch.zeros(c, device="cuda") for c in counts]
            torch.cuda.synchronize()   # the team streams are non-blocking: they do not wait for the stream that fills these tensors
            import time
            sends, recvs = [], []
            for i in range(len(counts)):
                for r, buf, lst in ((2, bs[i], sends), (3, bd[i], recvs)):
                    a = cargs("bcast", buf, None, "float32", root=2, count_dst=0, active_set=(2, 1, 2), tag=30 + i)
                    q = C.POINTER(U.ucc_coll_req_t)()
                    assert U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team) == U.UCC_OK
                    lst.append((q, a))
            for q, _ in sends:
                assert U.ucc_collective_post(q) == U.UCC_OK
            for _ in range(20):
                j.progress()
            for q, _ in recvs:
                assert U.ucc_collective_post(q) == U.UCC_OK
            t0 = time.time()
            while any(q.contents.status == U.UCC_INPROGRESS for q, _ in sends + recvs) and time.time() - t0 < 20:
                j.progress()
            for q, _ in sends + recvs:
                assert q.contents.status == U.UCC_OK, U.status_str(q.contents.status)
                U.ucc_collective_finalize(q)
            torch.cuda.synchronize()
            for i in range(len(counts)):
                assert torch.equal(bd[i], bs[i]), ("burst", i)
            assert ("rndv" in info().decode()) == (thresh == "64K"), info()


@pytest.mark.parametrize("slots", [1, 4])
def test_concurrent_collectives_on_lanes(slots):
    """reference tl_cuda MAX_CONCURRENT (tl_cuda.c:23-28, tl_cuda_coll.h:178-212): with UCC_TL_NVL_SLOTS=4 four allreduces of one team,
    posted stream-ordered on four streams per rank, run on four independent lanes; results must be right and (slots=4, printed) they
    overlap instead of running back to back"""
    import ctypes as C
    import time
    need_cuda()
    n, count, K = 2, 1 << 20, 4
    env = dict(ENV, UCC_TL_NVL_SLOTS=str(slots), UCC_TL_NVL_MAX_BLOCKS="8", **NOZC)
    env["UCC_TL_NVL_TUNE"] = "allreduce:cuda:inf:@twoshot"
    with UccJob(n, env=env) as j:
        team = j.create_team()
        streams = [[torch.cuda.Stream() for _ in range(K)] for _ in range(n)]
        ees = [[None] * K for _ in range(n)]
        for r in range(n):
            for k in range(K):
                ep = U.ucc_ee_params_t()
                ep.ee_type, ep.ee_context, ep.ee_context_size = U.UCC_EE_CUDA_STREAM, streams[r][k].cuda_stream, C.sizeof(C.c_void_p)
                ee = U.handle()
                U.check(U.ucc_ee_create(team.members[r].team, C.byref(ep), C.byref(ee)), "ee_create")
                ees[r][k] = ee
        src = [[gen("float32", count, 10 * r + k) for k in range(K)] for r in range(n)]
        dst = [[torch.zeros(count, device="cuda") for _ in range(K)] for _ in range(n)]
        torch.cuda.synchronize()
        for rep in range(3):
            reqs = []
            t0 = time.perf_counter()
            for k in range(K):                       # same post order on every rank: collective k takes lane k % slots
                for r in range(n):
                    a = cargs("allreduce", src[r][k], dst[r][k], "float32")
                    q = C.POINTER(U.ucc_coll_req_t)()
                    U.check(U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team), "init")
                    ev = U.ucc_ev_t()
                    ev.ev_type, ev.req = U.UCC_EVENT_COMPUTE_COMPLETE, C.cast(q, C.c_void_p)
                    U.check(U.ucc_collective_triggered_post(ees[r][k], C.byref(ev)), "triggered_post")
                    reqs.append((a, q))
            while any(q.contents.status == U.UCC_INPROGRESS for _, q in reqs):
                j.progress()
                assert time.perf_counter() - t0 < 30
            torch.cuda.synchronize()
            dt_ms = (time.perf_counter() - t0) * 1e3
            for _, q in reqs:
                assert q.contents.status == U.UCC_OK
                U.ucc_collective_finalize(q)
        print(f"slots={slots}: {K} allreduces x {count * 4 >> 20} MB on {K} streams took {dt_ms:.2f} ms")
        for k in range(K):
            exp = ref_reduce("sum", [src[r][k] for r in range(n)])
            for r in range(n):
                assert_close(dst[r][k], exp, "float32")
        for r in range(n):
            for k in range(K):
                U.ucc_ee_destroy(ees[r][k])


@pytest.mark.parametrize("alg", ["rab", "split_rail"])
def test_cl_hier_on_cuda_buffers(alg):
    """cl/hier with a synthetic 2-node x 4-GPU placement: node / leaders / rail sub-teams are tl/nvl teams over sub-group maps."""
    need_cuda()
    if alg == "rab" and os.environ.get("UCC_B200_RUN_RAB_EMU") != "1":
        # rab lets the non-leaders enter the node bcast while the leaders still run their cross-node allreduce through the host TL
        # (device buffers staged through mc/ec).  With ALL eight ranks emulated on ONE device, the leaders' device-wide
        # synchronisations (cudaFree / synchronous copies of that staging) wait for the other ranks' spinning bcast kernels, which
        # wait for the leaders: it only resolves through the device-side timeout.  One process per GPU has no such coupling: the
        # schedule is covered with real processes by tests/test_dist_gpu.py::test_multiproc_hier_fake_nodes.
        pytest.skip("single-device emulation couples the ranks through device-wide synchronisation; covered by test_multiproc_hier_fake_nodes")
    env = dict(ENV, UCC_CLS="hier,basic", UCC_CL_HIER_TUNE=f"allreduce:0-inf:@{alg}", **NOZC)
    with UccJob(8, ppn=4, env=env, cls="hier,basic") as j:
        team = j.create_team()
        n = 8
        for count in (16, 4096, 100000):
            src = [gen("float32", count, 7 * r + 1) for r in range(n)]
            dst = [torch.zeros(count, device="cuda") for _ in range(n)]
            run(team, [cargs("allreduce", src[r], dst[r], "float32") for r in range(n)])
            exp = ref_reduce("sum", src)
            for r in range(n):
                assert_close(dst[r], exp, "float32")
        b = [gen("float32", 5000, 3) if r == 0 else torch.zeros(5000, device="cuda") for r in range(n)]
        run(team, [cargs("bcast", b[r], None, "float32", root=0, count_dst=0) for r in range(n)])
        for r in range(n):
            assert torch.equal(b[r], b[0])


def test_asymmetric_memory_at_root(job):
    """reference test/gtest/asym_mem: root's src and dst live in different memory types (staged by the core)."""
    team = job[4]
    n, count = 4, 3000
    # reduce: everybody contributes CUDA data, the root wants the result in HOST memory
    src = [gen("float32", count, r) for r in range(n)]
    host_dst = np.zeros(count, np.float32)
    args = [cargs("reduce", src[r], None, "float32", root=1, count_dst=0) for r in range(n)]
    args[1] = coll_args("reduce", dt="float32", root=1, src_ptr=src[1].data_ptr(), dst_ptr=host_dst.ctypes.data, count_src=count, count_dst=count,
                        src_mem_type=CUDA, dst_mem_type=U.UCC_MEMORY_TYPE_HOST)
    run(team, args)
    assert np.allclose(host_dst, ref_reduce("sum", src).cpu().numpy(), rtol=1e-5)
    # scatter: the root's source is in HOST memory, every destination is CUDA
    host_src = np.arange(n * 100, dtype=np.float32)
    dst = [torch.zeros(100, device="cuda") for _ in range(n)]
    args = [coll_args("scatter", dt="float32", root=0, dst_ptr=dst[r].data_ptr(), count_dst=100, count_src=0, mem_type=CUDA) for r in range(n)]
    args[0] = coll_args("scatter", dt="float32", root=0, src_ptr=host_src.ctypes.data, dst_ptr=dst[0].data_ptr(), count_src=n * 100, count_dst=100,
                        src_mem_type=U.UCC_MEMORY_TYPE_HOST, dst_mem_type=CUDA)
    run(team, args)
    for r in range(n):
        assert np.array_equal(dst[r].cpu().numpy(), host_src[r * 100:(r + 1) * 100])
