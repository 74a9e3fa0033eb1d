"""Complex float / double reductions on tl/nvl on a real GPU (N emulated ranks on cuda:0, as in tests/test_nvl_gpu.py).  Inputs are
Gaussian integers with components in {-2..2}: sums and products over up to 8 ranks are exact in float whatever the order, so SUM /
PROD (and AVG on power-of-two teams) are compared with the complex128 reference for equality."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from test_nvl_gpu import U, alg_job, cargs, job, steps_job  # noqa: E402,F401  (module fixtures of the same jobs)
from test_nvl_gpu import run as run_coll  # noqa: E402

CDT = {"float32_complex": torch.complex64, "float64_complex": torch.complex128}
CASES = [(dt, op) for dt in CDT for op in ("sum", "avg", "prod")]


def gauss(dt, n, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    re, im = (torch.randint(-2, 3, (n,), generator=g).double() for _ in range(2))
    return torch.complex(re, im).to(CDT[dt]).cuda()


def run(team, args):
    torch.cuda.synchronize()   # the inputs were filled on torch's stream; the team streams do not wait for it
    run_coll(team, args)


def ref(op, xs):
    a = torch.stack([x.cpu().to(torch.complex128) for x in xs])
    if op == "prod":
        out = a[0]
        for x in a[1:]:
            out = out * x
        return out
    return a.sum(0) / len(xs) if op == "avg" else a.sum(0)


def check(got, exp, n, op):
    got = got.cpu().to(torch.complex128)
    if op != "avg" or n & (n - 1) == 0:
        assert torch.equal(got, exp), (got - exp).abs().max()
    else:
        assert torch.allclose(got, exp, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("n", [2, 3, 4, 8])
@pytest.mark.parametrize("dt,op", CASES)
def test_complex_allreduce(alg_job, dt, op, n):
    alg, teams = alg_job
    for count in (1, 7, 4097, 100001):
        src = [gauss(dt, count, 10 * r + count) for r in range(n)]
        dst = [torch.zeros(count, dtype=CDT[dt], device="cuda") for _ in range(n)]
        run(teams[n], [cargs("allreduce", src[r], dst[r], dt, op=op) for r in range(n)])
        exp = ref(op, src)
        for r in range(n):
            check(dst[r], exp, n, op)


@pytest.mark.parametrize("n", [2, 3, 4, 8])
@pytest.mark.parametrize("dt,op", CASES)
def test_complex_steps_allreduce(steps_job, dt, op, n):
    alg, teams = steps_job
    for count in (7, 100003):
        src = [gauss(dt, count, 31 * r + 1) for r in range(n)]
        dst = [torch.zeros(count, dtype=CDT[dt], device="cuda") for _ in range(n)]
        run(teams[n], [cargs("allreduce", src[r], dst[r], dt, op=op) for r in range(n)])
        exp = ref(op, src)
        for r in range(n):
            check(dst[r], exp, n, op)
    blk = 1001
    src = [gauss(dt, blk * n, 5 + r) for r in range(n)]
    dst = [torch.zeros(blk, dtype=CDT[dt], device="cuda") for _ in range(n)]
    run(teams[n], [cargs("reduce_scatter", src[r], dst[r], dt, op=op) for r in range(n)])
    exp = ref(op, src)
    for r in range(n):
        check(dst[r], exp[r * blk:(r + 1) * blk], n, op)


@pytest.mark.parametrize("n", [2, 3, 8])
@pytest.mark.parametrize("dt,op", CASES)
def test_complex_reduce_scatter(job, dt, op, n):
    """odd block sizes: the blocks of a complex float vector are only 8-byte aligned and take the staged kernel"""
    team = job[n]
    for blk in (1237, 40000):
        src = [gauss(dt, blk * n, r + blk) for r in range(n)]
        exp = ref(op, src)
        dst = [torch.zeros(blk, dtype=CDT[dt], device="cuda") for _ in range(n)]
        run(team, [cargs("reduce_scatter", src[r], dst[r], dt, op=op) for r in range(n)])
        for r in range(n):
            check(dst[r], exp[r * blk:(r + 1) * blk], n, op)
        bufs = [s.clone() for s in src]
        run(team, [cargs("reduce_scatter", None, bufs[r], dt, op=op, inplace=True) for r in range(n)])
        for r in range(n):
            check(bufs[r][r * blk:(r + 1) * blk], exp[r * blk:(r + 1) * blk], n, op)
    counts = [100 + 33 * r for r in range(n)]
    offs = np.concatenate([[0], np.cumsum(counts)[:-1]])
    src = [gauss(dt, sum(counts), 50 + r) for r in range(n)]
    dst = [torch.zeros(counts[r], dtype=CDT[dt], device="cuda") for r in range(n)]
    run(team, [cargs("reduce_scatterv", src[r], dst[r], dt, op=op, dst_counts=counts, dst_displs=offs) for r in range(n)])
    exp = ref(op, src)
    for r in range(n):
        check(dst[r], exp[offs[r]:offs[r] + counts[r]], n, op)


@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("dt,op", CASES)
def test_complex_reduce(job, dt, op, n):
    team = job[n]
    count = 5001
    for root in {0, n - 1}:
        src = [gauss(dt, count, 7 * r + root) for r in range(n)]
        dst = torch.zeros(count, dtype=CDT[dt], device="cuda")
        run(team, [cargs("reduce", src[r], dst if r == root else None, dt, op=op, root=root, count_dst=count) for r in range(n)])
        check(dst, ref(op, src), n, op)


@pytest.mark.parametrize("op", ["sum", "prod"])
def test_complex_allreduce_inplace_persistent_unaligned(alg_job, op):
    """complex float buffers that are only 8-byte aligned: the guarded element path of every kernel"""
    alg, teams = alg_job
    n, count, dt = 4, 3001, "float32_complex"
    base = [torch.zeros(count + 1, dtype=torch.complex64, device="cuda") for _ in range(n)]
    bufs = [b[1:] for b in base]
    assert all(b.data_ptr() % 16 == 8 for b in bufs)
    req = teams[n].coll([cargs("allreduce", None, bufs[r], dt, op=op, inplace=True, persistent=True) for r in range(n)])
    for it in range(3):
        src = [gauss(dt, count, 10 * it + r) for r in range(n)]
        for r in range(n):
            bufs[r].copy_(src[r])
        torch.cuda.synchronize()
        assert req.run() == U.UCC_OK
        torch.cuda.synchronize()
        exp = ref(op, src)
        for r in range(n):
            check(bufs[r], exp, n, op)
    req.finalize()
