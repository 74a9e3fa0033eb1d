"""INT128 / UINT128 on ec/cuda: REDUCE, REDUCE_STRIDED and REDUCE_MULTI_DST for every operator, bitwise against ec/cpu on the same
inputs (AVG with alpha = 1/N included: both divide the wrapped sum by N and truncate), and an allreduce of CUDA buffers on the host transport
(tl/shm), which reduces through ec/cuda."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from ucc_b200 import capi as U  # noqa: E402
from ucc_b200 import internal as I  # noqa: E402
from ucc_b200.harness import UccJob, coll_args  # noqa: E402

import nvl_int128 as Q  # noqa: E402

EC_OPS = [op for op in Q.OPS if op != "avg"]


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    job = UccJob(1)  # keeps mc/ec initialised
    yield
    job.cleanup()


class Twin:
    """the same bytes on the host and on the device, there `mis` bytes past a 16-byte boundary (the host copy stays aligned: ec/cpu
    loads 128-bit integers with 16-byte vector instructions)"""

    def __init__(self, data, mis):
        self.n = data.size
        self.h = np.zeros(self.n + 32, np.uint8)
        ho = -self.h.ctypes.data % 16
        self.hv = self.h[ho:ho + self.n]
        self.hv[:] = data
        self.d = torch.zeros(self.n + 32, dtype=torch.uint8, device="cuda")
        do = (mis - self.d.data_ptr()) % 16
        self.dv = self.d[do:do + self.n]
        self.dv.copy_(torch.from_numpy(self.hv.copy()))

    def hp(self):
        return self.hv.ctypes.data

    def dp(self):
        return self.dv.data_ptr()


def run_both(make_args, dsts):
    """the task on ec/cpu (host copies) and on ec/cuda (device copies): returns [(cpu bytes, cuda bytes)] per destination"""
    for ee, side in ((U.UCC_EE_CPU_THREAD, "h"), (U.UCC_EE_CUDA_STREAM, "d")):
        ex = I.Executor(ee)
        ex.run(make_args(side))
        ex.close()
    torch.cuda.synchronize()
    return [(d.hv.copy(), d.dv.cpu().numpy()) for d in dsts]


def ptr(b, side):
    return b.hp() if side == "h" else b.dp()


@pytest.mark.parametrize("mis", [0, 8])
@pytest.mark.parametrize("dt", Q.DTYPES)
def test_ec_cuda_int128_reduce(cuda, dt, mis):
    """REDUCE of 3 sources (and 5 with AVG) through the vector path (aligned) and the element path (device buffers 8 bytes off)"""
    n = 1003
    for k, op in enumerate(Q.OPS):
        nsrc = 5 if op == "avg" else 3
        x = Q.make_inputs(dt, n, nsrc, 17 * k + mis)
        srcs = [Twin(Q.encode(dt, row), mis) for row in x]
        dst = Twin(np.zeros(n * Q.SIZE, np.uint8), mis)

        def args(side):
            a = I.eee_task_args()
            a.task_type = I.EE_TASK_REDUCE
            a.reduce.dst = ptr(dst, side)
            for i, s in enumerate(srcs):
                a.reduce.srcs[i] = ptr(s, side)
            a.reduce.n_srcs, a.reduce.count, a.reduce.dt, a.reduce.op = nsrc, n, U.DT[dt], U.OP[op]
            if op == "avg":
                a.flags = I.EEE_FLAG_ALPHA
                a.reduce.alpha = 1.0 / nsrc
            return a

        (hb, db), = run_both(args, [dst])
        assert np.array_equal(hb, db), f"{dt} {op} mis={mis}: ec/cuda differs from ec/cpu"
        if op != "avg":
            Q.check_values(dt, op, x, Q.decode(dt, db), f"ec/cuda reduce {dt} {op} mis={mis}")
        else:
            got = Q.decode(dt, db)
            s = [Q.reference(dt, "sum", [row[i] for row in x]) for i in range(n)]
            assert all(abs(g - v / nsrc) <= 1 + abs(v) * 2.0 ** -52 for g, v in zip(got, s)), f"{dt} avg mis={mis} far from S/N"


@pytest.mark.parametrize("dt", Q.DTYPES)
def test_ec_cuda_int128_strided_and_multi_dst(cuda, dt):
    n = 517
    for k, op in enumerate(Q.OPS):
        # strided: src1 and 4 vectors back to back in src2 (AVG: alpha 1/5)
        x = Q.make_inputs(dt, n, 5, 1000 + k)
        s1 = Twin(Q.encode(dt, x[0]), 0)
        s2 = Twin(np.concatenate([Q.encode(dt, row) for row in x[1:]]), 0)
        dst = Twin(np.zeros(n * Q.SIZE, np.uint8), 0)

        def strided(side):
            a = I.eee_task_args()
            a.task_type = I.EE_TASK_REDUCE_STRIDED
            rs = a.reduce_strided
            rs.dst, rs.src1, rs.src2, rs.stride, rs.count = ptr(dst, side), ptr(s1, side), ptr(s2, side), n * Q.SIZE, n
            rs.dt, rs.op, rs.n_src2 = U.DT[dt], U.OP[op], 4
            if op == "avg":
                a.flags = I.EEE_FLAG_ALPHA
                rs.alpha = 1.0 / 5
            return a

        (hb, db), = run_both(strided, [dst])
        assert np.array_equal(hb, db), f"strided {dt} {op}: ec/cuda differs from ec/cpu"
        if op != "avg":
            Q.check_values(dt, op, x, Q.decode(dt, db), f"ec/cuda reduce_strided {dt} {op}")
            # multi dst: 3 independent pairs of different lengths
            ys = [Q.make_inputs(dt, 10 + 7 * j, 2, 2000 + 10 * k + j) for j in range(3)]
            a1 = [Twin(Q.encode(dt, y[0]), 0) for y in ys]
            a2 = [Twin(Q.encode(dt, y[1]), 0) for y in ys]
            ds = [Twin(np.zeros((10 + 7 * j) * Q.SIZE, np.uint8), 0) for j in range(3)]

            def multi(side):
                a = I.eee_task_args()
                a.task_type = I.EE_TASK_REDUCE_MULTI_DST
                m = a.reduce_multi_dst
                for j in range(3):
                    m.dst[j], m.src1[j], m.src2[j], m.counts[j] = ptr(ds[j], side), ptr(a1[j], side), ptr(a2[j], side), 10 + 7 * j
                m.dt, m.op, m.n_bufs = U.DT[dt], U.OP[op], 3
                return a

            for j, (hb, db) in enumerate(run_both(multi, ds)):
                assert np.array_equal(hb, db), f"multi_dst {dt} {op} buffer {j}: ec/cuda differs from ec/cpu"
                Q.check_values(dt, op, ys[j], Q.decode(dt, db), f"ec/cuda reduce_multi_dst {dt} {op} buffer {j}")


@pytest.mark.parametrize("dt", Q.DTYPES)
def test_shm_allreduce_int128_on_cuda_buffers(cuda, dt):
    """the host transport serves INT128 / UINT128 allreduce of device buffers (it reduces with ec/cuda)"""
    n, count = 4, 301
    with UccJob(n, env={"UCC_TLS": "shm,self"}) as job:
        team = job.create_team(range(n))
        for k, op in enumerate(EC_OPS):
            x = Q.make_inputs(dt, count, n, 3000 + k)
            src = [torch.from_numpy(Q.encode(dt, row)).cuda() for row in x]
            dst = [torch.zeros(count * Q.SIZE, dtype=torch.uint8, device="cuda") for _ in range(n)]
            torch.cuda.synchronize()
            req = team.coll([coll_args("allreduce", dt=dt, op=op, mem_type=U.UCC_MEMORY_TYPE_CUDA, src_ptr=src[r].data_ptr(),
                                       dst_ptr=dst[r].data_ptr(), count_src=count, count_dst=count) for r in range(n)])
            st = req.run()
            req.finalize()
            assert st == U.UCC_OK, f"{dt} {op}: {U.status_str(st)}"
            torch.cuda.synchronize()
            for r in range(n):
                Q.check_values(dt, op, x, Q.decode(dt, dst[r].cpu().numpy()), f"tl/shm allreduce {dt} {op} rank {r}")
