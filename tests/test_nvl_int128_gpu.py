"""INT128 / UINT128 reductions on tl/nvl on a real GPU (tests/nvl_int128.py, contract in tests/README.md): N emulated ranks share
cuda:0, as in test_nvl_numerics_gpu.py.  One test per (collective, path, team size); each runs both datatypes with all eleven
operators, at the small counts, in place, on buffers 8 bytes off 16-byte alignment (the guarded element path) and, staged two-shot,
over several heap rounds.  The job loads tl/nvl only, so a reduction it turned down would fail instead of running elsewhere."""
import ctypes as C
import os

import pytest

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from ucc_b200 import capi as U  # noqa: E402
from ucc_b200.harness import UccJob, coll_args  # noqa: E402

import nvl_numerics as V  # noqa: E402
import nvl_int128 as Q  # noqa: E402

SYMM = 1 << 20      # UCC_TL_NVL_SYMMETRIC_SIZE: a small heap, so the staged kernel takes several rounds at a modest count
ENV = {"UCC_TL_NVL_MAX_BLOCKS": "4", "UCC_TL_NVL_TIMEOUT": "5s", "UCC_TL_NVL_SYMMETRIC_SIZE": "1Mb"}
SIZES = (2, 3, 4, 8)
COUNT = 67


def colls_of(path):
    return ["allreduce", "reduce_scatter", "reduce_scatterv"] + (["reduce"] if path in ("twoshot", "zcopy") else [])


CASES = [(c, p, n) for p in V.PATHS for c in colls_of(p) for n in SIZES if not (p == "rhd" and n & (n - 1))]


class Buf:
    def __init__(self, nbytes):
        self.t = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        self.ptr = self.t.data_ptr()

    def write(self, b):
        self.t.copy_(torch.from_numpy(b))

    def read(self):
        return self.t.cpu().numpy()


class Mem:
    @staticmethod
    def alloc(nbytes):
        return Buf(nbytes)


def run(team, args):
    torch.cuda.synchronize()      # the inputs were written on torch's stream, the collective runs on the library's
    req = team.coll(args)
    st = req.run()
    req.finalize()
    assert st == U.UCC_OK, U.status_str(st)
    torch.cuda.synchronize()


def last_launch():
    f = C.CDLL(os.path.join(os.path.dirname(U.LIB_PATH), "ucc", "libucc_tl_nvl.so")).ucc_tl_nvl_last_launch_info
    f.restype = C.c_char_p
    return f().decode()


def args(coll, sp, dp, dt, **kw):
    return coll_args(coll, dt=dt, mem_type=U.UCC_MEMORY_TYPE_CUDA, src_ptr=sp, dst_ptr=dp, **kw)


@pytest.fixture(scope="module")
def jobs():
    """one job of 8 ranks per path (its TUNE / zero-copy settings), kept while the tests of that path run"""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    state = {"path": None, "job": None, "teams": {}}

    def team(path, n):
        if state["path"] != path:
            if state["job"] is not None:
                state["job"].cleanup()
            state.update(path=path, job=UccJob(8, env=dict(ENV, **V.path_env(path))), teams={})
        if n not in state["teams"]:
            state["teams"][n] = state["job"].create_team(range(n), team_id=n)
        return state["teams"][n]

    yield team
    if state["job"] is not None:
        state["job"].cleanup()


@pytest.mark.parametrize("coll,path,n", CASES, ids=[f"{c}-{p}-n{n}" for c, p, n in CASES])
def test_int128_reductions(jobs, coll, path, n):
    team = jobs(path, n)
    h = V.Harness(Mem, run, last_launch, args)
    seed = 100000 * n + 1000 * list(V.PATHS).index(path) + 100 * colls_of(path).index(coll)
    blk = COUNT if coll in ("allreduce", "reduce") else COUNT // n + 1
    rsv = [blk + 3 * r for r in range(n)]
    for dt in Q.DTYPES:
        for op in Q.OPS:
            seed += 1
            if coll == "reduce":
                for root in (0, n - 1):
                    Q.run_case(h, team, n, coll, path, dt, op, blk, seed, root=root)
            else:
                Q.run_case(h, team, n, coll, path, dt, op, blk, seed, rs_counts=rsv)
            # 8 bytes off alignment: every operator through the guarded element path
            Q.run_case(h, team, n, coll, path, dt, op, blk, seed + 50, mis=8, root=n - 1,
                       rs_counts=[0 if r == n // 2 else r + 1 for r in range(n)])
            if coll != "reduce":
                Q.run_case(h, team, n, coll, path, dt, op, blk, seed + 60, inplace=True, rs_counts=rsv)
        seed += 1
        if coll == "reduce_scatterv":      # ragged blocks with an empty one
            Q.run_case(h, team, n, coll, path, dt, "sum", None, seed, rs_counts=[0 if r == n // 2 else 2 * r + 1 for r in range(n)])
            continue
        for c in sorted({1, 2, n - 1, n + 1} - {0}):
            Q.run_case(h, team, n, coll, path, dt, "sum", c, seed, root=n - 1)
    if path == "twoshot":                   # several heap rounds, the last one short and ragged
        dt = Q.DTYPES[colls_of(path).index(coll) % 2]
        big = (5 * SYMM // 2) // Q.SIZE + 7 if coll in ("allreduce", "reduce") else (5 * SYMM // 2) // (n * Q.SIZE) + 7
        Q.run_case(h, team, n, coll, path, dt, "sum", big if coll != "reduce_scatterv" else None, seed + 3, root=n - 1,
                   rs_counts=[big + r for r in range(n)])
