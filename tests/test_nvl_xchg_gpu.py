"""The byte contract of the tl/nvl data-movement collectives (tests/nvl_xchg.py, written down in tests/README.md) on a real GPU: N
emulated ranks share cuda:0, as in test_nvl_numerics_gpu.py.  One test per (path, collective family, team size): every layout of
every collective of the family, each run twice with fresh data and another layout, with rotating element sizes (1..16 bytes),
misalignments (0, 1, 4, 8 bytes) and 32- / 64-bit counts, in place where the path allows it, both roots of the rooted collectives;
the tests of the allgather family also check the heap bound of their path.  push_bulk is the only place the TMA mover runs."""
import ctypes as C
import os

import pytest

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from ucc_b200 import capi as U  # noqa: E402
from ucc_b200.harness import UccJob, coll_args  # noqa: E402

import nvl_xchg as X  # noqa: E402

SYMM = 1 << 20      # UCC_TL_NVL_SYMMETRIC_SIZE: the heap bound is tested against it
ENV = {"UCC_TL_NVL_MAX_BLOCKS": "4", "UCC_TL_NVL_TIMEOUT": "5s", "UCC_TL_NVL_SYMMETRIC_SIZE": "1Mb"}
SIZES = range(2, 9)

CASES = [(p, f, n) for p in X.PATHS if p != "self" for f in X.PATHS[p][1] for n in SIZES]


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
    """one job of 8 ranks per path (its TUNE / zero-copy / bulk settings), kept while the tests of that path run"""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    state = {"path": None, "job": None, "teams": {}}

    def team(path, n, team_id=None):
        if state["path"] != path:
            if state["job"] is not None:
                state["job"].cleanup()
            env = dict(ENV, **X.path_env(path))
            state.update(path=path, job=UccJob(1, env=env, with_ctx_oob=False) if path == "self" else UccJob(8, env=env), teams={})
        key = team_id or n
        if key not in state["teams"]:
            j = state["job"]
            state["teams"][key] = j.create_team(team_id=1) if path == "self" else j.create_team(range(n), team_id=key)
        return state["teams"][key]

    yield team
    if state["job"] is not None:
        state["job"].cleanup()


@pytest.mark.parametrize("path,family,n", CASES, ids=[f"{p}-{f}-n{n}" for p, f, n in CASES])
def test_xchg_contract(jobs, path, family, n):
    h = X.Harness(Mem, run, last_launch, args)
    k = list(X.FAMILIES).index(family)
    X.run_cases(h, jobs(path, n), n, path, family, 100000 * n + 1000 * k + 10 * list(X.PATHS).index(path), k + n)
    if family == "allgather":
        X.run_heap_bound(h, jobs(path, n, team_id=10 + n), n, path, SYMM, 555 + n)


def test_xchg_contract_team_of_one(jobs):
    h = X.Harness(Mem, run, last_launch, args)
    for k, family in enumerate(X.FAMILIES):
        X.run_cases(h, jobs("self", 1), 1, "self", family, 77 + 1000 * k, k)
