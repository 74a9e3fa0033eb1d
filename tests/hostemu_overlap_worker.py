"""Worker of tests/test_nvl_overlap.py: UCC_COLL_ARGS_HINT_OPTIMIZE_OVERLAP_GPU (tests/nvl_overlap.py) on the tl/nvl plugin built
against the emulated CUDA runtime (tests/emu/build_hostemu.sh), N ranks in this process.  `hostemu_overlap_worker.py <scenario>`
runs one scenario (numerics<n>: the reductions on a team of n), `all` every one."""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from hostemu_worker import BASE, Dev, U, UccJob, coll_args, last_launch, run  # noqa: E402  (loads the emulated runtime)
from hostemu_graph_worker import Ranks  # noqa: E402
from hostemu_managed_worker import Buf  # noqa: E402
import nvl_numerics as V  # noqa: E402
import nvl_overlap as O  # noqa: E402

from hostemu_worker import rt  # noqa: E402

ENV = dict({k: v for k, v in BASE.items() if k != "UCC_COLL_TRACE"}, **O.ENV)
DTYPES = ["int32", "int64", "uint8", "float32", "float64", "bfloat16", "float32_complex", "float64_complex", "int128", "uint128"]


class Bytes:
    def __init__(self, nbytes):
        self.d = Dev(nbytes, np.uint8)
        self.ptr = self.d.ptr

    def write(self, b):
        self.d.a[:] = b

    def read(self):
        return self.d.a.copy()


class H:
    class mem:
        @staticmethod
        def alloc(nbytes):
            return Bytes(nbytes)

    @staticmethod
    def alloc(nelems, managed):
        return Buf(nelems, managed)

    @staticmethod
    def args(coll, s, d, smt, dmt, **kw):
        return coll_args(coll, dt="int32", src_ptr=s.ptr if s is not None else None, dst_ptr=d.ptr if d is not None else None,
                         src_mem_type=smt, dst_mem_type=dmt, **kw)

    @staticmethod
    def nargs(coll, sp, dp, dt, **kw):
        return coll_args(coll, dt=dt, mem_type=U.UCC_MEMORY_TYPE_CUDA, src_ptr=sp, dst_ptr=dp, **kw)

    @staticmethod
    def sync():
        rt.cudaDeviceSynchronize()

    run = staticmethod(run)
    last_launch = staticmethod(last_launch)


def numerics(n):
    with UccJob(n, env=ENV) as j:
        k = O.run_numerics(H, j.create_team(range(n), team_id=n), n, [d for d in DTYPES if d in V.SIZE], seed=1000 * n)
    print(f"  numerics n={n}: {k} cases bitwise equal to twoshot_zcopy", flush=True)


def rounds():
    symm = 256 << 10
    with UccJob(4, env=dict(ENV, UCC_TL_NVL_SYMMETRIC_SIZE="256K")) as j:
        for n in (2, 3, 4):
            k = O.run_rounds(H, j.create_team(range(n), team_id=n), n, symm)
            print(f"  rounds n={n}: {k} cases ok", flush=True)


def colls():
    with UccJob(4, env=ENV) as j:
        for n in (2, 3, 4):
            team = j.create_team(range(n), team_id=n)
            k = O.run_colls(H, team, n, seed=100 * n)
            k += O.run_vforms(H, team, n)
            print(f"  collectives n={n}: {k} cases ok", flush=True)


def persistent():
    with UccJob(4, env=ENV) as j:
        for n in (2, 4):
            team = j.create_team(range(n), team_id=n)
            k = O.run_persistent(H, team, n)
            k += O.run_registered(H, team, n, [j.procs[r].ctx for r in range(n)])
            print(f"  persistent and registered n={n}: {k} requests ok", flush=True)


def fallbacks():
    with UccJob(4, env=ENV) as j:
        for n in (2, 3):
            k = O.run_fallbacks(H, j.create_team(range(n), team_id=n), n)
            print(f"  managed fallbacks n={n}: {k} cases ok", flush=True)
    with UccJob(1, env=ENV, with_ctx_oob=False) as j:
        k = O.run_self(H, j.create_team(team_id=1))
    print(f"  team of one: {k} cases ok", flush=True)


def captured():
    """a hinted allreduce and bcast posted into a capturing stream, with no cached tables: every rank captures the staged kernel,
    the replay gives the exact result"""
    n, cnt = 3, 20000
    with UccJob(n, env=ENV) as j:
        team = j.create_team(range(n), team_id=n)
        R = Ranks(j, team, n)
        src = [Dev(cnt, np.int32, fill=np.arange(cnt) + r) for r in range(n)]
        dst = [Dev(cnt, np.int32, fill=0) for _ in range(n)]
        buf = [Dev(cnt, np.int32, fill=(np.arange(cnt) * 3 if r == 1 else 0)) for r in range(n)]
        reqs = [[R.init(r, O.hint(coll_args("allreduce", dt="int32", mem_type=U.UCC_MEMORY_TYPE_CUDA, src_ptr=src[r].ptr, dst_ptr=dst[r].ptr,
                                          count_src=cnt, count_dst=cnt))),
                 R.init(r, O.hint(coll_args("bcast", dt="int32", mem_type=U.UCC_MEMORY_TYPE_CUDA, src_ptr=buf[r].ptr, root=1, count_src=cnt,
                                          count_dst=0)))] for r in range(n)]
        graphs, notes = [], []
        for r in range(n):
            graphs.append(R.capture(r, reqs[r]))
            notes.append(last_launch())
        assert all(x.startswith("exchange_pull_staged") for x in notes), notes
        R.replay(graphs)
        for r in range(n):
            assert np.array_equal(dst[r].a, sum(np.arange(cnt) + p for p in range(n)).astype(np.int32)), ("captured allreduce", r)
            assert np.array_equal(buf[r].a, np.arange(cnt) * 3), ("captured bcast", r)
        for r in range(n):
            for q in reqs[r]:
                U.ucc_collective_finalize(q)
            rt.cudaGraphExecDestroy(graphs[r])
        R.close()
    print("  captured posts without tables: staged, exact", flush=True)


SCENARIOS = {"numerics2": lambda: numerics(2), "numerics3": lambda: numerics(3), "numerics4": lambda: numerics(4), "rounds": rounds, "colls": colls, "persistent": persistent, "fallbacks": fallbacks, "captured": captured}

if __name__ == "__main__":
    for name in (SCENARIOS if sys.argv[1] == "all" else sys.argv[1:]):
        SCENARIOS[name]()
    print("HOSTEMU_WORKER_OK", flush=True)
