"""Worker of tests/test_nvl_xchg.py: the byte contract of tests/nvl_xchg.py on the tl/nvl plugin built against the emulated CUDA
runtime (tests/emu/build_hostemu.sh), N ranks in this process.  `hostemu_xchg_worker.py <path>` runs every collective family the
path serves (nvl_xchg.PATHS) for teams of 2..5 (`self`: a team of one), and the heap bound of the path on a 1 MB heap."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from hostemu_worker import BASE, Dev, U, UccJob, coll_args, last_launch, run  # noqa: E402  (loads the emulated runtime)
import nvl_xchg as X  # noqa: E402

SIZES = (2, 3, 4, 5)
SYMM = 1 << 20


class Buf:
    def __init__(self, nbytes):
        self.d = Dev(nbytes, np.uint8)
        self.ptr = self.d.ptr

    def write(self, b):
        self.d.a[:] = b

    def read(self):
        return self.d.a.copy()


class Mem:
    @staticmethod
    def alloc(nbytes):
        return Buf(nbytes)


def args(coll, sp, dp, dt, **kw):
    return coll_args(coll, dt=dt, mem_type=U.UCC_MEMORY_TYPE_CUDA, src_ptr=sp, dst_ptr=dp, **kw)


def main(path):
    h = X.Harness(Mem, run, last_launch, args)
    env = {k: v for k, v in BASE.items() if k != "UCC_COLL_TRACE"}
    env.update(X.path_env(path), UCC_TL_NVL_SYMMETRIC_SIZE="1Mb")
    ncases = 0
    fams = X.PATHS[path][1]
    if path == "self":
        with UccJob(1, env=env, with_ctx_oob=False) as j:
            team = j.create_team(team_id=1)
            for k, fam in enumerate(fams):
                ncases += X.run_cases(h, team, 1, path, fam, 77 + 1000 * k, k)
        print(f"  {path} n=1 ok, {ncases} cases", flush=True)
        return
    with UccJob(max(SIZES), env=env) as j:
        for n in SIZES:
            team = j.create_team(range(n), team_id=n)
            for k, fam in enumerate(fams):
                ncases += X.run_cases(h, team, n, path, fam, 100000 * n + 1000 * k, k + n)
            ncases += X.run_heap_bound(h, j.create_team(range(n), team_id=10 + n), n, path, SYMM, 555 + n)
            print(f"  {path} n={n} ok", flush=True)
    print(f"  {ncases} cases", flush=True)


if __name__ == "__main__":
    main(sys.argv[1])
    print("HOSTEMU_WORKER_OK", flush=True)
