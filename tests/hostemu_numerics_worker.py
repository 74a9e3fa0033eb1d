"""Worker of tests/test_nvl_numerics.py: the numerical contract of tests/nvl_numerics.py on the tl/nvl plugin built against the
emulated CUDA runtime (tests/emu/build_hostemu.sh), N ranks in this process.  `hostemu_numerics_worker.py <path>` runs allreduce,
reduce_scatter(v) and reduce on one path (nvl_numerics.PATHS) for teams of 2..5, the eight datatypes the emulated plugin builds
besides INT128 / UINT128 (those: hostemu_int128_worker.py)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from hostemu_worker import BASE, Dev, U, UccJob, coll_args, last_launch, run  # noqa: E402  (loads the emulated runtime)
import nvl_numerics as V  # noqa: E402

DTYPES = ["int32", "int64", "uint8", "float32", "float64", "bfloat16", "float32_complex", "float64_complex"]
SIZES = (2, 3, 4, 5)


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


def colls_of(path):
    return ["allreduce", "reduce_scatter", "reduce_scatterv"] + (["reduce"] if path in ("twoshot", "zcopy") else [])


def main(path):
    h = V.Harness(Mem, run, last_launch, args)
    env = {k: v for k, v in BASE.items() if k != "UCC_COLL_TRACE"}
    env.update(V.path_env(path))
    ncases = 0
    with UccJob(max(SIZES), env=env) as j:
        for n in SIZES:
            if path == "rhd" and n & (n - 1):
                continue
            team = j.create_team(range(n), team_id=n)
            for coll in colls_of(path):
                seed = 1000 * n + 17 * len(coll)
                for dt in DTYPES:
                    e = 16 // V.SIZE[dt]
                    for op in V.ops_of(dt):
                        seed += 1
                        if coll == "reduce":
                            for root in (0, n - 1):
                                V.run_case(h, team, n, coll, path, dt, op, 3 * e + 5, seed, root=root)
                                ncases += 1
                        elif coll == "reduce_scatterv":
                            V.run_case(h, team, n, coll, path, dt, op, None, seed, rs_counts=[e + 3 * r for r in range(n)])
                            ncases += 1
                        else:
                            V.run_case(h, team, n, coll, path, dt, op, 3 * e + 5, seed)
                            ncases += 1
                    # shapes, misalignment, in place, an empty block: SUM
                    for c in V.small_counts(dt, n):
                        seed += 1
                        if coll == "reduce_scatterv":
                            continue
                        V.run_case(h, team, n, coll, path, dt, "sum", c, seed, root=n - 1)
                        ncases += 1
                    if coll == "reduce_scatterv":
                        V.run_case(h, team, n, coll, path, dt, "sum", None, seed + 1, rs_counts=[e + 1 if r != 1 else 0 for r in range(n)])
                        ncases += 1
                    elif V.SIZE[dt] < 16:
                        V.run_case(h, team, n, coll, path, dt, "sum", 2 * e + 3, seed + 2, mis=V.SIZE[dt], root=n - 1)
                        ncases += 1
                    if coll in ("allreduce", "reduce_scatter"):
                        V.run_case(h, team, n, coll, path, dt, V.ops_of(dt)[-1], 2 * e + 1, seed + 3, inplace=True)
                        ncases += 1
            print(f"  {path} n={n} ok", flush=True)
    print(f"  {ncases} cases", flush=True)


if __name__ == "__main__":
    main(sys.argv[1])
    print("HOSTEMU_WORKER_OK", flush=True)
