"""Worker of tests/test_nvl_int128.py: the INT128 / UINT128 contract of tests/nvl_int128.py on the tl/nvl plugin built against the
emulated CUDA runtime (tests/emu/build_hostemu.sh), N ranks in this process.  `hostemu_int128_worker.py <path>` runs allreduce,
reduce_scatter(v) and reduce on one path (nvl_numerics.PATHS) for teams of 2..5, both datatypes, every operator."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from hostemu_worker import UccJob, last_launch, run  # noqa: E402  (loads the emulated runtime)
from hostemu_numerics_worker import Mem, args, colls_of  # noqa: E402
import nvl_numerics as V  # noqa: E402
import nvl_int128 as Q  # noqa: E402

SIZES = (2, 3, 4, 5)
ENV = {"UCC_TL_NVL_MAX_BLOCKS": "2", "UCC_TL_NVL_NTHREADS": "64", "UCC_TL_NVL_TIMEOUT": "30s", "UCC_TL_NVL_SYMMETRIC_SIZE": "1Mb"}


def main(path):
    h = V.Harness(Mem, run, last_launch, args)
    env = dict(ENV, **V.path_env(path))
    ncases = 0
    with UccJob(max(SIZES), env=env) as j:
        for n in SIZES:
            if path == "rhd" and n & (n - 1):
                continue
            team = j.create_team(range(n), team_id=n)
            for coll in colls_of(path):
                seed = 1000 * n + 17 * len(coll)
                blk = 7 if coll in ("allreduce", "reduce") else 3
                rsv = [r + 1 for r in range(n)]
                for dt in Q.DTYPES:
                    for op in Q.OPS:
                        seed += 1
                        for root in ((0, n - 1) if coll == "reduce" else (0,)):
                            Q.run_case(h, team, n, coll, path, dt, op, blk, seed, root=root, rs_counts=rsv)
                            ncases += 1
                    # 8 bytes off alignment (the guarded element path), in place, an empty block
                    for op in ("sum", "prod", "max", "avg"):
                        seed += 1
                        Q.run_case(h, team, n, coll, path, dt, op, blk, seed, mis=8, root=n - 1,
                                   rs_counts=[0 if r == 1 else r + 2 for r in range(n)])
                        ncases += 1
                    if coll != "reduce":
                        Q.run_case(h, team, n, coll, path, dt, "bxor", blk, seed + 1, inplace=True, rs_counts=rsv)
                        ncases += 1
                    for c in (1, n + 1):
                        if coll != "reduce_scatterv":
                            Q.run_case(h, team, n, coll, path, dt, "sum", c, seed + 2, root=n - 1)
                            ncases += 1
            print(f"  {path} n={n} ok", flush=True)
    print(f"  {ncases} cases", flush=True)


if __name__ == "__main__":
    main(sys.argv[1])
    print("HOSTEMU_WORKER_OK", flush=True)
