"""Worker of tests/test_nvl_int128.py: the INT128 / UINT128 contract of tests/nvl_int128.py on the tl/nvl plugin built against the
emulated CUDA runtime with INT128 / UINT128 in its datatype table (tests/emu/build_hostemu_int128.sh), N ranks in this process.
`hostemu_int128_worker.py <path>` runs allreduce, reduce_scatter(v) and reduce on one path (nvl_numerics.PATHS) for teams of 2..5,
both datatypes, every operator."""
import ctypes as C
import faulthandler
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ["UCC_MODULE_DIR"] = os.path.join(ROOT, "build-emu", "lib", "ucc_int128")
faulthandler.dump_traceback_later(240, exit=True)
rt = C.CDLL(os.path.join(ROOT, "build-emu", "lib", "libcudart_emu.so"), mode=C.RTLD_GLOBAL)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ucc_b200 import capi as U  # noqa: E402
from ucc_b200.harness import UccJob, coll_args  # noqa: E402
import nvl_numerics as V  # noqa: E402
import nvl_int128 as Q  # noqa: E402

SIZES = (2, 3, 4, 5)
ENV = {"UCC_TL_NVL_MAX_BLOCKS": "2", "UCC_TL_NVL_NTHREADS": "64", "UCC_TL_NVL_TIMEOUT": "30s", "UCC_TL_NVL_SYMMETRIC_SIZE": "1Mb"}


class Buf:
    """a buffer of the emulated cudaMalloc"""

    def __init__(self, nbytes):
        p = C.c_void_p()
        assert rt.cudaMalloc(C.byref(p), C.c_size_t(max(nbytes, 1))) == 0
        self.ptr = p.value
        self.a = np.frombuffer((C.c_char * max(nbytes, 1)).from_address(p.value), dtype=np.uint8)[:nbytes]

    def write(self, b):
        self.a[:] = b

    def read(self):
        return self.a.copy()


class Mem:
    @staticmethod
    def alloc(nbytes):
        return Buf(nbytes)


def run(team, args):
    q = team.coll(args)
    st = q.run()
    q.finalize()
    assert st == U.UCC_OK, U.status_str(st)
    rt.cudaDeviceSynchronize()


def last_launch():
    info = C.CDLL(os.path.join(os.environ["UCC_MODULE_DIR"], "libucc_tl_nvl.so")).ucc_tl_nvl_last_launch_info
    info.restype = C.c_char_p
    return info().decode()


def args(coll, sp, dp, dt, **kw):
    return coll_args(coll, dt=dt, mem_type=U.UCC_MEMORY_TYPE_CUDA, src_ptr=sp, dst_ptr=dp, **kw)


def colls_of(path):
    return ["allreduce", "reduce_scatter", "reduce_scatterv"] + (["reduce"] if path in ("twoshot", "zcopy") else [])


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
