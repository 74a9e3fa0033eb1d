"""Worker of tests/test_nvl_complex.py: complex float / double reductions through the public UCC API on the tl/nvl plugin built
against the emulated CUDA runtime (tests/emu/build_hostemu_complex.sh), N ranks in this process.  Inputs are Gaussian integers with
components in {-2..2}, so SUM / PROD (and AVG on power-of-two teams) are exact and compared with equality."""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from hostemu_worker import BASE, NOZC, ZC, Dev, U, UccJob, ca, coll_args, rt, run  # noqa: E402  (loads the emulated runtime)

# the emulated plugin with the complex datatypes (tests/emu/build_hostemu_complex.sh), next to the runtime loaded above
os.environ["UCC_MODULE_DIR"] = os.path.join(os.path.dirname(os.environ["UCC_MODULE_DIR"]), "ucc_complex")

DTS = {"float32_complex": np.complex64, "float64_complex": np.complex128}
TRACE = {"UCC_COLL_TRACE": "debug"}   # a coll_init line for every rank, naming the TL that serves the collective


def last_launch():
    info = C.CDLL(os.path.join(os.environ["UCC_MODULE_DIR"], "libucc_tl_nvl.so")).ucc_tl_nvl_last_launch_info
    info.restype = C.c_char_p
    return info().decode()


def gauss(n, seed, dtype):
    g = np.random.default_rng(seed)
    return (g.integers(-2, 3, n) + 1j * g.integers(-2, 3, n)).astype(dtype)


def ref(op, xs):
    st = np.stack([x.astype(np.complex128) for x in xs])
    return {"sum": st.sum(0), "prod": st.prod(0), "avg": st.sum(0) / len(xs)}[op]


def check(got, exp, n, op, what):
    if op != "avg" or n & (n - 1) == 0:
        assert np.array_equal(got.astype(np.complex128), exp), what
    else:
        assert np.allclose(got, exp, rtol=1e-6, atol=1e-6), what


class Shifted:
    """the same device buffer seen k elements further on (an 8-byte aligned complex float vector for odd k)"""

    def __init__(self, dev, k):
        self.ptr = dev.ptr + k * dev.a.itemsize
        self.a = dev.a[k:]


def reductions(extra):
    with UccJob(4, env=dict(BASE, **TRACE, **extra)) as j:
        for n in (3, 4):
            team = j.create_team(range(n))
            for dt, npdt in DTS.items():
                for op in ("sum", "avg", "prod"):
                    for blk in (5, 30011):   # odd blocks: block offsets of a complex float vector are 8-byte aligned only
                        what = (dt, op, n, blk, "zcopy" if extra is ZC else "staged")
                        # allreduce, out of place and in place (30011 * n complex doubles take several heap rounds)
                        src = [Dev(blk * n, npdt, fill=gauss(blk * n, r, npdt)) for r in range(n)]
                        exp = ref(op, [s.a for s in src])
                        dst = [Dev(blk * n, npdt, fill=0) for _ in range(n)]
                        run(team, [ca("allreduce", src[r], dst[r], dt=dt, op=op) for r in range(n)])
                        kern = last_launch()   # (small vectors take the one-shot kernel either way)
                        assert "oneshot" in kern or ("zcopy" in kern) == (extra is ZC), (kern,) + what
                        for r in range(n):
                            check(dst[r].a, exp, n, op, ("allreduce",) + what + (r,))
                        run(team, [ca("allreduce", None, src[r], dt=dt, op=op, inplace=True) for r in range(n)])
                        for r in range(n):
                            check(src[r].a, exp, n, op, ("allreduce inplace",) + what + (r,))
                        # reduce_scatter, out of place and in place
                        src = [Dev(blk * n, npdt, fill=gauss(blk * n, r + 10, npdt)) for r in range(n)]
                        exp = ref(op, [s.a for s in src])
                        dst = [Dev(blk, npdt, fill=0) for _ in range(n)]
                        run(team, [ca("reduce_scatter", src[r], dst[r], dt=dt, op=op) for r in range(n)])
                        for r in range(n):
                            check(dst[r].a, exp[r * blk:(r + 1) * blk], n, op, ("reduce_scatter",) + what + (r,))
                        run(team, [ca("reduce_scatter", None, src[r], dt=dt, op=op, inplace=True) for r in range(n)])
                        for r in range(n):
                            check(src[r].a[r * blk:(r + 1) * blk], exp[r * blk:(r + 1) * blk], n, op, ("reduce_scatter inplace",) + what + (r,))
                        # reduce_scatterv with ragged blocks
                        counts = [blk + 3 * r for r in range(n)]
                        offs = np.concatenate([[0], np.cumsum(counts)[:-1]])
                        src = [Dev(sum(counts), npdt, fill=gauss(sum(counts), r + 20, npdt)) for r in range(n)]
                        exp = ref(op, [s.a for s in src])
                        dst = [Dev(counts[r], npdt, fill=0) for r in range(n)]
                        run(team, [ca("reduce_scatterv", src[r], dst[r], dt=dt, op=op, dst_counts=counts, dst_displs=offs) for r in range(n)])
                        for r in range(n):
                            check(dst[r].a, exp[offs[r]:offs[r] + counts[r]], n, op, ("reduce_scatterv",) + what + (r,))
                        # reduce to the last rank
                        src = [Dev(blk, npdt, fill=gauss(blk, r + 30, npdt)) for r in range(n)]
                        out = Dev(blk, npdt, fill=0)
                        run(team, [ca("reduce", src[r], out if r == n - 1 else None, dt=dt, op=op, root=n - 1, count_dst=blk if r == n - 1 else 0) for r in range(n)])
                        check(out.a, ref(op, [s.a for s in src]), n, op, ("reduce",) + what)
    print(f"  complex reductions {'zcopy' if extra is ZC else 'staged'} ok", flush=True)


def persistent():
    """persistent in-place allreduce, zero-copy where the buffers allow it: complex float buffers 16-byte aligned and 8-byte aligned"""
    n, count = 4, 20001
    with UccJob(n, env=dict(BASE, **TRACE, **ZC, UCC_TL_NVL_ALLREDUCE_ONESHOT_THRESH="0")) as j:
        team = j.create_team(range(n))
        for dt, npdt, shift in (("float32_complex", np.complex64, 0), ("float32_complex", np.complex64, 1), ("float64_complex", np.complex128, 0)):
            bufs = [Shifted(Dev(count + shift, npdt, fill=0), shift) for _ in range(n)]
            for op in ("sum", "prod"):
                q = team.coll([ca("allreduce", None, bufs[r], dt=dt, op=op, inplace=True, persistent=True) for r in range(n)])
                for it in range(3):
                    src = [gauss(count, 100 * it + r, npdt) for r in range(n)]
                    for r in range(n):
                        bufs[r].a[:] = src[r]
                    assert q.run() == U.UCC_OK
                    rt.cudaDeviceSynchronize()
                    assert ("zcopy" in last_launch()) == (shift == 0), (last_launch(), dt, shift)   # 8-byte aligned: staged
                    for r in range(n):
                        check(bufs[r].a, ref(op, src), n, op, ("persistent", dt, op, shift, it, r))
                q.finalize()
    print("  complex persistent in-place allreduce ok", flush=True)


def unsupported_op():
    """MAX has no meaning on complex numbers: tl/nvl rejects it at init and the collective goes down the fallback chain (the test
    checks in the trace that no complex MAX ran on tl/nvl), while the same team serves a complex SUM"""
    n = 2
    with UccJob(n, env=dict(BASE, **TRACE)) as j:
        team = j.create_team(range(n))
        src = [Dev(16, np.complex64, fill=1) for _ in range(n)]
        dst = [Dev(16, np.complex64, fill=0) for _ in range(n)]
        for r in range(n):
            a = ca("allreduce", src[r], dst[r], dt="float32_complex", op="max")
            q = C.POINTER(U.ucc_coll_req_t)()
            st = U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team)
            print(f"  complex max allreduce init on rank {r}: {U.status_str(st)}", flush=True)
            if st == U.UCC_OK:
                U.ucc_collective_finalize(q)
        run(team, [ca("allreduce", src[r], dst[r], dt="float32_complex") for r in range(n)])
        assert all(np.array_equal(d.a, np.full(16, 2, np.complex64)) for d in dst)
    print("  complex sum served after the rejected max ok", flush=True)


if __name__ == "__main__":
    reductions(NOZC)
    reductions(ZC)
    persistent()
    unsupported_op()
    print("HOSTEMU_WORKER_OK", flush=True)
