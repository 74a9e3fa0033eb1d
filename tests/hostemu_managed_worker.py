"""Worker of tests/test_nvl_managed.py: tl/nvl on CUDA managed memory (tests/nvl_managed.py) with the plugin built against the
emulated CUDA runtime (tests/emu/build_hostemu.sh), N ranks in this process.  The emulated cudaMallocManaged registers its
allocations as cudaMemoryTypeManaged, and the emulated cudaIpcGetMemHandle refuses them, as the real runtime does.
`hostemu_managed_worker.py all` runs every scenario; any one of them can be named instead."""
import ctypes as C
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from hostemu_worker import BASE, U, UccJob, coll_args, last_launch, rt  # noqa: E402  (loads the emulated runtime)
import nvl_managed as M  # noqa: E402


class Buf:
    def __init__(self, nelems, managed):
        p = C.c_void_p()
        nbytes = nelems * 4
        fn = rt.cudaMallocManaged if managed else rt.cudaMalloc
        assert (fn(C.byref(p), C.c_size_t(nbytes), 1) if managed else fn(C.byref(p), C.c_size_t(nbytes))) == 0
        self.ptr = p.value
        self.a = np.frombuffer((C.c_char * nbytes).from_address(p.value), dtype=np.int32)

    def write(self, b):
        self.a[:len(b)] = b

    def read(self):
        return self.a.copy()


class H:
    @staticmethod
    def alloc(nelems, managed):
        return Buf(nelems, managed)

    @staticmethod
    def args(coll, s, d, smt, dmt, **kw):
        return coll_args(coll, dt="int32", src_ptr=s.ptr if s is not None else None, dst_ptr=d.ptr if d is not None else None,
                         src_mem_type=smt, dst_mem_type=dmt, **kw)

    @staticmethod
    def sync():
        rt.cudaDeviceSynchronize()

    @staticmethod
    def stream():
        rt.cudaStreamCreate.argtypes = [C.POINTER(C.c_void_p)]
        s = C.c_void_p()
        assert rt.cudaStreamCreate(C.byref(s)) == 0
        return s.value

    @staticmethod
    def run(team, args):
        q = team.coll(args)
        st = q.run()
        q.finalize()
        assert st == U.UCC_OK, U.status_str(st)
        rt.cudaDeviceSynchronize()

    @staticmethod
    def run_p2p(team, args):
        reqs = []
        for r, a in args.items():
            q = C.POINTER(U.ucc_coll_req_t)()
            U.check(U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team), "init")
            reqs.append((a, q))
        for _, q in reqs:
            U.check(U.ucc_collective_post(q), "post")
        t0 = time.time()
        while any(q.contents.status == U.UCC_INPROGRESS for _, q in reqs):
            for m in team.members:
                U.ucc_context_progress(m.proc.ctx)
            assert time.time() - t0 < 120, "send / recv did not complete"
        rt.cudaDeviceSynchronize()
        for _, q in reqs:
            assert q.contents.status == U.UCC_OK, q.contents.status
            U.ucc_collective_finalize(q)

    last_launch = staticmethod(last_launch)


ENV = dict({k: v for k, v in BASE.items() if k != "UCC_COLL_TRACE"}, **M.ENV)


def colls():
    with UccJob(4, env=ENV) as j:
        for n in (2, 3, 4):
            team = j.create_team(range(n), team_id=n)
            k = M.run_colls(H, team, n, seed=100 * n)
            print(f"  collectives n={n}: {k} cases ok", flush=True)
        M.run_controls(H, j.create_team(range(3), team_id=13), 3)
        print("  per-buffer decision ok", flush=True)


def persistent():
    with UccJob(4, env=ENV) as j:
        for n in (2, 4):
            M.run_persistent(H, j.create_team(range(n), team_id=n), n)
    print("  persistent requests ok", flush=True)


def p2p():
    with UccJob(4, env=ENV) as j:
        for n in (2, 3, 4):
            k = M.run_p2p(H, j.create_team(range(n), team_id=n), n)
            print(f"  send / recv n={n}: {k} messages ok", flush=True)


def push():
    for mover, (env, _) in M.MOVERS.items():
        with UccJob(4, env=dict(ENV, **env)) as j:
            for n in (2, 4):
                k = M.run_push(H, j.create_team(range(n), team_id=n), n, mover)
                print(f"  @{mover} on managed buffers n={n}: {k} cases ok", flush=True)


def triggered():
    with UccJob(4, env=ENV) as j:
        for n in (2, 3):
            k = M.run_triggered(H, j.create_team(range(n), team_id=n), n)
            print(f"  triggered posts n={n}: {k} cases ok", flush=True)


def self_team():
    with UccJob(1, env=ENV, with_ctx_oob=False) as j:
        team = j.create_team(team_id=1)
        k = M.run_self(H, team)
        k += M.run_self_large(H, team)
    print(f"  team of one: {k} cases ok", flush=True)


def mem_map():
    with UccJob(1, env=ENV, with_ctx_oob=False) as j:
        M.mem_map_refused(U.lib, j.procs[0].ctx, Buf(1024, False), Buf(1024, True), 4096)
    print("  ucc_mem_map of a managed segment refused ok", flush=True)


SCENARIOS = {"colls": colls, "persistent": persistent, "p2p": p2p, "push": push, "triggered": triggered, "self": self_team, "mem_map": mem_map}

if __name__ == "__main__":
    for name in (SCENARIOS if sys.argv[1] == "all" else sys.argv[1:]):
        SCENARIOS[name]()
    print("HOSTEMU_WORKER_OK", flush=True)
