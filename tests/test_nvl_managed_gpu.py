"""tl/nvl on CUDA managed memory on a real GPU: the cases of tests/nvl_managed.py with N emulated ranks on cuda:0, buffers from
the library's own managed allocator (mc/cuda: cudaMallocManaged).  Every case runs twice: with the inputs written from the CPU
through the pointer (the pages start on the host) and with the inputs copied in on the device (the pages start on the GPU).
Results are read back through the managed pointer after a device synchronise.  A second test runs two processes on one GPU, so
the buffers cross the exchange board as CUDA IPC candidates (tests/managed_ipc_worker.py)."""
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from ucc_b200 import capi as U  # noqa: E402
from ucc_b200.harness import UccJob, coll_args  # noqa: E402

import nvl_managed as M  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENV = dict(M.ENV, UCC_TL_NVL_MAX_BLOCKS="4", UCC_TL_NVL_TIMEOUT="10s")
_mc_ready = False


def managed_alloc(nbytes, keep):
    """cudaMallocManaged through the library's memory component; the header is freed with the job"""
    global _mc_ready
    if not _mc_ready:
        U.lib.ucc_mc_alloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t, C.c_int]
        U.lib.ucc_mc_free.argtypes = [C.c_void_p]
        _mc_ready = True
    hdr = C.c_void_p()
    assert U.lib.ucc_mc_alloc(C.byref(hdr), nbytes, M.MANAGED) == 0
    keep.append(hdr)
    return C.c_void_p.from_address(hdr.value + 8).value     # ucc_mc_buffer_header_t: {int mt; int from_pool; void *addr}


class _CAI:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 3}


class ManagedBuf:
    def __init__(self, n, keep, on_device):
        self.n, self.on_device = n, on_device
        self.ptr = managed_alloc(n * 4, keep)
        self.a = np.frombuffer((C.c_char * (n * 4)).from_address(self.ptr), dtype=np.int32)

    def write(self, b):
        if self.on_device:      # a copy kernel stores the inputs: the pages move to the GPU
            torch.as_tensor(_CAI(self.ptr, self.n), device="cuda")[:len(b)].copy_(torch.from_numpy(np.ascontiguousarray(b)).cuda())
            torch.cuda.synchronize()
        else:                   # CPU stores through the pointer: the pages start on the host
            self.a[:len(b)] = b

    def read(self):
        return self.a.copy()


class DevBuf:
    def __init__(self, n):
        self.t = torch.zeros(n, dtype=torch.int32, device="cuda")
        self.ptr = self.t.data_ptr()

    def write(self, b):
        self.t[:len(b)].copy_(torch.from_numpy(np.ascontiguousarray(b)))

    def read(self):
        return self.t.cpu().numpy()


def last_launch():
    f = C.CDLL(os.path.join(os.path.dirname(U.LIB_PATH), "ucc", "libucc_tl_nvl.so")).ucc_tl_nvl_last_launch_info
    f.restype = C.c_char_p
    return f().decode()


class H:
    def __init__(self, on_device):
        self.on_device, self.keep, self.streams = on_device, [], []

    def alloc(self, n, managed):
        return ManagedBuf(n, self.keep, self.on_device) if managed else DevBuf(n)

    @staticmethod
    def args(coll, s, d, smt, dmt, **kw):
        return coll_args(coll, dt="int32", src_ptr=s.ptr if s is not None else None, dst_ptr=d.ptr if d is not None else None,
                         src_mem_type=smt, dst_mem_type=dmt, **kw)

    @staticmethod
    def sync():
        torch.cuda.synchronize()

    def stream(self):
        s = torch.cuda.Stream()
        self.streams.append(s)
        return s.cuda_stream

    @staticmethod
    def run(team, args):
        torch.cuda.synchronize()
        q = team.coll(args)
        st = q.run()
        q.finalize()
        assert st == U.UCC_OK, U.status_str(st)
        torch.cuda.synchronize()

    @staticmethod
    def run_p2p(team, args):
        torch.cuda.synchronize()
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
        torch.cuda.synchronize()
        for _, q in reqs:
            assert q.contents.status == U.UCC_OK, q.contents.status
            U.ucc_collective_finalize(q)

    last_launch = staticmethod(last_launch)

    def free(self):
        for hdr in self.keep:
            U.lib.ucc_mc_free(hdr)
        self.keep = []


def need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)


WRITES = ["host_pages", "device_pages"]


@pytest.mark.parametrize("pages", WRITES)
def test_managed_collectives(pages):
    need_cuda()
    h = H(pages == "device_pages")
    with UccJob(4, env=ENV) as j:
        for n in (2, 3, 4):
            M.run_colls(h, j.create_team(range(n), team_id=n), n, seed=100 * n)
        M.run_controls(h, j.create_team(range(3), team_id=13), 3)
        h.free()


@pytest.mark.parametrize("pages", WRITES)
def test_managed_p2p_persistent_triggered(pages):
    need_cuda()
    h = H(pages == "device_pages")
    with UccJob(4, env=ENV) as j:
        for n in (2, 4):
            team = j.create_team(range(n), team_id=n)
            M.run_p2p(h, team, n)
            M.run_persistent(h, team, n)
            M.run_triggered(h, team, n)
        h.free()


@pytest.mark.parametrize("mover", list(M.MOVERS))
def test_managed_push_movers(mover):
    need_cuda()
    h = H(False)
    with UccJob(4, env=dict(ENV, **M.MOVERS[mover][0])) as j:
        for n in (2, 4):
            M.run_push(h, j.create_team(range(n), team_id=n), n, mover)
        h.free()


@pytest.mark.parametrize("pages", WRITES)
def test_managed_team_of_one(pages):
    need_cuda()
    h = H(pages == "device_pages")
    with UccJob(1, env=ENV, with_ctx_oob=False) as j:
        team = j.create_team(team_id=1)
        M.run_self(h, team)
        M.run_self_large(h, team)
        h.free()


def test_managed_mem_map_refused():
    need_cuda()
    h = H(False)
    with UccJob(1, env=ENV, with_ctx_oob=False) as j:
        M.mem_map_refused(U.lib, j.procs[0].ctx, DevBuf(1024), ManagedBuf(1024, h.keep, False), 4096)
        h.free()


def test_managed_two_processes_one_gpu(tmp_path):
    """two processes share cuda:0: the board carries CUDA IPC candidates; managed buffers must stage, device buffers still map"""
    need_cuda()
    env = dict(os.environ, PYTHONPATH=ROOT, **{k: v for k, v in ENV.items() if k != "UCC_TLS"})   # (the service team needs tl/shm)
    worker = os.path.join(ROOT, "tests", "managed_ipc_worker.py")
    store = str(tmp_path / "store")
    procs = [subprocess.Popen([sys.executable, worker, store, str(r)], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = []
    for p in procs:
        try:
            outs.append(p.communicate(timeout=300)[0])
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and "MANAGED_IPC_OK" in o, (r, o[-4000:])
