"""Worker of tests/test_nvl_managed_gpu.py::test_managed_two_processes_one_gpu: one of two processes on the same GPU (argv: store
file, rank).  Allreduce, allgather, alltoall and send / recv on managed buffers (the library's cudaMallocManaged allocator), above
the zero-copy and rendezvous thresholds, must each run the staged form, because the owner of a managed buffer publishes it as not
mappable; the same allreduce on device tensors must still go zero-copy through CUDA IPC.  Consecutive checks expect different
launch notes, so a collective that another TL served (which leaves the note as it was) cannot pass."""
import ctypes as C
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ucc_b200 import capi as U  # noqa: E402
from ucc_b200.dist import Communicator  # noqa: E402
from ucc_b200.harness import coll_args  # noqa: E402

MANAGED, CUDA = U.UCC_MEMORY_TYPE_CUDA_MANAGED, U.UCC_MEMORY_TYPE_CUDA
N = 2
CNT = 1 << 16          # 256 KB of int32 per block: above ZCOPY_THRESH and P2P_RNDV_THRESH, and the staged payload fits the 1 MB heap


class Managed:
    def __init__(self, n, keep):
        hdr = C.c_void_p()
        assert U.lib.ucc_mc_alloc(C.byref(hdr), n * 4, MANAGED) == 0
        keep.append(hdr)
        self.ptr = C.c_void_p.from_address(hdr.value + 8).value
        self.a = np.frombuffer((C.c_char * (n * 4)).from_address(self.ptr), dtype=np.int32)


def main():
    store_path, rank = sys.argv[1], int(sys.argv[2])
    torch.cuda.set_device(0)
    comm = Communicator(store=dist.FileStore(store_path, N), rank=rank, size=N)
    U.lib.ucc_mc_alloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t, C.c_int]
    U.lib.ucc_mc_free.argtypes = [C.c_void_p]
    keep = []

    def run(coll, src, dst, **kw):
        a = coll_args(coll, dt="int32", src_ptr=src.ptr if src is not None else None, dst_ptr=dst.ptr if dst is not None else None,
                      mem_type=MANAGED, **kw)
        torch.cuda.synchronize()
        req = comm.init(a).post()
        req.wait()
        req.finalize()
        torch.cuda.synchronize()
        return comm.request_info_last()

    def data(seed, n):
        return np.random.default_rng(seed).integers(-50, 50, n).astype(np.int32)

    # allreduce: staged two-shot
    src, dst = Managed(CNT * N, keep), Managed(CNT * N, keep)
    src.a[:] = data(rank, CNT * N)
    note = run("allreduce", src, dst, count_src=CNT * N, count_dst=CNT * N)
    assert note.startswith("twoshot_staged"), note
    assert np.array_equal(dst.a, data(0, CNT * N) + data(1, CNT * N)), "allreduce"
    # alltoall: staged pull
    src, dst = Managed(CNT * N, keep), Managed(CNT * N, keep)
    src.a[:] = data(20 + rank, CNT * N)
    note = run("alltoall", src, dst, count_src=CNT * N, count_dst=CNT * N)
    assert note.startswith("exchange_pull_staged"), note
    assert np.array_equal(dst.a, np.concatenate([data(20 + p, CNT * N)[rank * CNT:(rank + 1) * CNT] for p in range(N)])), "alltoall"
    # send / recv 0 -> 1 on managed buffers: the receiver cannot export its buffer, so both sides use the eager ring
    buf = Managed(CNT, keep)
    buf.a[:] = data(30, CNT) if rank == 0 else 0
    note = run("bcast", buf, None, root=0, count_src=CNT, count_dst=0, active_set=(0, 1, 2), tag=5)
    assert note.startswith("p2p_send " if rank == 0 else "p2p_recv "), note
    assert np.array_equal(buf.a, data(30, CNT)), "send / recv"
    # allgather: staged pull
    src, dst = Managed(CNT, keep), Managed(CNT * N, keep)
    src.a[:] = data(10 + rank, CNT)
    note = run("allgather", src, dst, count_src=CNT, count_dst=CNT * N)
    assert note.startswith("exchange_pull_staged"), note
    assert np.array_equal(dst.a, np.concatenate([data(10, CNT), data(11, CNT)])), "allgather"
    # the same allreduce on device tensors still maps the peer's buffer
    t = torch.full((CNT * N,), rank + 1, dtype=torch.int32, device="cuda")
    out = torch.zeros_like(t)
    a = coll_args("allreduce", dt="int32", src_ptr=t.data_ptr(), dst_ptr=out.data_ptr(), count_src=CNT * N, count_dst=CNT * N, mem_type=CUDA)
    torch.cuda.synchronize()
    req = comm.init(a).post()
    req.wait()
    req.finalize()
    torch.cuda.synchronize()
    assert "zcopy" in comm.request_info_last(), comm.request_info_last()
    assert bool((out == 3).all())
    for hdr in keep:
        U.lib.ucc_mc_free(hdr)
    comm.destroy()
    print("MANAGED_IPC_OK", flush=True)


if __name__ == "__main__":
    main()
