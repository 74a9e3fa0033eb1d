"""Worker of tests/test_nvl_graph_gpu.py::test_graphed_direct_two_processes_one_gpu: one of two processes on the same GPU
(argv: store file, rank).  Communicator.graphed() warms up and captures a 4 MB allreduce, which runs the zero-copy form through
CUDA IPC mappings of the peer's buffer; then more distinct peer allocations than the tl/nvl mapping cache holds go through eager
zero-copy allreduces, and the graph must still replay exactly.  Run with PYTORCH_NO_CUDA_MEMORY_CACHING=1, so that every tensor
is an allocation of its own."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ucc_b200 import ops  # noqa: E402
from ucc_b200.dist import Communicator  # noqa: E402


def main():
    store_path, rank = sys.argv[1], int(sys.argv[2])
    torch.cuda.set_device(0)
    comm = Communicator(store=dist.FileStore(store_path, 2), rank=rank, size=2)
    n = 1 << 20                                    # 4 MB: above UCC_TL_NVL_ZCOPY_THRESH
    x = torch.zeros(n, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with comm.graphed():
        with torch.cuda.stream(side):
            for _ in range(2):
                ops.all_reduce(x, comm=comm)
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            ops.all_reduce(x, comm=comm)
        note = comm.request_info_last()
    assert "zcopy" in note, note

    def replay_and_check(it):
        base = torch.arange(n, device="cuda", dtype=torch.float32) % 1000
        x.copy_(base * (rank + 1) + it)
        g.replay()
        torch.cuda.synchronize()
        exp = base * 3 + 2 * it
        assert torch.equal(x, exp), (rank, it)
    for it in range(3):
        replay_and_check(it)
    keep = []
    for k in range(80):                            # distinct allocations, each mapped by the peer
        t = torch.full((n,), float(k + rank), device="cuda")
        ops.all_reduce(t, comm=comm)
        assert "zcopy" in comm.request_info_last(), comm.request_info_last()
        assert bool((t == 2 * k + 1).all()), (rank, k)
        keep.append(t)
    for it in range(3, 6):
        replay_and_check(it)
    assert not comm.take_device_error()
    del g
    comm.destroy()
    print("GRAPH_IPC_OK", flush=True)


if __name__ == "__main__":
    main()
