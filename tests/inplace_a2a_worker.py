"""Worker under torchrun: all_to_all_single whose output IS its input, through ucc_b200.ops and through the torch.distributed backend
"ucc_b200", must give the in-place alltoall / alltoallv result.  Host tensors (tl/shm) with "cpu", CUDA tensors (tl/nvl, CUDA IPC
mappings between the processes) with "cuda"."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ucc_b200.torch_backend  # noqa: F401,E402  (registers the backend)
from ucc_b200 import ops  # noqa: E402
from ucc_b200.dist import init_distributed  # noqa: E402


def fill(rank, n, dtype):
    return (torch.arange(n, dtype=torch.float64) % 1000 + 1000 * rank).to(dtype)


def main():
    use_cuda = len(sys.argv) > 1 and sys.argv[1] == "cuda"
    rank, world, _ = init_distributed("cpu:gloo,cuda:nccl" if use_cuda else "gloo")
    dev = torch.device("cuda", torch.cuda.current_device()) if use_cuda else torch.device("cpu")
    pg = dist.new_group(backend="ucc_b200")
    ops.init()
    ok = True
    for blk in (3, 1000, 300001):
        for dtype in (torch.float32, torch.bfloat16):
            for via in ("ops", "backend"):
                allb = [fill(r, blk * world, dtype) for r in range(world)]
                x = allb[rank].to(dev)
                if via == "ops":
                    ops.all_to_all_single(x, x)
                else:
                    dist.all_to_all_single(x, x, group=pg)
                exp = torch.cat([allb[p][rank * blk:(rank + 1) * blk] for p in range(world)])
                if use_cuda:
                    torch.cuda.synchronize()
                if not torch.equal(x.cpu(), exp):
                    print(f"rank {rank}: in-place alltoall mismatch blk {blk} {dtype} via {via}", flush=True)
                    ok = False
        # alltoallv: symmetric split sizes (rows of 2), rank 0 hot, in place
        splits = [[(blk if 0 in (r, p) else blk // 3 + 1) for p in range(world)] for r in range(world)]
        for via in ("ops", "backend"):
            allb = [fill(r, 2 * sum(splits[r]), torch.float32).view(-1, 2) for r in range(world)]
            x = allb[rank].to(dev)
            if via == "ops":
                ops.all_to_all_single(x, x, splits[rank], splits[rank])
            else:
                dist.all_to_all_single(x, x, splits[rank], splits[rank], group=pg)
            offs = [[sum(splits[r][:p]) for p in range(world)] for r in range(world)]
            exp = torch.cat([allb[p][offs[p][rank]:offs[p][rank] + splits[p][rank]] for p in range(world)])
            if use_cuda:
                torch.cuda.synchronize()
            if not torch.equal(x.cpu(), exp):
                print(f"rank {rank}: in-place alltoallv mismatch blk {blk} via {via}", flush=True)
                ok = False
    flag = torch.tensor([1.0 if ok else 0.0])
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("INPLACE_A2A_WORKER_OK" if flag.item() == 1 else "INPLACE_A2A_WORKER_FAIL", flush=True)
    ops.shutdown()
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 1 else 1)


if __name__ == "__main__":
    main()
