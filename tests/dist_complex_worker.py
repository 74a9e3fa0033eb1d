"""Worker run under torchrun by tests/test_dist_complex_gpu.py: complex allreduce through ucc_b200.dist, one process per GPU.
Gaussian-integer inputs with components in {-2..2} keep SUM and PROD exact, so results are compared for equality."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ucc_b200.dist import Communicator, init_distributed  # noqa: E402


def gauss(n, seed, dt):
    g = torch.Generator().manual_seed(seed)
    return torch.complex(*(torch.randint(-2, 3, (n,), generator=g).double() for _ in range(2))).to(dt)


def main():
    dt, op = {"c64": torch.complex64, "c128": torch.complex128}[sys.argv[1]], sys.argv[2]
    rank, world, _ = init_distributed("cpu:gloo,cuda:nccl")
    dev = torch.device("cuda", torch.cuda.current_device())
    comm = Communicator()
    ok = True
    for count in (1, 1000, 100001, 3000001):
        alls = [gauss(count, 17 * r + count, dt) for r in range(world)]
        dst = torch.zeros(count, dtype=dt, device=dev)
        req = comm.allreduce_init(alls[rank].to(dev), dst, op=op)
        req.post_on_stream()
        req.wait()
        req.finalize()
        torch.cuda.synchronize()
        exp = alls[0].to(torch.complex128)
        for a in alls[1:]:
            exp = exp * a.to(torch.complex128) if op == "prod" else exp + a.to(torch.complex128)
        if not torch.equal(dst.cpu().to(torch.complex128), exp):
            print(f"rank {rank}: {sys.argv[1]} {op} allreduce mismatch at count {count}", flush=True)
            ok = False
    comm.barrier()
    flag = torch.tensor([1 if ok else 0])
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    comm.destroy()
    if rank == 0:
        print("DIST_COMPLEX_OK" if flag.item() == 1 else "DIST_COMPLEX_FAIL", flush=True)
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 1 else 1)


if __name__ == "__main__":
    main()
