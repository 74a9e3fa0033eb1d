"""Worker for test_dist_gpu.py::test_multiproc_symm: allreduce on tensors inside the symmetric user region of the tl/nvl heap
(in-place in-switch reduction, kernels/nvl_symm.cuh).  Also prints the bus bandwidth of a large message next to the default path."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ucc_b200.dist import Communicator, init_distributed  # noqa: E402


def main():
    rank, world, _ = init_distributed("cpu:gloo,cuda:nccl")
    dev = torch.device("cuda", torch.cuda.current_device())
    comm = Communicator(symm_size=os.environ.get("SYMM_SIZE", "1G"))
    ok = True
    reg = comm.symm_region()
    if reg is None or not reg[2]:
        if rank == 0:
            print("SYMM_WORKER_SKIP (no symmetric region / no NVLS on this team)", flush=True)
        comm.destroy()
        dist.destroy_process_group()
        return 0
    for dt, tol in ((torch.float32, 1e-5), (torch.bfloat16, 3e-2), (torch.float16, 1e-2), (torch.int32, 0), (torch.int64, 0)):
        for count in (4, 1000, 262144 + 3, 3000001, 16 * 1024 * 1024):
            comm.symm_reset()
            g = torch.Generator().manual_seed(77 + count)
            alls = [(torch.rand(count, generator=g) * 4 + r).to(dt) for r in range(world)]
            src = comm.symm_empty(count, dt)
            dst = comm.symm_empty(count, dt)
            guard = comm.symm_empty(64, torch.int32)          # must survive: the ragged tail may not write behind dst
            guard.fill_(12345)
            src.copy_(alls[rank].to(dev))
            dst.zero_()
            for inplace in (False, True):
                if inplace:
                    dst.copy_(alls[rank].to(dev))
                torch.cuda.synchronize()
                comm.barrier()
                req = comm.allreduce_init(dst if inplace else src, dst)
                req.post_on_stream()
                req.wait()
                req.finalize()
                torch.cuda.synchronize()
                exp = sum(a.double() for a in alls)
                if not torch.allclose(dst.cpu().double(), exp, rtol=tol * world, atol=tol * world):
                    print(f"rank {rank}: symm allreduce mismatch dt {dt} count {count} inplace {inplace}", flush=True)
                    ok = False
                if not bool((guard == 12345).all()):
                    print(f"rank {rank}: guard behind dst overwritten dt {dt} count {count}", flush=True)
                    ok = False
    # reduce_scatter out of a symmetric source into an ordinary tensor (ZeRO / FSDP gradient shape)
    for dt, tol in ((torch.float32, 1e-5), (torch.bfloat16, 3e-2)):
        for blk in (8, 1000, 262144 + 8):
            comm.symm_reset()
            g = torch.Generator().manual_seed(5 + blk)
            alls = [(torch.rand(blk * world, generator=g) * 4 + r).to(dt) for r in range(world)]
            src = comm.symm_empty(blk * world, dt)
            src.copy_(alls[rank].to(dev))
            dst = torch.zeros(blk, dtype=dt, device=dev)
            torch.cuda.synchronize()
            comm.barrier()
            req = comm.coll_init("reduce_scatter", src, dst)
            req.post_on_stream()
            req.wait()
            req.finalize()
            torch.cuda.synchronize()
            exp = sum(a.double() for a in alls)[rank * blk:(rank + 1) * blk]
            if not torch.allclose(dst.cpu().double(), exp, rtol=tol * world, atol=tol * world):
                print(f"rank {rank}: symm reduce_scatter mismatch dt {dt} blk {blk}", flush=True)
                ok = False
    # allgather into a symmetric destination (multimem.st of every block), plain and in place
    for blk in (4, 1000, 262144 + 4):
        for inplace in (False, True):
            comm.symm_reset()
            dst = comm.symm_empty(blk * world, torch.float32)
            guard = comm.symm_empty(64, torch.int32)
            guard.fill_(777)
            dst.zero_()
            mine = torch.arange(blk, dtype=torch.float32, device=dev) + 1000 * rank
            if inplace:
                dst[rank * blk:(rank + 1) * blk].copy_(mine)
            torch.cuda.synchronize()
            comm.barrier()
            req = comm.coll_init("allgather", None if inplace else mine, dst, inplace=inplace)
            req.post_on_stream()
            req.wait()
            req.finalize()
            torch.cuda.synchronize()
            exp = torch.cat([torch.arange(blk, dtype=torch.float32) + 1000 * r for r in range(world)])
            if not torch.equal(dst.cpu(), exp) or not bool((guard == 777).all()):
                print(f"rank {rank}: symm allgather mismatch blk {blk} inplace {inplace}", flush=True)
                ok = False
    # bandwidth: 1 GiB f32 in place, symmetric vs ordinary tensors
    n = int(os.environ.get("SYMM_BENCH_BYTES", str(1 << 30))) // 4
    comm.symm_reset()
    res = {}
    for name, buf in (("symm", comm.symm_empty(n, torch.float32)), ("plain", torch.empty(n, device=dev))):
        buf.fill_(1.0)
        req = comm.allreduce_init(buf, buf, persistent=True)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for it in range(8):
            if it == 3:
                torch.cuda.synchronize()
                comm.barrier()
                e0.record()
            req.post_on_stream()
            req.wait()
        e1.record()
        torch.cuda.synchronize()
        req.finalize()
        ms = torch.tensor([e0.elapsed_time(e1) / 5])
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        res[name] = 2 * (world - 1) / world * n * 4 / (ms.item() * 1e-3) / 1e9
    flag = torch.tensor([1 if ok else 0])
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print(f"SYMM_BUSBW_GBS symm={res['symm']:.1f} plain={res['plain']:.1f} n_gpus={world}", flush=True)
        print("SYMM_WORKER_OK" if flag.item() == 1 else "SYMM_WORKER_FAIL", flush=True)
    comm.destroy()
    dist.destroy_process_group()
    return 0 if flag.item() == 1 else 1


if __name__ == "__main__":
    sys.exit(main())
