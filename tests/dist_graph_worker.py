"""Worker under torchrun for tests/test_dist_graph_gpu.py: the "ucc_b200" torch.distributed backend inside torch.cuda.graph, one
process per GPU.  Warm-up and capture run inside the process group's graphed(); the graph is replayed three times with new inputs
and every result is checked exactly."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ucc_b200.torch_backend  # noqa: F401,E402


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)) % torch.cuda.device_count())
    dist.init_process_group("ucc_b200", rank=rank, world_size=world)
    pg = dist.group.WORLD._get_backend(torch.device("cuda"))
    n = 1 << 20
    ar = torch.zeros(n, device="cuda")
    ag_in, ag_out = torch.zeros(n, device="cuda"), torch.zeros(n * world, device="cuda")
    rs_in, rs_out = torch.zeros(n * world, device="cuda"), torch.zeros(n, device="cuda")
    a2_in, a2_out = torch.zeros(n * world, device="cuda"), torch.zeros(n * world, device="cuda")
    bc = torch.zeros(n, device="cuda")
    snd, rcv = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")

    def step():
        dist.all_reduce(ar)
        dist.all_gather_into_tensor(ag_out, ag_in)
        dist.reduce_scatter_tensor(rs_out, rs_in)
        dist.all_to_all_single(a2_out, a2_in)
        dist.broadcast(bc, src=world - 1)
        reqs = [dist.isend(snd, (rank + 1) % world), dist.irecv(rcv, (rank - 1) % world)]
        for r in reqs:
            r.wait()

    def fill(it):
        base = torch.arange(n, device="cuda", dtype=torch.float32) % 977
        ar.copy_(base + rank + it)
        ag_in.copy_(base * (rank + 1) + it)
        rs_in.copy_(torch.arange(n * world, device="cuda", dtype=torch.float32) % 911 + rank)
        a2_in.copy_(torch.arange(n * world, device="cuda", dtype=torch.float32) % 613 + 1000 * rank + it)
        bc.copy_(base + it if rank == world - 1 else torch.zeros_like(base))
        snd.copy_(base + 10 * rank + it)
        rcv.zero_()

    def check(it):
        base = torch.arange(n, device="cuda", dtype=torch.float32) % 977
        ok = torch.equal(ar, base * world + sum(range(world)) + world * it)
        ok &= all(torch.equal(ag_out[p * n:(p + 1) * n], base * (p + 1) + it) for p in range(world))
        full = torch.arange(n * world, device="cuda", dtype=torch.float32) % 911
        ok &= torch.equal(rs_out, full[rank * n:(rank + 1) * n] * world + sum(range(world)))
        src_all = torch.arange(n * world, device="cuda", dtype=torch.float32) % 613
        ok &= all(torch.equal(a2_out[p * n:(p + 1) * n], src_all[rank * n:(rank + 1) * n] + 1000 * p + it) for p in range(world))
        ok &= torch.equal(bc, base + it)
        ok &= torch.equal(rcv, base + 10 * ((rank - 1) % world) + it)
        return bool(ok)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with pg.graphed():
        with torch.cuda.stream(side):
            for it in range(2):
                fill(it)
                step()
                torch.cuda.current_stream().synchronize()
                assert check(it), ("eager", rank, it)
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
    for it in range(3):
        fill(it)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        assert check(it), ("replay", rank, it)
    del g
    pg.release_graphed()
    dist.destroy_process_group()
    print("DIST_GRAPH_WORKER_OK", flush=True)


if __name__ == "__main__":
    main()
