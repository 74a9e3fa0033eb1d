"""Worker under torchrun for tests/test_nvl_overlap_gpu.py::test_overlap_torch_two_processes: two processes (rank r on cuda:<r % device
count>, so one GPU serves both and the buffers cross the exchange board as CUDA IPC handles) on the "ucc_b200" backend.  Every
collective of the torch API runs twice on the same inputs, on the group without and with set_overlap_gpu(True); the two results
must be bitwise equal, and the hinted large ones must have run the copy-engine direct form (the launch note).  Then an FSDP2
fully_shard model trains three steps on the hinted group and a copy of it on the plain group: the parameters must end bitwise
equal.  Rank 0 prints OVERLAP_TORCH_OK when every check passed on every rank."""
import os
import sys
import traceback

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ucc_b200.torch_backend  # noqa: F401,E402  (registers the backend)

CE = ("reduce_copy_engine", "exchange_copy_engine", "exchange_push_copy_engine")


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(rank % torch.cuda.device_count())
    dev = torch.device("cuda", torch.cuda.current_device())
    dist.init_process_group("ucc_b200", rank=rank, world_size=world)
    pg = dist.group.WORLD
    fails = []

    def data(n, seed, dtype=torch.float32):
        g = torch.Generator().manual_seed(seed)
        return torch.randn(n, generator=g).to(dtype).to(dev)

    def both(name, fn, n):
        """fn(hinted) -> output tensor; run without and with the hint, compare bitwise, check the hinted note"""
        try:
            pg.set_overlap_gpu(False)
            ref = fn(False).clone()
            note_ref = pg._comm.request_info_last()
            pg.set_overlap_gpu(True)
            got = fn(True)
            note = pg._comm.request_info_last()
            pg.set_overlap_gpu(False)
            torch.cuda.synchronize()
            assert torch.equal(ref.view(torch.int32), got.view(torch.int32)), f"{name}: results differ ({note_ref} / {note})"
            if n * 4 >= (1 << 20):
                assert note.startswith(CE), f"{name}: hinted request served by {note!r}"
        except Exception as e:  # noqa: BLE001
            fails.append(f"{name}: {type(e).__name__}: {e}\n{traceback.format_exc()[-1500:]}")

    for n in (1000, 1 << 20):
        x = data(n, rank)

        def ar(_):
            t = x.clone()
            dist.all_reduce(t)
            return t

        def rs(_):
            out = torch.empty(n // world, device=dev)
            dist.reduce_scatter_tensor(out, x)
            return out

        def ag(_):
            out = torch.empty(n * world, device=dev)
            dist.all_gather_into_tensor(out, x)
            return out

        def bc(_):
            t = x.clone()
            dist.broadcast(t, src=1)
            return t

        def a2a(_):
            out = torch.empty(n, device=dev)
            dist.all_to_all_single(out, x)
            return out

        def ga(_):
            outs = [torch.empty(n, device=dev) for _ in range(world)] if rank == 0 else None
            dist.gather(x, outs, dst=0)
            return torch.cat(outs) if rank == 0 else x

        def sc(_):
            out = torch.empty(n // world, device=dev)
            dist.scatter(out, list(x.chunk(world)) if rank == 1 else None, src=1)
            return out

        for name, fn in (("all_reduce", ar), ("reduce_scatter_tensor", rs), ("all_gather_into_tensor", ag), ("broadcast", bc),
                         ("all_to_all_single", a2a), ("gather", ga), ("scatter", sc)):
            both(f"{name} n={n}", fn, n)

    # FSDP2: the same model trained on the hinted and on the plain group ends with the same bits
    try:
        from torch.distributed.device_mesh import init_device_mesh
        from torch.distributed.fsdp import fully_shard
        mesh = init_device_mesh("cuda", (world,))
        params = []
        for overlap in (False, True):
            torch.manual_seed(0)
            model = torch.nn.Sequential(torch.nn.Linear(64, 300), torch.nn.ReLU(), torch.nn.Linear(300, 8)).to(dev)
            for layer in (model[0], model[2]):
                fully_shard(layer, mesh=mesh)
            fully_shard(model, mesh=mesh)
            mesh.get_group().set_overlap_gpu(overlap)
            opt = torch.optim.SGD(model.parameters(), lr=0.1)
            for step in range(3):
                g = torch.Generator().manual_seed(100 * step + rank)
                xb, yb = torch.randn(16, 64, generator=g).to(dev), torch.randn(16, 8, generator=g).to(dev)
                torch.nn.functional.mse_loss(model(xb), yb).backward()
                opt.step()
                opt.zero_grad()
            params.append([p.full_tensor().detach().cpu() for p in model.parameters()])
            mesh.get_group().set_overlap_gpu(False)
        for a, b in zip(*params):
            assert torch.equal(a, b), "FSDP2 parameters differ between the plain and the hinted group"
    except Exception as e:  # noqa: BLE001
        fails.append(f"fsdp2: {type(e).__name__}: {e}\n{traceback.format_exc()[-1500:]}")

    for f in fails:
        print(f"rank {rank}: FAIL {f}", flush=True)
    ok = torch.tensor([0 if fails else 1], device=dev)
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    if rank == 0 and ok.item() == 1:
        print("OVERLAP_TORCH_OK", flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
