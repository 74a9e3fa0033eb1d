"""Worker under torchrun for tests/test_torch_native_cpu.py and tests/test_torch_native_gpu.py: PyTorch's own parallel stack on the
"ucc_b200" backend - functional collectives (eager and under torch.compile), DeviceMesh / DTensor redistribution, FSDP2
(fully_shard, HSDP) and tensor parallelism - plus the list forms of all_gather / reduce_scatter with blocks of different sizes, the
stream order Work.wait() gives across streams, and the refusal of PREMUL_SUM.

argv[1] is "cpu" (host tensors, tl/shm) or "cuda" (rank r on cuda:<LOCAL_RANK % device count>, tl/nvl); argv[2] is a comma-separated
list of sections (funcol, dtensor, fsdp, tp, uneven, stream, refusals).  On CUDA every direct collective must leave a tl/nvl kernel
as this process's last launch.  Collectives and their references use integer-valued data, so the sums are exact in any order and
compare bitwise; only the training runs (FSDP2, tensor parallel) compare to a tolerance.  Every check runs even when an earlier
one failed; each rank prints its failures, and rank 0 prints TORCH_NATIVE_OK when every check passed on every rank."""
import os
import sys
import traceback

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ucc_b200.torch_backend  # noqa: F401,E402  (registers the backend)

MOVERS = ("exchange_", "self_copy")                       # launch notes of the tl/nvl data-movement kernels
REDUCERS = ("oneshot", "twoshot", "nvls", "ring", "rhd")   # ... and of its reduction kernels


def ints(shape, seed, scale=1, dtype=torch.float32):
    """integer values in [-8, 8] times `scale`, the same for a seed on every rank"""
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(-8, 9, shape, generator=g) * scale).to(dtype)


class Worker:
    def __init__(self, use_cuda):
        self.rank, self.world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
        self.cuda = use_cuda
        if use_cuda:
            torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", self.rank)) % torch.cuda.device_count())
        self.dev = torch.device("cuda", torch.cuda.current_device()) if use_cuda else torch.device("cpu")
        self.dtype = self.dev.type
        dist.init_process_group("ucc_b200", rank=self.rank, world_size=self.world)
        self.pg = dist.group.WORLD
        self.fails = []
        self.passed = 0

    def on(self, t):
        return t.to(self.dev)

    def ran(self, kinds, what):
        """on CUDA: the call launched a tl/nvl kernel of `kinds` (it did not go to a host transport)"""
        if self.cuda:
            note = self.pg._comm.request_info_last()
            assert note.startswith(kinds), f"{what}: last tl/nvl launch is {note!r}"

    def case(self, name, fn, *args):
        try:
            fn(*args)
            if self.cuda:
                torch.cuda.current_stream().synchronize()
            self.passed += 1
        except Exception as e:  # noqa: BLE001  (every failure is reported, then the next check runs)
            self.fails.append(f"{name}{args}: {type(e).__name__}: {e}")
            if os.environ.get("TORCH_NATIVE_TRACE"):
                traceback.print_exc()

    def same(self, got, exp, what):
        got = got.cpu()
        assert got.dtype == exp.dtype and got.shape == exp.shape and torch.equal(got, exp), \
            f"{what}: {got.dtype} {tuple(got.shape)} vs {exp.dtype} {tuple(exp.shape)}, max diff {(got.double() - exp.double()).abs().max() if got.shape == exp.shape else '-'}"

    # ---- functional collectives
    def a2a_size(self, s, d):
        return (s + 2 * d) % 3 + (s == d)     # blocks of 0, 1, 2 and 3 rows

    def funcol_inputs(self, r):
        n = self.world
        return (ints((5, 3), 10 + r, scale=n),                                            # all_reduce (sum, avg), all_gather
                ints((4 * n, 3), 20 + r),                                                  # reduce_scatter
                torch.cat([ints((self.a2a_size(r, p), 2), 100 * r + p) for p in range(n)]))  # all_to_all_single

    def funcol_refs(self):
        me, n = self.rank, self.world
        xs, ys, zs = zip(*(self.funcol_inputs(r) for r in range(n)))
        a2a = torch.cat([zs[p][sum(self.a2a_size(p, q) for q in range(me)):][:self.a2a_size(p, me)] for p in range(n)])
        return [sum(xs), sum(xs) / n, torch.cat(xs), sum(ys)[4 * me:4 * me + 4], a2a]

    def funcol_fn(self):
        import torch.distributed._functional_collectives as funcol
        me, n, group = self.rank, self.world, dist.group.WORLD
        out_splits = [self.a2a_size(p, me) for p in range(n)]
        in_splits = [self.a2a_size(me, p) for p in range(n)]

        def fn(x, y, z):
            outs = (funcol.all_reduce(x, "sum", group), funcol.all_reduce(x, "avg", group), funcol.all_gather_tensor(x, 0, group),
                    funcol.reduce_scatter_tensor(y, "sum", 0, group), funcol.all_to_all_single(z, out_splits, in_splits, group))
            return [funcol.wait_tensor(t) for t in outs]
        return fn

    def funcol_eager(self):
        import torch.distributed._functional_collectives as funcol
        me, n, group = self.rank, self.world, dist.group.WORLD
        assert isinstance(self.pg.group_name, str) and self.pg.group_name, self.pg.group_name
        assert dist.distributed_c10d._resolve_process_group(self.pg.group_name) is self.pg, "the group does not resolve by its name"
        x, y, z = (self.on(t) for t in self.funcol_inputs(me))
        exp = self.funcol_refs()
        calls = [("all_reduce sum", REDUCERS, lambda: funcol.all_reduce(x, "sum", group)),
                 ("all_reduce avg", REDUCERS, lambda: funcol.all_reduce(x, "avg", group)),
                 ("all_gather_tensor", MOVERS, lambda: funcol.all_gather_tensor(x, 0, group)),
                 ("reduce_scatter_tensor", REDUCERS, lambda: funcol.reduce_scatter_tensor(y, "sum", 0, group)),
                 ("all_to_all_single", MOVERS, lambda: funcol.all_to_all_single(z, [self.a2a_size(p, me) for p in range(n)],
                                                                                   [self.a2a_size(me, p) for p in range(n)], group))]
        for (what, kinds, call), e in zip(calls, exp):
            got = funcol.wait_tensor(call())
            self.ran(kinds, what)
            self.same(got, e, what)
        for what, got, e in zip(("sum", "avg", "all_gather", "reduce_scatter", "all_to_all"), self.funcol_fn()(x, y, z), exp):
            self.same(got, e, f"together: {what}")

    def funcol_compiled(self):
        torch._dynamo.reset()
        fn = torch.compile(self.funcol_fn(), fullgraph=True, backend="aot_eager")
        x, y, z = (self.on(t) for t in self.funcol_inputs(self.rank))
        for it in range(2):
            got = fn(x, y, z)
            self.ran(MOVERS + REDUCERS, "compiled")
            for what, g, e in zip(("sum", "avg", "all_gather", "reduce_scatter", "all_to_all"), got, self.funcol_refs()):
                self.same(g, e, f"compiled call {it}: {what}")

    # ---- DeviceMesh / DTensor
    def dtensor_1d(self):
        from torch.distributed.device_mesh import init_device_mesh
        from torch.distributed.tensor import Partial, Replicate, Shard, distribute_tensor, DTensor
        n, me = self.world, self.rank
        mesh = init_device_mesh(self.dtype, (n,))
        full = ints((7, 2 * n), 1, scale=n)             # 7 rows: not divisible by the mesh size
        places = [Shard(0), Shard(1), Replicate()]
        for src in places:
            for dst in places:
                d = distribute_tensor(self.on(full), mesh, [src]).redistribute(mesh, [dst])
                self.same(d.full_tensor(), full, f"{src} -> {dst}")
                exp = full if isinstance(dst, Replicate) else (list(full.chunk(n, dst.dim)) + [full[:0]] * n)[me]
                if isinstance(dst, Shard) and exp.numel() == 0:
                    exp = full.narrow(dst.dim, 0, 0)
                self.same(d.to_local(), exp.contiguous(), f"{src} -> {dst}: local")
        parts = [ints((7, 2 * n), 40 + r, scale=n) for r in range(n)]
        for red, exp in (("sum", sum(parts)), ("avg", sum(parts) / n)):
            for dst in places:
                d = DTensor.from_local(self.on(parts[me]), mesh, [Partial(red)]).redistribute(mesh, [dst])
                self.same(d.full_tensor(), exp, f"Partial({red}) -> {dst}")

    def dtensor_2d(self):
        from torch.distributed.device_mesh import init_device_mesh
        from torch.distributed.tensor import Partial, Replicate, Shard, distribute_tensor, DTensor
        import torch.distributed._functional_collectives as funcol
        n, me = self.world, self.rank
        mesh = init_device_mesh(self.dtype, (2, n // 2), mesh_dim_names=("dp", "tp"))
        full = ints((6, 5), 2, scale=n)                  # 5 columns: not divisible by either mesh dimension
        for src, dst in (([Shard(0), Shard(1)], [Replicate(), Replicate()]), ([Replicate(), Shard(1)], [Shard(1), Shard(0)]),
                         ([Shard(1), Replicate()], [Replicate(), Shard(1)]), ([Shard(0), Shard(0)], [Shard(1), Replicate()])):
            d = distribute_tensor(self.on(full), mesh, src).redistribute(mesh, dst)
            self.same(d.full_tensor(), full, f"{src} -> {dst}")
        parts = [ints((6, 5), 50 + r, scale=n) for r in range(n)]
        coord = mesh.get_coordinate()
        for red in ("sum", "avg"):
            # Partial on the tp dimension only: the sum runs over the ranks of this rank's tp group
            tp_ranks = [r for r in range(n) if r // (n // 2) == coord[0]]
            exp = sum(parts[r] for r in tp_ranks) / (len(tp_ranks) if red == "avg" else 1)
            for dst in (Replicate(), Shard(0), Shard(1)):
                d = DTensor.from_local(self.on(parts[me]), mesh, [Replicate(), Partial(red)]).redistribute(mesh, [Replicate(), dst])
                self.same(d.full_tensor(), exp, f"Partial({red}) on tp -> {dst}")
        # an all_reduce on one mesh dimension
        x = self.on(parts[me])
        got = funcol.wait_tensor(funcol.all_reduce(x, "sum", (mesh, 1)))
        self.ran(REDUCERS, "all_reduce on mesh dimension tp")
        self.same(got, sum(parts[r] for r in range(n) if r // (n // 2) == coord[0]), "all_reduce on mesh dimension tp")
        dp = mesh.get_group("dp")
        assert isinstance(dp.group_name, str) and dp.group_name != self.pg.group_name, dp.group_name
        y = self.on(parts[me].clone())
        dist.all_reduce(y, group=dp)
        self.ran(REDUCERS, "all_reduce on mesh dimension dp")
        self.same(y, sum(parts[r] for r in range(n) if r % (n // 2) == coord[1]), "all_reduce on mesh dimension dp")

    # ---- FSDP2 and tensor parallel: a few SGD steps against one process on the concatenated batch
    def mlp(self, hidden):
        torch.manual_seed(0)
        return torch.nn.Sequential(torch.nn.Linear(8, hidden), torch.nn.ReLU(), torch.nn.Linear(hidden, 4)).to(self.dev)

    def batch(self, step, rows):
        return self.on(torch.randn(rows, 8, generator=torch.Generator().manual_seed(step))), \
            self.on(torch.randn(rows, 4, generator=torch.Generator().manual_seed(1000 + step)))

    def fsdp(self, mixed, hsdp):
        from torch.distributed.device_mesh import init_device_mesh
        from torch.distributed.fsdp import MixedPrecisionPolicy, fully_shard
        n, me, rows = self.world, self.rank, 3
        model, ref = self.mlp(20), self.mlp(20)         # 20 rows of the first weight: not divisible by 3
        mesh = init_device_mesh(self.dtype, (2, n // 2), mesh_dim_names=("replicate", "shard")) if hsdp else init_device_mesh(self.dtype, (n,))
        kw = {"mesh": mesh}
        if mixed:
            kw["mp_policy"] = MixedPrecisionPolicy(param_dtype=torch.bfloat16, reduce_dtype=torch.float32)
        for layer in (model[0], model[2]):
            fully_shard(layer, **kw)
        fully_shard(model, **kw)
        opt, ref_opt = torch.optim.SGD(model.parameters(), lr=0.1), torch.optim.SGD(ref.parameters(), lr=0.1)
        for step in range(3):
            x, y = self.batch(step, rows * n)
            loss = torch.nn.functional.mse_loss(model(x[me * rows:(me + 1) * rows]).float(), y[me * rows:(me + 1) * rows])
            loss.backward()
            opt.step()
            opt.zero_grad()
            torch.nn.functional.mse_loss(ref(x), y).backward()
            ref_opt.step()
            ref_opt.zero_grad()
        tol = {"rtol": 2e-2, "atol": 2e-2} if mixed else {"rtol": 1e-5, "atol": 1e-6}
        for (name, p), q in zip(model.named_parameters(), ref.parameters()):
            full = p.full_tensor().cpu()
            assert full.dtype == torch.float32 and torch.allclose(full, q.detach().cpu(), **tol), \
                f"{name}: max diff {(full - q.detach().cpu()).abs().max()}"
            assert not torch.equal(q.detach().cpu(), self.mlp(20).state_dict()[name].cpu()), f"{name} did not train"

    def tp(self):
        from torch.distributed.device_mesh import init_device_mesh
        from torch.distributed.tensor.parallel import ColwiseParallel, RowwiseParallel, parallelize_module
        n = self.world
        model, ref = self.mlp(4 * n), self.mlp(4 * n)
        parallelize_module(model, init_device_mesh(self.dtype, (n,)), {"0": ColwiseParallel(), "2": RowwiseParallel()})
        x, _ = self.batch(7, 5)
        out, ref_out = model(x), ref(x)
        assert torch.allclose(out.cpu(), ref_out.detach().cpu(), rtol=1e-5, atol=1e-6), f"forward: max diff {(out - ref_out).abs().max()}"
        out.square().sum().backward()
        ref_out.square().sum().backward()
        for (name, p), q in zip(model.named_parameters(), ref.parameters()):
            g = p.grad.full_tensor().cpu()
            assert torch.allclose(g, q.grad.cpu(), rtol=1e-5, atol=1e-6), f"grad of {name}: max diff {(g - q.grad.cpu()).abs().max()}"

    # ---- list all_gather / reduce_scatter with blocks of different sizes
    def spy(self):
        """the collectives the next calls post, by name"""
        posted, comm = [], self.pg._comm
        orig = comm.coll_init

        def coll_init(coll, *a, **kw):
            posted.append(coll)
            return orig(coll, *a, **kw)
        comm.coll_init = coll_init
        return posted, lambda: setattr(comm, "coll_init", orig)

    def sizes(self, kind):
        n = self.world
        return {"equal": [3] * n, "rank+1": [p + 1 for p in range(n)], "zero": [0 if p == 1 else p + 2 for p in range(n)],
                "all_zero_but_last": [0] * (n - 1) + [5]}[kind]

    def all_gather_list(self, kind):
        me, n = self.rank, self.world
        size = self.sizes(kind)
        outs = [self.on(torch.full((size[p],), -1, dtype=torch.int64)) for p in range(n)]
        posted, restore = self.spy()
        try:
            dist.all_gather(outs, self.on(torch.arange(size[me], dtype=torch.int64) + 100 * me))
        finally:
            restore()
        assert posted == ["allgather" if kind == "equal" else "allgatherv"], posted
        self.ran(MOVERS, "all_gather")
        for p in range(n):
            self.same(outs[p], torch.arange(size[p], dtype=torch.int64) + 100 * p, f"block of rank {p}")

    def all_gather_coalesced(self):
        me, n = self.rank, self.world
        shape = lambda r, i: (r + i + 1, 2) if i else (3,)  # noqa: E731  (input 0: the same everywhere, input 1: per rank)
        ins = [self.on(ints(shape(me, i), 60 + 10 * me + i)) for i in range(2)]
        outs = [[self.on(torch.zeros(shape(p, i))) for i in range(2)] for p in range(n)]
        posted, restore = self.spy()
        try:
            dist.all_gather_coalesced(outs, ins)
        finally:
            restore()
        assert posted == ["allgather", "allgatherv"], posted
        for p in range(n):
            for i in range(2):
                self.same(outs[p][i], ints(shape(p, i), 60 + 10 * p + i), f"input {i} of rank {p}")

    def reduce_scatter_list(self, kind, op):
        me, n = self.rank, self.world
        size = self.sizes(kind)
        ins = [self.on(ints((size[p],), 70 + 10 * me + p, scale=n)) for p in range(n)]
        out = self.on(torch.full((size[me],), -1.0))
        posted, restore = self.spy()
        try:
            dist.reduce_scatter(out, ins, op=op)
        finally:
            restore()
        assert posted == ["reduce_scatter" if kind == "equal" else "reduce_scatterv"], posted
        if size[me]:
            self.ran(REDUCERS, "reduce_scatter")
        exp = sum(ints((size[me],), 70 + 10 * r + me, scale=n) for r in range(n))
        self.same(out, exp / n if op == dist.ReduceOp.AVG else exp, "reduce_scatter")

    # ---- Work.wait() across streams: the collective waits behind a delay kernel on a side stream, the caller reads on its own
    def cross_stream(self, count, how):
        me, n = self.rank, self.world
        x = self.on(torch.empty(count))
        side = torch.cuda.Stream()
        # The first round, with a short delay, loads every kernel involved: loading a module synchronizes the device, which would
        # hide a missing stream order in the second round.  The second delay is ~50 ms at the H100's clock, a bounded wait.
        for delay in (1000, 100_000_000):
            x.fill_(me + 1)
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                torch.cuda._sleep(delay)
                w = dist.all_reduce(x, async_op=True)
            self.ran(REDUCERS, "all_reduce")
            if how == "wait":
                w.wait()
            else:
                assert w.get_future().wait()[0] is x
            y = x * 2                           # on the default stream: must see the reduced values
            exp = float(n * (n + 1))
            assert torch.equal(y.cpu(), torch.full((count,), exp)), \
                f"delay {delay}: read {y[:4].tolist()} ... on the waiting stream, expected {exp}"
            torch.cuda.synchronize()

    # ---- refusals
    def refusals(self):
        t = self.on(torch.ones(4))
        try:
            dist.all_reduce(t, op=dist._make_nccl_premul_sum(0.5))
        except (ValueError, RuntimeError) as e:
            assert "PREMUL_SUM" in str(e), e
        else:
            raise AssertionError("PREMUL_SUM was accepted")

    def run(self, sections):
        n = self.world
        if "funcol" in sections:
            self.case("funcol_eager", self.funcol_eager)
            self.case("funcol_compiled", self.funcol_compiled)
        if "dtensor" in sections:
            self.case("dtensor_1d", self.dtensor_1d)
            if n == 4:
                self.case("dtensor_2d", self.dtensor_2d)
        if "fsdp" in sections:
            for mixed in (False, True):
                self.case("fsdp", self.fsdp, mixed, False)
            if n == 4:
                self.case("hsdp", self.fsdp, False, True)
        if "tp" in sections:
            self.case("tp", self.tp)
        if "uneven" in sections:
            for kind in ("equal", "rank+1", "zero", "all_zero_but_last"):
                self.case("all_gather_list", self.all_gather_list, kind)
                for op in (dist.ReduceOp.SUM, dist.ReduceOp.AVG):
                    self.case("reduce_scatter_list", self.reduce_scatter_list, kind, op)
            self.case("all_gather_coalesced", self.all_gather_coalesced)
        if "stream" in sections and self.cuda:
            for count in (4096, 1 << 20):       # 16 KB and 4 MB: below and above tl/nvl's zero-copy threshold (1 MB)
                for how in ("wait", "future"):
                    self.case("cross_stream", self.cross_stream, count, how)
        if "refusals" in sections:
            self.case("refusals", self.refusals)
        for f in self.fails:
            print(f"TORCH_NATIVE_FAIL rank {self.rank}: {f}", flush=True)
        flag = self.on(torch.tensor([0.0 if self.fails else 1.0]))
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        ok = flag.item() == 1
        if self.rank == 0:
            print(f"TORCH_NATIVE_{'OK' if ok else 'FAIL'} world {n} sections {','.join(sections)} checks {self.passed + len(self.fails)} "
                  f"passed {self.passed}", flush=True)
        dist.destroy_process_group()
        return ok


if __name__ == "__main__":
    sys.exit(0 if Worker(sys.argv[1] == "cuda").run(sys.argv[2].split(",")) else 1)
