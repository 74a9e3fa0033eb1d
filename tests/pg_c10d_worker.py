"""Worker under torchrun for tests/test_torch_backend_c10d_cpu.py and tests/test_torch_backend_c10d_gpu.py: the parts of the c10d
surface beyond the basic collectives, called through the public torch.distributed API on the "ucc_b200" backend - gather and
scatter (equal and unequal blocks), list all_to_all, the object collectives, all_gather_coalesced, _coalescing_manager over the
three fast-path collectives, torch.bool tensors, and the errors of what the backend does not serve.  Every result is compared with
a plain torch reference computed on each rank.

argv[1] is "cpu" (host tensors, tl/shm) or "cuda" (all ranks on cuda:<LOCAL_RANK % device count>, tl/nvl).  On CUDA each call must
leave a tl/nvl kernel as this process's last launch, and a gather and a list all_to_all are captured in a CUDA graph and replayed.
Every check runs even when an earlier one failed; each rank prints its failures, and rank 0 prints PG_C10D_WORKER_OK when every
check passed on every rank."""
import os
import sys
import traceback

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ucc_b200.torch_backend  # noqa: F401,E402  (registers the backend)

MOVERS = ("exchange_", "self_copy")                       # launch notes of the tl/nvl data-movement kernels
REDUCERS = ("oneshot", "twoshot", "nvls", "ring", "rhd")   # ... and of its reduction kernels


def val(src, dst, shape, dtype=torch.float32, salt=0):
    """the block rank `src` contributes for rank `dst`: distinct per (src, dst, element)"""
    n = 1
    for d in shape:
        n *= d
    return (torch.arange(n, dtype=torch.float64) + 1000 * src + 100 * dst + salt).reshape(shape).to(dtype)


class Worker:
    def __init__(self, use_cuda):
        self.rank, self.world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
        self.cuda = use_cuda
        if use_cuda:
            torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", self.rank)) % torch.cuda.device_count())
        self.dev = torch.device("cuda", torch.cuda.current_device()) if use_cuda else torch.device("cpu")
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
            if os.environ.get("PG_C10D_TRACE"):
                traceback.print_exc()

    # ---- gather / scatter
    def gather(self, root, sizes, alias):
        """rank p contributes sizes[p] elements; with `alias` the root's own gather_list entry is its input tensor"""
        me, n = self.rank, self.world
        inp = self.on(val(me, root, (sizes[me],), torch.int64))
        outs = [self.on(torch.full((sizes[p],), -1, dtype=torch.int64)) for p in range(n)] if me == root else None
        if alias and me == root:
            outs[root] = inp
        dist.gather(inp, outs, dst=root)
        self.ran(MOVERS, "gather")
        if me == root:
            for p in range(n):
                assert torch.equal(outs[p].cpu(), val(p, root, (sizes[p],), torch.int64)), f"block of rank {p}"

    def scatter(self, root, sizes):
        me, n = self.rank, self.world
        blocks = [self.on(val(root, p, (sizes[p], 2))) for p in range(n)] if me == root else None
        out = self.on(torch.full((sizes[me], 2), -1.0))
        dist.scatter(out, blocks, src=root)
        self.ran(MOVERS, "scatter")
        assert torch.equal(out.cpu(), val(root, me, (sizes[me], 2))), "scattered block"
        if me == root:      # the source list is left as it was
            assert all(torch.equal(blocks[p].cpu(), val(root, p, (sizes[p], 2))) for p in range(n))

    # ---- list all_to_all
    def all_to_all(self, pattern):
        me, n = self.rank, self.world
        size = {"uniform": lambda s, d: 4,
                "skewed": lambda s, d: (s + 2 * d) % 3,                           # zero-sized blocks
                "hot": lambda s, d: 64 if d == 1 % n else 1,                      # one hot receiver
                "idle": lambda s, d: 0 if n - 1 in (s, d) else s + d + 1}[pattern]  # the last rank has nothing to move
        ins = [self.on(val(me, p, (size(me, p), 3), torch.bfloat16)) for p in range(n)]
        outs = [self.on(torch.full((size(p, me), 3), -1.0, dtype=torch.bfloat16)) for p in range(n)]
        dist.all_to_all(outs, ins)
        self.ran(MOVERS, "all_to_all")
        for p in range(n):
            assert torch.equal(outs[p].cpu(), val(p, me, (size(p, me), 3), torch.bfloat16)), f"block from rank {p}"

    # ---- object collectives, all_gather_coalesced
    def objects(self, root):
        me, n = self.rank, self.world
        got = [None] * n if me == root else None
        dist.gather_object({"rank": me, "payload": list(range(me * 7))}, got, dst=root)
        if me == root:
            assert got == [{"rank": p, "payload": list(range(p * 7))} for p in range(n)], got
        recv = [None]
        dist.scatter_object_list(recv, [("to", p, "x" * (3 * p)) for p in range(n)] if me == root else None, src=root)
        assert recv[0] == ("to", me, "x" * (3 * me)), recv

    def all_gather_coalesced(self):
        me, n = self.rank, self.world
        shapes = [(2, 2), (1,), (3,)]
        ins = [self.on(val(me, 0, s, salt=i)) for i, s in enumerate(shapes)]
        outs = [[self.on(torch.zeros(s)) for s in shapes] for _ in range(n)]
        dist.all_gather_coalesced(outs, ins)
        self.ran(MOVERS, "all_gather_coalesced")
        for p in range(n):
            for i, s in enumerate(shapes):
                assert torch.equal(outs[p][i].cpu(), val(p, 0, s, salt=i)), (p, i)

    # ---- _coalescing_manager over the fast-path collectives
    def coalescing(self, coll, async_ops, with_device):
        me, n = self.rank, self.world
        counts = [5, 1, 33]
        if coll == "all_reduce":
            ts = [self.on(val(me, 0, (c,), salt=i)) for i, c in enumerate(counts)]
            exp = [sum(val(p, 0, (c,), torch.float64, salt=i) for p in range(n)).float() for i, c in enumerate(counts)]
        elif coll == "all_gather_into_tensor":
            ins = [self.on(val(me, 0, (c,), salt=i)) for i, c in enumerate(counts)]
            ts = [self.on(torch.zeros(c * n)) for c in counts]
            exp = [torch.cat([val(p, 0, (c,), salt=i) for p in range(n)]) for i, c in enumerate(counts)]
        else:
            ins = [self.on(val(me, 0, (c * n,), salt=i)) for i, c in enumerate(counts)]
            ts = [self.on(torch.zeros(c)) for c in counts]
            exp = [sum(val(p, 0, (c * n,), torch.float64, salt=i) for p in range(n))[me * c:(me + 1) * c].float() for i, c in enumerate(counts)]
        with dist._coalescing_manager(device=self.dev if with_device else None, async_ops=async_ops) as cm:
            for i, t in enumerate(ts):
                if coll == "all_reduce":
                    dist.all_reduce(t)
                elif coll == "all_gather_into_tensor":
                    dist.all_gather_into_tensor(t, ins[i])
                else:
                    dist.reduce_scatter_tensor(t, ins[i])
        if async_ops:
            cm.wait()
        self.ran(REDUCERS if coll != "all_gather_into_tensor" else MOVERS, coll)
        for t, e in zip(ts, exp):
            assert torch.equal(t.cpu(), e), coll

    def coalescing_nested(self):
        self.pg._start_coalescing(self.dev)
        try:
            self.pg._start_coalescing(self.dev)
        except RuntimeError as e:
            assert "coalescing" in str(e), e
        else:
            raise AssertionError("a second _start_coalescing was accepted")
        finally:
            self.pg._end_coalescing(self.dev).wait()

    # ---- torch.bool
    def bool_all_reduce(self, op):
        me, n = self.rank, self.world
        mine = lambda r: torch.tensor([bool((i >> r) & 1) or i == 0 for i in range(2 << n)] * 3)  # noqa: E731  (i = 2^n: false everywhere)
        t = self.on(mine(me))
        dist.all_reduce(t, op=op)
        self.ran(REDUCERS, f"bool all_reduce {op}")
        stack = torch.stack([mine(p) for p in range(n)])
        exp = {dist.ReduceOp.SUM: stack.any(0), dist.ReduceOp.MAX: stack.any(0), dist.ReduceOp.BOR: stack.any(0),
               dist.ReduceOp.PRODUCT: stack.all(0), dist.ReduceOp.MIN: stack.all(0), dist.ReduceOp.BAND: stack.all(0),
               dist.ReduceOp.BXOR: stack.sum(0) % 2 == 1}[op]
        assert t.dtype == torch.bool and torch.equal(t.cpu(), exp), op
        assert exp.any() and not exp.all(), "the pattern must give both values"

    def bool_movement(self):
        me, n = self.rank, self.world
        flags = lambda r: torch.arange(11) % (r + 2) == 0  # noqa: E731
        b = self.on(flags(n - 1) if me == n - 1 else torch.zeros(11, dtype=torch.bool))
        dist.broadcast(b, src=n - 1)
        self.ran(MOVERS, "bool broadcast")
        assert torch.equal(b.cpu(), flags(n - 1)), "broadcast"
        outs = [self.on(torch.zeros(11, dtype=torch.bool)) for _ in range(n)]
        dist.all_gather(outs, self.on(flags(me)))
        self.ran(MOVERS, "bool all_gather")
        assert all(torch.equal(outs[p].cpu(), flags(p)) for p in range(n)), "all_gather"
        big = self.on(torch.zeros(11 * n, dtype=torch.bool))
        dist.all_gather_into_tensor(big, self.on(flags(me)))
        assert torch.equal(big.cpu(), torch.cat([flags(p) for p in range(n)])), "all_gather_into_tensor"

    # ---- what the backend refuses
    def refusals(self):
        t = self.on(torch.ones(4, dtype=torch.bool))
        try:
            dist.all_reduce(t, op=dist.ReduceOp.AVG)
        except ValueError as e:
            assert "AVG" in str(e) and "bool" in str(e), e
        else:
            raise AssertionError("AVG on a bool tensor was accepted")
        for name, call in (("recv_anysource", lambda: dist.recv(self.on(torch.zeros(2)))),
                           ("monitored_barrier", lambda: self.pg.monitored_barrier()),
                           ("split_group", lambda: self.pg.split_group([0]))):
            try:
                call()
            except RuntimeError as e:
                assert name in str(e), e
            else:
                raise AssertionError(f"{name} was accepted")

    def graphed_lockstep(self):
        """Inside graphed() the requests are cached by their buffers, and every rank must create a new one or re-post a cached one in
        step with the others (on CUDA the zero-copy exchange is matched by post order).  Same user tensors on every call: after each
        call every rank holds as many cached requests as the others."""
        me, n, root = self.rank, self.world, self.world - 1
        g_in, g_out = self.on(val(me, root, (6,))), [self.on(torch.zeros(6)) for _ in range(n)] if me == root else None
        s_in, s_out = [self.on(val(root, p, (6,))) for p in range(n)] if me == root else None, self.on(torch.zeros(6))
        a_in, a_out = [self.on(val(me, p, (p + 1,))) for p in range(n)], [self.on(torch.zeros(me + 1)) for _ in range(n)]
        with self.pg.graphed():
            for it in range(3):
                dist.gather(g_in, g_out, dst=root)
                dist.scatter(s_out, s_in, src=root)
                dist.all_to_all(a_out, a_in)
                held = [None] * n
                dist.all_gather_object(held, len(self.pg._comm._graph_reqs))
                assert len(set(held)) == 1, f"call {it}: cached requests per rank {held}"
        self.pg.release_graphed()
        if me == root:
            assert all(torch.equal(g_out[p].cpu(), val(p, root, (6,))) for p in range(n)), "gather"
        assert torch.equal(s_out.cpu(), val(root, me, (6,))), "scatter"
        assert all(torch.equal(a_out[p].cpu(), val(p, me, (me + 1,))) for p in range(n)), "all_to_all"

    # ---- CUDA graph: gather and list all_to_all captured inside pg.graphed(), replayed with new inputs
    def graph(self):
        me, n, root = self.rank, self.world, self.world - 1
        size = lambda s, d: (s + d) % 3 * 1000 + 1  # noqa: E731
        g_in = self.on(torch.zeros(4096))
        g_out = [self.on(torch.zeros(4096)) for _ in range(n)] if me == root else None
        a_in = [self.on(torch.zeros(size(me, p))) for p in range(n)]
        a_out = [self.on(torch.zeros(size(p, me))) for p in range(n)]

        def step():
            dist.gather(g_in, g_out, dst=root)
            dist.all_to_all(a_out, a_in)

        def fill(it):
            g_in.copy_(val(me, root, (4096,), salt=it))
            for p in range(n):
                a_in[p].copy_(val(me, p, (size(me, p),), salt=it))

        def check(it, what):
            torch.cuda.current_stream().synchronize()
            if me == root:
                assert all(torch.equal(g_out[p].cpu(), val(p, root, (4096,), salt=it)) for p in range(n)), f"{what} gather {it}"
            assert all(torch.equal(a_out[p].cpu(), val(p, me, (size(p, me),), salt=it)) for p in range(n)), f"{what} all_to_all {it}"

        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with self.pg.graphed():
            with torch.cuda.stream(side):
                for it in range(2):
                    fill(it)
                    step()
                    check(it, "warm-up")
            torch.cuda.current_stream().wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                step()
        for it in range(10, 13):
            fill(it)
            g.replay()
            check(it, "replay")
        assert not self.pg._comm.take_device_error()
        del g
        self.pg.release_graphed()

    def run(self):
        n, last = self.world, self.world - 1
        equal, unequal = [5] * n, [(p * 2 + 1) % 4 for p in range(n)]   # unequal: (1, 3, 1, 3 ...) and a zero from rank 2 on
        unequal[min(2, last)] = 0
        for root in (0, last):
            for sizes in (equal, unequal):
                self.case("gather", self.gather, root, sizes, False)
                self.case("scatter", self.scatter, root, sizes)
            self.case("gather", self.gather, root, equal, True)
            self.case("objects", self.objects, root)
        for pattern in ("uniform", "skewed", "hot", "idle"):
            self.case("all_to_all", self.all_to_all, pattern)
        self.case("all_gather_coalesced", self.all_gather_coalesced)
        for coll in ("all_reduce", "all_gather_into_tensor", "reduce_scatter_tensor"):
            for async_ops in (False, True):
                for with_device in (True, False):
                    self.case("coalescing", self.coalescing, coll, async_ops, with_device)
        self.case("coalescing_nested", self.coalescing_nested)
        for op in (dist.ReduceOp.SUM, dist.ReduceOp.PRODUCT, dist.ReduceOp.MAX, dist.ReduceOp.MIN, dist.ReduceOp.BAND,
                   dist.ReduceOp.BOR, dist.ReduceOp.BXOR):
            self.case("bool_all_reduce", self.bool_all_reduce, op)
        self.case("bool_movement", self.bool_movement)
        self.case("refusals", self.refusals)
        self.case("graphed_lockstep", self.graphed_lockstep)
        if self.cuda:
            self.case("graph", self.graph)
        for f in self.fails:
            print(f"PG_C10D_FAIL rank {self.rank}: {f}", flush=True)
        flag = self.on(torch.tensor([0.0 if self.fails else 1.0]))
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        ok = flag.item() == 1
        if self.rank == 0:
            print(f"PG_C10D_WORKER_{'OK' if ok else 'FAIL'} world {n} checks {self.passed + len(self.fails)} passed {self.passed}", flush=True)
        dist.destroy_process_group()
        return ok


if __name__ == "__main__":
    sys.exit(0 if Worker(len(sys.argv) > 1 and sys.argv[1] == "cuda").run() else 1)
