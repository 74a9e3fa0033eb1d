"""Worker under torchrun for tests/test_torch_float8_cpu.py and tests/test_torch_float8_gpu.py: float8 and complex32 tensors on the
"ucc_b200" torch.distributed backend and in ucc_b200.ops / ucc_b200.parallel.

Every data-movement operation must return the bytes it was given, checked byte for byte through `.view(torch.uint8)` (NaN != NaN,
so never with `==`), and must leave the guard bytes around every output unchanged.  The inputs hold every one of the 256 byte
patterns of each float8 dtype, rotated by rank (NaNs, infinities where the format has them, -0 and subnormals included); complex32
inputs start with NaN payloads, -0, an infinity and a subnormal in both halves.  complex32 SUM / AVG must equal a float32 reference
on the same halves (small integers, so exactly).  Every other reduction of these dtypes must raise a ValueError that names the
dtype on every rank, after which a float8 all_gather still works.

argv[1] is "cpu" (host tensors, tl/shm) or "cuda" (rank r on cuda:<LOCAL_RANK % device count>, tl/nvl); argv[2] is a comma-separated
list of sections: small / big (every data-movement operation with blocks below / above the 1 MB zero-copy threshold; small also
runs the list forms on float16 / bfloat16 NaN payloads, which torch's c10d layer hands over for complex32), p2p (send /
recv below and above the 1 MB rendezvous threshold), stack (functional collectives eager and compiled, DTensor, ops, MoE), reduce
(complex32 sums and the refusals) and graph (graphed() keys and, on CUDA, a captured all_gather replayed).  On CUDA each direct
call must leave a tl/nvl kernel as this process's last launch.  Every check runs even when an earlier one failed; each rank
prints its failures, and rank 0 prints FLOAT8_WORKER_OK when every check passed on every rank."""
import functools
import os
import sys
import traceback

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ucc_b200.torch_backend  # noqa: F401,E402  (registers the backend)
from ucc_b200 import ops  # noqa: E402
from ucc_b200.parallel import moe_combine, moe_dispatch  # noqa: E402

MOVERS = ("exchange_", "self_copy")                       # launch notes of the tl/nvl data-movement kernels
REDUCERS = ("oneshot", "twoshot", "nvls", "ring", "rhd")   # ... and of its reduction kernels
P2P = ("p2p_",)                                            # ... and of send / recv
FLOAT8 = [getattr(torch, n) for n in ("float8_e4m3fn", "float8_e5m2", "float8_e4m3fnuz", "float8_e5m2fnuz", "float8_e8m0fnu")
          if hasattr(torch, n)]
TOKENS = [t for t in FLOAT8 if t != getattr(torch, "float8_e8m0fnu", None)]   # the element formats (e8m0 is a scale format)
DTYPES = FLOAT8 + [torch.complex32]
GUARD = 64                       # guard bytes before and after every output
POISON = 0xA5
# float16 bit patterns the complex32 inputs start with: quiet and signalling NaNs with payloads, -0, -inf, a subnormal
HALF_SPECIALS = (0x7E01, 0xFE33, 0x7C01, 0x8000, 0x8000, 0x7D55, 0x0001, 0xFC00)
SMALL, BIG = 1031, 3 << 19       # block bytes: an odd count, and 1.5 MB (over ZCOPY_THRESH and P2P_RNDV_THRESH, both 1 MB)


def esize(dtype):
    return torch.empty((), dtype=dtype).element_size()


@functools.lru_cache(maxsize=512)
def data(dtype, numel, rank, salt=0):
    """`numel` elements of `dtype`: byte i is (i + 97 * (i // 256) + 61 * rank + 13 * salt) % 256, so every run of 256 bytes holds
    each byte once, and the pattern differs by rank, by salt and between runs.  complex32 begins with HALF_SPECIALS, rotated."""
    i = torch.arange(numel * esize(dtype), dtype=torch.int64)
    b = ((i + 97 * (i // 256) + 61 * rank + 13 * salt) % 256).to(torch.uint8)
    if dtype == torch.complex32:
        halves = b.view(torch.int16)
        k = min(len(HALF_SPECIALS), halves.numel())
        halves[:k] = torch.tensor(HALF_SPECIALS, dtype=torch.int32).roll(rank + salt)[:k].to(torch.int16)
    return b.view(dtype)


def count(dtype, nbytes):
    return max(1, nbytes // esize(dtype))


def small_ints(shape, seed, n):
    """float16 halves holding integers in [-8, 8] times n: their sums and averages over n ranks are exact in float16"""
    g = torch.Generator().manual_seed(seed)
    return torch.view_as_complex((torch.randint(-8, 9, tuple(shape) + (2,), generator=g) * n).to(torch.float32)).to(torch.complex32)


class Worker:
    def __init__(self, use_cuda):
        self.rank, self.world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
        self.cuda = use_cuda
        if use_cuda:
            torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", self.rank)) % torch.cuda.device_count())
        self.dev = torch.device("cuda", torch.cuda.current_device()) if use_cuda else torch.device("cpu")
        dist.init_process_group("ucc_b200", rank=self.rank, world_size=self.world)
        self.pg = dist.group.WORLD
        self.comm = ops.init(dist.new_group(backend="gloo"))   # ucc_b200.ops / .parallel: a communicator of their own
        self.fails = []
        self.passed = 0
        self.guarded_bufs = []

    # ---- helpers
    def on(self, t):
        return t.to(self.dev)

    def ran(self, kinds, what):
        """on CUDA: the call launched a tl/nvl kernel of `kinds` (it did not go to a host transport)"""
        if self.cuda:
            note = self.pg._comm.request_info_last()
            assert note.startswith(kinds), f"{what}: last tl/nvl launch is {note!r}"

    def ran_ops(self, kinds, what):
        if self.cuda:
            note = self.comm.request_info_last()
            assert note.startswith(kinds), f"{what}: last tl/nvl launch is {note!r}"

    def out(self, dtype, numel):
        """an output of `numel` elements with GUARD poison bytes on each side (the inside is poisoned too)"""
        g = GUARD // esize(dtype)
        buf = torch.full(((numel + 2 * g) * esize(dtype),), POISON, dtype=torch.uint8, device=self.dev).view(dtype)
        self.guarded_bufs.append((buf, g, numel))
        return buf[g:g + numel]

    def check_guards(self):
        bufs, self.guarded_bufs = self.guarded_bufs, []
        for buf, g, numel in bufs:
            b = buf.cpu().view(torch.uint8)
            lo, hi = b[:g * esize(buf.dtype)], b[(g + numel) * esize(buf.dtype):]
            assert bool((lo == POISON).all()) and bool((hi == POISON).all()), \
                f"guard bytes around a {buf.dtype} output of {numel} elements were overwritten"

    def same(self, got, exp, what):
        got = got.detach().cpu()
        assert got.dtype == exp.dtype and got.shape == exp.shape, f"{what}: {got.dtype} {tuple(got.shape)} vs {exp.dtype} {tuple(exp.shape)}"
        g, e = got.reshape(-1).view(torch.uint8), exp.reshape(-1).contiguous().view(torch.uint8)
        if not torch.equal(g, e):
            bad = (g != e).nonzero()[0].item()
            raise AssertionError(f"{what}: byte {bad} of {g.numel()} is {g[bad].item():#04x}, expected {e[bad].item():#04x}")

    def case(self, name, fn, *args):
        try:
            fn(*args)
            if self.cuda:
                torch.cuda.current_stream().synchronize()
            self.check_guards()
            self.passed += 1
        except Exception as e:  # noqa: BLE001  (every failure is reported, then the next check runs)
            self.guarded_bufs = []
            self.fails.append(f"{name}{args}: {type(e).__name__}: {e}")
            if os.environ.get("FLOAT8_TRACE"):
                traceback.print_exc()

    # ---- data movement through torch.distributed
    def broadcast(self, dtype, m, root):
        t = self.out(dtype, m)
        t.copy_(self.on(data(dtype, m, self.rank, 1)))
        dist.broadcast(t, src=root)
        self.ran(MOVERS, "broadcast")
        self.same(t, data(dtype, m, root, 1), "broadcast")

    def all_gather_list(self, dtype, m, uneven):
        me, n = self.rank, self.world
        size = [(0 if p == 1 else m + p) if uneven else m for p in range(n)]   # uneven: odd and even counts, one empty block
        outs = [self.out(dtype, size[p]) for p in range(n)]
        dist.all_gather(outs, self.on(data(dtype, size[me], me, 2)))
        self.ran(MOVERS, "all_gather")
        for p in range(n):
            self.same(outs[p], data(dtype, size[p], p, 2), f"all_gather block of rank {p}")

    def all_gather_into_tensor(self, dtype, m):
        n = self.world
        o = self.out(dtype, m * n)
        dist.all_gather_into_tensor(o, self.on(data(dtype, m, self.rank, 3)))
        self.ran(MOVERS, "all_gather_into_tensor")
        self.same(o, torch.cat([data(dtype, m, p, 3) for p in range(n)]), "all_gather_into_tensor")

    def all_gather_into_tensor_coalesced(self, dtype, m):
        n, counts = self.world, (m, m // 2 + 1)
        outs = [self.out(dtype, c * n) for c in counts]
        with dist._coalescing_manager(device=self.dev):
            for i, (o, c) in enumerate(zip(outs, counts)):
                dist.all_gather_into_tensor(o, self.on(data(dtype, c, self.rank, 4 + i)))
        self.ran(MOVERS, "all_gather_into_tensor coalesced")
        for i, (o, c) in enumerate(zip(outs, counts)):
            self.same(o, torch.cat([data(dtype, c, p, 4 + i) for p in range(n)]), f"coalesced all_gather_into_tensor {i}")

    def all_gather_coalesced(self, dtype, m):
        me, n = self.rank, self.world
        size = lambda r, i: m if i == 0 else r + 1  # noqa: E731  (input 0: equal blocks, input 1: one size per rank)
        outs = [[self.out(dtype, size(p, i)) for i in range(2)] for p in range(n)]
        dist.all_gather_coalesced(outs, [self.on(data(dtype, size(me, i), me, 6 + i)) for i in range(2)])
        self.ran(MOVERS, "all_gather_coalesced")
        for p in range(n):
            for i in range(2):
                self.same(outs[p][i], data(dtype, size(p, i), p, 6 + i), f"all_gather_coalesced input {i} of rank {p}")

    def a2a_size(self, m, s, d):
        return 0 if (s + 2 * d) % 3 == 0 else m + s + 2 * d     # empty blocks, odd and even counts

    def all_to_all_single(self, dtype, m, uneven):
        me, n = self.rank, self.world
        size = (lambda s, d: self.a2a_size(m, s, d)) if uneven else (lambda s, d: m)
        inp = self.on(torch.cat([data(dtype, size(me, p), me, 10 + p) for p in range(n)]))
        o = self.out(dtype, sum(size(p, me) for p in range(n)))
        if uneven:
            dist.all_to_all_single(o, inp, [size(p, me) for p in range(n)], [size(me, p) for p in range(n)])
        else:
            dist.all_to_all_single(o, inp)
        self.ran(MOVERS, "all_to_all_single")
        self.same(o, torch.cat([data(dtype, size(p, me), p, 10 + me) for p in range(n)]), "all_to_all_single")

    def all_to_all_single_inplace(self, dtype, m):
        me, n = self.rank, self.world
        x = self.out(dtype, m * n)
        x.copy_(self.on(torch.cat([data(dtype, m, me, 10 + p) for p in range(n)])))
        dist.all_to_all_single(x, x)
        self.ran(MOVERS, "in-place all_to_all_single")
        self.same(x, torch.cat([data(dtype, m, p, 10 + me) for p in range(n)]), "in-place all_to_all_single")

    def all_to_all_list(self, dtype, m):
        me, n = self.rank, self.world
        outs = [self.out(dtype, self.a2a_size(m, p, me)) for p in range(n)]
        dist.all_to_all(outs, [self.on(data(dtype, self.a2a_size(m, me, p), me, 20 + p)) for p in range(n)])
        self.ran(MOVERS, "all_to_all")
        for p in range(n):
            self.same(outs[p], data(dtype, self.a2a_size(m, p, me), p, 20 + me), f"all_to_all block from rank {p}")

    def gather(self, dtype, m, root):
        me, n = self.rank, self.world
        size = [0 if p == 1 else m + p for p in range(n)]
        outs = [self.out(dtype, size[p]) for p in range(n)] if me == root else None
        dist.gather(self.on(data(dtype, size[me], me, 30)), outs, dst=root)
        self.ran(MOVERS, "gather")
        if me == root:
            for p in range(n):
                self.same(outs[p], data(dtype, size[p], p, 30), f"gather block of rank {p}")

    def scatter(self, dtype, m, root):
        me, n = self.rank, self.world
        size = [0 if p == 1 else m + p for p in range(n)]
        o = self.out(dtype, size[me])
        dist.scatter(o, [self.on(data(dtype, size[p], root, 40 + p)) for p in range(n)] if me == root else None, src=root)
        self.ran(MOVERS, "scatter")
        self.same(o, data(dtype, size[me], root, 40 + me), "scatter")

    def movement(self, nbytes):
        n = self.world
        for dtype in DTYPES:
            m = count(dtype, nbytes)
            for root in (0, n - 1):
                self.case("broadcast", self.broadcast, dtype, m, root)
                self.case("gather", self.gather, dtype, m, root)
                self.case("scatter", self.scatter, dtype, m, root)
            for uneven in (False, True):
                self.case("all_gather_list", self.all_gather_list, dtype, m, uneven)
                self.case("all_to_all_single", self.all_to_all_single, dtype, m, uneven)
            self.case("all_gather_into_tensor", self.all_gather_into_tensor, dtype, m)
            self.case("all_gather_into_tensor_coalesced", self.all_gather_into_tensor_coalesced, dtype, m)
            self.case("all_gather_coalesced", self.all_gather_coalesced, dtype, m)
            self.case("all_to_all_single_inplace", self.all_to_all_single_inplace, dtype, m)
            self.case("all_to_all_list", self.all_to_all_list, dtype, m)

    # ---- send / recv
    def p2p(self, dtype, m, how):
        me, n = self.rank, self.world
        nxt, prv = (me + 1) % n, (me - 1) % n
        src, dst = self.on(data(dtype, m, me, 50)), self.out(dtype, m)
        if how == "batch":
            works = dist.batch_isend_irecv([dist.P2POp(dist.irecv, dst, prv), dist.P2POp(dist.isend, src, nxt)])
        else:     # even ranks send first, odd ranks receive first
            first, second = (dist.isend(src, nxt), dist.irecv(dst, prv)) if me % 2 == 0 else (dist.irecv(dst, prv), dist.isend(src, nxt))
            works = [first, second]
        for w in works:
            w.wait()
        self.ran(P2P, f"{how} send / recv")
        self.same(dst, data(dtype, m, prv, 50), f"{how} receive from rank {prv}")

    # ---- functional collectives, DTensor, ops, MoE
    def funcol(self, dtype, compiled):
        import torch.distributed._functional_collectives as funcol
        me, n, group = self.rank, self.world, dist.group.WORLD
        m = count(dtype, SMALL)
        out_splits, in_splits = [self.a2a_size(m, p, me) for p in range(n)], [self.a2a_size(m, me, p) for p in range(n)]

        def fn(x, z):
            return [funcol.wait_tensor(t) for t in (funcol.all_gather_tensor(x, 0, group), funcol.all_to_all_single(z, out_splits, in_splits, group))]
        if compiled:
            torch._dynamo.reset()
            fn = torch.compile(fn, fullgraph=True, backend="aot_eager")
        x = self.on(data(dtype, m, me, 60))
        z = self.on(torch.cat([data(dtype, self.a2a_size(m, me, p), me, 70 + p) for p in range(n)]))
        got = [fn(x, z) for _ in range(2 if compiled else 1)]
        self.ran(MOVERS, "funcol")
        for it, (ag, a2a) in enumerate(got):
            self.same(ag, torch.cat([data(dtype, m, p, 60) for p in range(n)]), f"all_gather_tensor, call {it}")
            self.same(a2a, torch.cat([data(dtype, self.a2a_size(m, p, me), p, 70 + me) for p in range(n)]), f"all_to_all_single, call {it}")

    def dtensor(self, dtype):
        from torch.distributed.device_mesh import init_device_mesh
        from torch.distributed.tensor import Replicate, Shard, distribute_tensor
        n = self.world
        mesh = init_device_mesh(self.dev.type, (n,))
        full = data(dtype, 7 * 33, 0, 80).view(7, 33)      # 7 rows: not divisible by the mesh size
        d = distribute_tensor(self.on(full), mesh, [Shard(0)])
        r, whole = d.redistribute(mesh, [Replicate()]), d.full_tensor()
        self.same(d.to_local(), (list(full.chunk(n)) + [full[:0]] * n)[self.rank].contiguous(), "Shard(0) local")
        self.same(r.to_local(), full, "Shard(0) -> Replicate()")
        self.same(whole, full, "full_tensor")

    def ops_all_to_all(self, dtype, uneven):
        me, n = self.rank, self.world
        m = count(dtype, BIG if uneven else SMALL)
        size = (lambda s, d: self.a2a_size(m, s, d)) if uneven else (lambda s, d: m)
        o = self.out(dtype, sum(size(p, me) for p in range(n)))
        inp = self.on(torch.cat([data(dtype, size(me, p), me, 90 + p) for p in range(n)]))
        if uneven:
            ops.all_to_all_single(o, inp, [size(p, me) for p in range(n)], [size(me, p) for p in range(n)], comm=self.comm)
        else:
            ops.all_to_all_single(o, inp, comm=self.comm)
        self.ran_ops(MOVERS, "ops.all_to_all_single")
        self.same(o, torch.cat([data(dtype, size(p, me), p, 90 + me) for p in range(n)]), "ops.all_to_all_single")

    def moe(self, dtype, hidden):
        me, n = self.rank, self.world
        T = 50 + 7 * me
        tok = data(dtype, T * hidden, me, 100).view(T, hidden)
        dest = (torch.arange(T) * (me + 2)) % n
        dest[: T // 2] = 0                                 # rank 0's expert is hot
        recv, sc, rc, order = moe_dispatch(self.on(tok), self.on(dest), comm=self.comm)
        note = self.comm.request_info_last()
        back = moe_combine(recv, sc, rc, order, comm=self.comm)
        self.ran_ops(MOVERS, "moe_combine")
        assert not self.cuda or note.startswith(MOVERS), f"moe_dispatch: last tl/nvl launch is {note!r}"
        assert recv.dtype == dtype and recv.shape == (sum(rc), hidden), (recv.dtype, recv.shape)
        # what arrived from rank p: its tokens for this rank, in token order (the dispatch sorts stably by destination)
        exp = []
        for p in range(n):
            tp = 50 + 7 * p
            dp = (torch.arange(tp) * (p + 2)) % n
            dp[: tp // 2] = 0
            exp.append(data(dtype, tp * hidden, p, 100).view(tp, hidden)[dp == me])
        self.same(recv, torch.cat(exp), "moe_dispatch")
        self.same(back, tok, "moe_combine round trip")

    # ---- complex32 SUM / AVG
    def c32_ref(self, shape, seed, op):
        n = self.world
        total = sum(torch.view_as_real(small_ints(shape, seed + r, n).to(torch.complex64)) for r in range(n))   # float32
        return torch.view_as_complex(total / n if op == "avg" else total).to(torch.complex32)

    def c32_all_reduce(self, m, op, via):
        x = self.on(small_ints((m,), 200 + self.rank, self.world))
        if via == "dist":
            dist.all_reduce(x, op=dist.ReduceOp.SUM if op == "sum" else dist.ReduceOp.AVG)
            self.ran(REDUCERS, "all_reduce")
        else:
            ops.all_reduce(x, op=op, comm=self.comm)
            self.ran_ops(REDUCERS, "ops.all_reduce")
        self.same(x, self.c32_ref((m,), 200, op), f"complex32 all_reduce {op} via {via}")

    def c32_reduce(self, m, op, root):
        x = self.on(small_ints((m,), 210 + self.rank, self.world))
        dist.reduce(x, dst=root, op=dist.ReduceOp.SUM if op == "sum" else dist.ReduceOp.AVG)
        self.ran(REDUCERS, "reduce")
        if self.rank == root:
            self.same(x, self.c32_ref((m,), 210, op), f"complex32 reduce {op}")

    def c32_reduce_scatter(self, m, op, form):
        me, n = self.rank, self.world
        rop = dist.ReduceOp.SUM if op == "sum" else dist.ReduceOp.AVG
        if form == "tensor":
            o = self.out(torch.complex32, m)
            dist.reduce_scatter_tensor(o, self.on(small_ints((m * n,), 220 + me, n)), op=rop)
            exp = self.c32_ref((m * n,), 220, op)[me * m:(me + 1) * m]
        else:                      # blocks of different sizes, one of them empty: REDUCE_SCATTERV
            size = [0 if p == 1 else m + p for p in range(n)]
            o = self.out(torch.complex32, size[me])
            full = small_ints((sum(size),), 230 + me, n)
            dist.reduce_scatter(o, [self.on(b) for b in full.split(size)], op=rop)
            exp = self.c32_ref((sum(size),), 230, op).split(size)[me]
        if o.numel():
            self.ran(REDUCERS, "reduce_scatter")
        self.same(o, exp, f"complex32 reduce_scatter {form} {op}")

    def c32_reduce_scatter_ops(self, m, op):
        me, n = self.rank, self.world
        o = self.out(torch.complex32, m)
        ops.reduce_scatter_tensor(o, self.on(small_ints((m * n,), 240 + me, n)), op=op, comm=self.comm)
        self.ran_ops(REDUCERS, "ops.reduce_scatter_tensor")
        self.same(o, self.c32_ref((m * n,), 240, op)[me * m:(me + 1) * m], f"complex32 ops.reduce_scatter_tensor {op}")

    # ---- refusals
    def refused(self, dtype, opname, call, names_dtype=True):
        try:
            call()
        except ValueError as e:
            if names_dtype:
                assert str(dtype) in str(e) and opname in str(e), f"{dtype} {opname}: {e}"
            else:          # torch's own check, in front of the backend: it names complex tensors
                assert "complex" in str(e), f"{dtype} {opname}: {e}"
        else:
            raise AssertionError(f"{opname} of {dtype} tensors was accepted")

    def refusals(self, dtype):
        import torch.distributed._functional_collectives as funcol
        n = self.world
        t = lambda k=4: self.on(data(dtype, k, self.rank, 300))  # noqa: E731
        R = dist.ReduceOp
        if dtype == torch.complex32:
            for rop, opname in ((R.PRODUCT, "PROD"), (R.MAX, "MAX")):
                self.refused(dtype, opname, lambda: dist.all_reduce(t(), op=rop), names_dtype=False)
                self.refused(dtype, opname, lambda: dist.reduce(t(), dst=0, op=rop))
                self.refused(dtype, opname, lambda: dist.reduce_scatter_tensor(t(), t(4 * n), op=rop))
                self.refused(dtype, opname, lambda: dist.reduce_scatter(t(), [t() for _ in range(n)], op=rop))
                self.refused(dtype, opname, lambda: ops.all_reduce(t(), op=opname.lower(), comm=self.comm))
        else:
            for rop, opname in ((R.SUM, "SUM"), (R.AVG, "AVG"), (R.MAX, "MAX")):
                self.refused(dtype, opname, lambda: dist.all_reduce(t(), op=rop))
                self.refused(dtype, opname, lambda: dist.reduce(t(), dst=0, op=rop))
                self.refused(dtype, opname, lambda: dist.reduce_scatter_tensor(t(), t(4 * n), op=rop))
                self.refused(dtype, opname, lambda: dist.reduce_scatter(t(), [t() for _ in range(n)], op=rop))
            self.refused(dtype, "SUM", lambda: dist.all_reduce_coalesced([t(), t(3)]))
            # a float32 tensor in front of the float8 one: refused before the float32 request is created
            made, comm = [], self.pg._comm
            comm.init = lambda *a, **kw: made.append(a) or type(comm).init(comm, *a, **kw)
            try:
                self.refused(dtype, "SUM", lambda: self.pg.allreduce([self.on(torch.ones(3)), t()]))
            finally:
                del comm.init
            assert not made, f"{len(made)} request(s) created by a refused all_reduce"
            self.refused(dtype, "SUM", lambda: funcol.wait_tensor(funcol.all_reduce(t(), "sum", dist.group.WORLD)))
            self.refused(dtype, "SUM", lambda: ops.all_reduce(t(), comm=self.comm))
            self.refused(dtype, "SUM", lambda: ops.all_reduce_from_host(data(dtype, 64, self.rank, 301), t(64), comm=self.comm))
        # no member was left inside a collective: the next one runs on every rank
        self.all_gather_into_tensor(FLOAT8[0], 257)

    # ---- graphed(): requests cached by their dtype, and a float8 all_gather captured in a CUDA graph
    def graph_keys(self):
        me, n = self.rank, self.world
        m = 301
        raw = self.on(data(torch.uint8, m, me, 400))
        outs = [self.out(torch.uint8, m * n)]
        views = [torch.uint8] + FLOAT8
        reqs = self.pg._comm._graph_reqs
        with self.pg.graphed():
            before = len(reqs)
            held = []
            for it in range(2):
                for dt in views:
                    dist.all_gather_into_tensor(outs[0].view(dt), raw.view(dt))
                held.append(len(reqs) - before)
        self.pg.release_graphed()
        self.ran(MOVERS, "graphed all_gather")
        assert held == [len(views)] * 2, f"cached requests after each round {held}, for {len(views)} dtypes"
        self.same(outs[0], torch.cat([data(torch.uint8, m, p, 400) for p in range(n)]), "graphed all_gather")

    def graph_capture(self, dtype, nbytes):
        me, n = self.rank, self.world
        m = count(dtype, nbytes)
        inp, o = self.on(torch.empty(m, dtype=dtype)), self.out(dtype, m * n)

        got = {}          # every collective runs before any check, so that a failed check leaves no rank behind

        def check(it, what):
            torch.cuda.current_stream().synchronize()
            got[(what, it)] = o.cpu()

        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with self.pg.graphed():
            with torch.cuda.stream(side):
                for it in range(2):
                    inp.copy_(self.on(data(dtype, m, me, 500 + it)))
                    dist.all_gather_into_tensor(o, inp)
                    check(it, "warm-up")
            torch.cuda.current_stream().wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                dist.all_gather_into_tensor(o, inp)
        for it in range(10, 13):
            inp.copy_(self.on(data(dtype, m, me, 500 + it)))
            g.replay()
            check(it, "replay")
        error = self.pg._comm.take_device_error()
        del g
        self.pg.release_graphed()
        assert not error, "a replayed kernel gave up a device-side wait"
        for (what, it), t in got.items():
            self.same(t, torch.cat([data(dtype, m, p, 500 + it) for p in range(n)]), f"{what} {it}")

    def run(self, sections):
        if "small" in sections:
            self.movement(SMALL)
            for dtype in (torch.float16, torch.bfloat16):   # the list forms pack and unpack bit for bit: NaN payloads survive
                m = count(dtype, SMALL)
                self.case("all_gather_list", self.all_gather_list, dtype, m, True)
                self.case("all_to_all_list", self.all_to_all_list, dtype, m)
                self.case("gather", self.gather, dtype, m, 0)
                self.case("scatter", self.scatter, dtype, m, 0)
        if "big" in sections:
            self.movement(BIG)
        if "p2p" in sections:
            for dtype in DTYPES:
                for nbytes in (SMALL, BIG):
                    for how in ("batch", "pair"):
                        self.case("p2p", self.p2p, dtype, count(dtype, nbytes), how)
        if "stack" in sections:
            for dtype in DTYPES:
                self.case("funcol", self.funcol, dtype, False)
                for uneven in (False, True):
                    self.case("ops_all_to_all", self.ops_all_to_all, dtype, uneven)
            for dtype in FLOAT8[:2]:
                self.case("funcol compiled", self.funcol, dtype, True)
                self.case("dtensor", self.dtensor, dtype)
            for dtype in TOKENS:
                self.case("moe", self.moe, dtype, 24)
        if "reduce" in sections:
            for nbytes in (SMALL, BIG):
                m = count(torch.complex32, nbytes)
                for op in ("sum", "avg"):
                    for via in ("dist", "ops"):
                        self.case("c32_all_reduce", self.c32_all_reduce, m, op, via)
                    self.case("c32_reduce", self.c32_reduce, m, op, self.world - 1)
                    for form in ("tensor", "list"):
                        self.case("c32_reduce_scatter", self.c32_reduce_scatter, m, op, form)
                    self.case("c32_reduce_scatter_ops", self.c32_reduce_scatter_ops, m, op)
            for dtype in DTYPES:
                self.case("refusals", self.refusals, dtype)
        if "graph" in sections:
            self.case("graph_keys", self.graph_keys)
            if self.cuda:
                for nbytes in (SMALL, BIG):
                    self.case("graph_capture", self.graph_capture, FLOAT8[0], nbytes)
        for f in self.fails:
            print(f"FLOAT8_FAIL rank {self.rank}: {f}", flush=True)
        flag = self.on(torch.tensor([0.0 if self.fails else 1.0]))
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        ok = flag.item() == 1
        if self.rank == 0:
            print(f"FLOAT8_WORKER_{'OK' if ok else 'FAIL'} world {self.world} sections {','.join(sections)} "
                  f"checks {self.passed + len(self.fails)} passed {self.passed}", flush=True)
        ops.shutdown()
        dist.destroy_process_group()
        return ok


if __name__ == "__main__":
    sys.exit(0 if Worker(sys.argv[1] == "cuda").run(sys.argv[2].split(",")) else 1)
