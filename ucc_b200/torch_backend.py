"""`torch.distributed` backend "ucc_b200": the role PyTorch's ProcessGroupUCC plays for the reference
(torch/csrc/distributed/c10d/ProcessGroupUCC.cpp consumes ucc_collective_init / triggered_post / test).

    import ucc_b200.torch_backend            # registers the backend
    torch.distributed.init_process_group("ucc_b200", rank=..., world_size=...)
    torch.distributed.all_reduce(t)          # -> libucc: tl/nvl NVLink kernels for CUDA tensors, tl/shm for host tensors
    torch.nn.parallel.DistributedDataParallel(model)   # gradient buckets go through the same path

The process group is a Python subclass of `torch.distributed.ProcessGroup`; wire-up uses the rendezvous store as the
UCC out-of-band allgather.  Every group it makes (the default group, `new_group` groups, DeviceMesh dimension groups) keeps
the name and description torch gives it, so PyTorch's own parallel stack runs on it: `_functional_collectives` (also under
`torch.compile`, whose `_c10d_functional` ops find the group by that name), DeviceMesh, DTensor, FSDP2 (`fully_shard`, HSDP)
and `torch.distributed.tensor.parallel`.

CUDA collectives are posted stream-ordered on the caller's current stream; the host does not wait for the GPU.  `Work.wait()`
makes sure the kernels are in that stream and then makes the stream current at wait() wait for them, as ProcessGroupNCCL's does:
a collective posted on a side stream and waited for on another is read there only after it has run.

c10d operations served: allreduce (+ _coalesced), broadcast, reduce, allgather (+ _coalesced, _into_tensor_coalesced,
_allgather_base), reduce_scatter (+ _tensor_coalesced, _reduce_scatter_base), alltoall (lists) and alltoall_base, gather, scatter,
send, recv, barrier and the coalescing hooks _start_coalescing / _end_coalescing, so also gather_object, scatter_object_list,
all_gather_coalesced and _coalescing_manager.  The list forms of allgather, reduce_scatter, gather, scatter and alltoall take
blocks of any size, zero included.  torch.bool tensors travel as uint8: SUM / MAX are logical or, PRODUCT / MIN logical and, AVG
is refused.  float8 tensors (float8_e4m3fn, float8_e5m2, their fnuz forms, float8_e8m0fnu) travel as uint8 and complex32 as uint32,
byte for byte, in every data-movement operation; complex32 SUM / AVG reduce its float16 halves, and every other reduction of these
dtypes raises a ValueError that names the dtype and the operator, on every rank and before anything is posted.
Not served, each with an error that names it: ReduceOp.PREMUL_SUM (its factor cannot be read from Python and the library has no
scaled sum; FSDP2 uses it only for a custom gradient divide factor), recv_anysource (on CUDA tensors a send / recv pair matches in
post order, so a receive must name its source), monitored_barrier and split_group.

Every collective works inside `torch.cuda.graph`.  Wrap the warm-up iterations and the capture in `pg.graphed()` (see
Communicator.graphed) so that the captured collectives reuse the zero-copy tables their warm-up posts resolved."""
from __future__ import annotations

import itertools

import torch
import torch.distributed as dist

from .dist import Communicator, op_of
from .ops import _alltoall_init

_OPS = {dist.ReduceOp.SUM: "sum", dist.ReduceOp.PRODUCT: "prod", dist.ReduceOp.MIN: "min", dist.ReduceOp.MAX: "max", dist.ReduceOp.AVG: "avg",
        dist.ReduceOp.BAND: "band", dist.ReduceOp.BOR: "bor", dist.ReduceOp.BXOR: "bxor"}


def _op(o):
    o = getattr(o, "op", o)   # ReduceOp object or RedOpType
    for k, v in _OPS.items():
        if o == k:
            return v
    if o == dist.ReduceOp.PREMUL_SUM:
        # the factor of a PREMUL_SUM op cannot be read from Python, and the library has no scaled sum
        raise ValueError("ucc_b200 does not support ReduceOp.PREMUL_SUM: use SUM or AVG and scale the tensor")
    raise ValueError(f"unsupported reduce op {o}")


def _reduce_op(opts, tensors):
    """the operator of a reduction over `tensors`; a (dtype, operator) pair the library cannot reduce raises ValueError here,
    before any request of the call exists"""
    op = _op(opts.reduceOp) if opts is not None else "sum"
    for t in tensors:
        op_of(op, t)
    return op


def _flat(n, like):
    """1-D buffer of `n` elements of `like`'s dtype and device, never at address 0, even when `n` is 0"""
    return torch.empty(max(n, 1), dtype=like.dtype, device=like.device)[:n]


def _views(flat, tensors):
    """`flat` cut into consecutive views, one per tensor and shaped like it"""
    offs = itertools.accumulate((t.numel() for t in tensors), initial=0)
    return [flat[o:o + t.numel()].view(t.shape) for o, t in zip(offs, tensors)]


_INT_OF_SIZE = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def _copy(dsts, srcs):
    """dsts[i] <- srcs[i] bit for bit, stream-ordered on CUDA.  torch's CUDA _foreach_copy_ converts floating-point elements
    through float, which rewrites the NaN payloads of float16, bfloat16 and float8, and it has no float8_e8m0fnu kernel: tensors
    of one dtype are copied as integers of their element size"""
    def raw(t):
        size = t.element_size()
        return t.view(_INT_OF_SIZE[size]) if size in _INT_OF_SIZE else t.unsqueeze(-1).view(torch.int64)
    pairs = [(raw(d), raw(s)) if d.dtype == s.dtype else (d, s) for d, s in zip(dsts, srcs)]
    torch._foreach_copy_([d for d, _ in pairs], [s for _, s in pairs])


def _pack(tensors):
    flat = _flat(sum(t.numel() for t in tensors), tensors[0])
    _copy(_views(flat, tensors), list(tensors))
    return flat


def _displs(counts):
    return list(itertools.accumulate(counts, initial=0))[:-1]


class _Work(dist._Work):
    def __init__(self, pg, reqs, result, cuda, side_stream=None, parts=(), posted=None):
        super().__init__()
        self._pg, self._reqs, self._result, self._cuda = pg, reqs, result, cuda
        self._side = side_stream      # CUDA p2p runs on an internal stream; wait() makes the caller's stream wait for it
        self._posted = posted         # CUDA collectives: (stream, event recorded on it behind the collective's kernels)
        self._parts = parts           # the Work of every operation of a coalescing block
        self._fut = torch.futures.Future()
        self._done = False
        if pg._coalesced is not None:
            pg._coalesced.append(self)

    def _finish(self):
        if self._done:
            return
        for r in self._reqs:
            if not self._cuda:
                r.wait()            # host buffers: completion == data valid
            else:
                r.wait_posted()     # the kernel is in the stream (idempotent; immediate for everything but p2p)
            r.finalize_later() if self._cuda else r.finalize()
        if self._side is not None:
            torch.cuda.current_stream().wait_stream(self._side)
        if self._posted is not None:
            # c10d contract (ProcessGroupNCCL's WorkNCCL::wait): work the caller queues after wait() on its current stream runs
            # after the collective, also when it was posted on another stream.  The host does not wait.
            stream, event = self._posted
            current = torch.cuda.current_stream()
            if current != stream:
                current.wait_event(event)
        for w in self._parts:
            w._finish()
        self._done = True
        self._fut.set_result(self._result)

    def is_completed(self):
        return all(r.test() == 0 for r in self._reqs) and all(w.is_completed() for w in self._parts)

    def is_success(self):
        return True

    def wait(self, timeout=None):
        self._finish()
        return True

    def get_future(self):
        self._finish()
        return self._fut

    def result(self):
        return self._result


class ProcessGroupUCCB200(dist.ProcessGroup):
    def __init__(self, store, rank, size, timeout=None):
        super().__init__(rank, size)
        self._comm = Communicator(store=store, rank=rank, size=size)
        self._pending = []   # CUDA requests whose kernels are in flight; finalized lazily
        self._p2p_streams = {}
        self._coalesced = None   # between _start_coalescing and _end_coalescing: the Work of every operation
        self._name, self._desc = None, None
        self._overlap_gpu = False

    def getBackendName(self):
        return "ucc_b200"

    # torch uses this object as the group itself, with no c10d Backend registered inside it, and ProcessGroup keeps its name and
    # description in such a Backend.  Keep them here instead: _functional_collectives, DeviceMesh, DTensor and FSDP2 find the group
    # by its name (the _c10d_functional ops resolve the name torch registered with this object and call back into it).
    def _set_group_name(self, name):
        self._name = name

    @property
    def group_name(self):
        if self._name is None:
            raise RuntimeError("ucc_b200: the process group has no name yet")
        return self._name

    def _set_group_desc(self, desc):
        self._desc = desc

    @property
    def group_desc(self):
        return self._desc if self._desc is not None else "undefined"

    def graphed(self):
        """context manager for the warm-up and the capture of a CUDA graph: Communicator.graphed() of this group"""
        return self._comm.graphed()

    def release_graphed(self):
        self._comm.release_graphed()

    def set_overlap_gpu(self, on=True):
        """Every collective of this group from now on carries UCC_COLL_ARGS_HINT_OPTIMIZE_OVERLAP_GPU (send / recv does not): on tl/nvl
        its data crosses NVLink by the copy engines and the SMs stay free for the kernels that run next to it, e.g. the compute of
        FSDP2 or DDP, whose group is `mesh.get_group()` / the process group passed to DDP.  Every member sets the same value, before
        the same collective.  Results are bitwise those of the group without it (docs/user_guide.md)."""
        self._overlap_gpu = bool(on)

    def _init(self, coll, src=None, dst=None, **kw):
        return self._comm.coll_init(coll, src, dst, overlap_gpu=self._overlap_gpu, **kw)

    # ---- helpers
    def _run(self, reqs, tensors, result, wait_posted=True, outs=(), views=()):
        """post `reqs`; then outs[i] <- views[i] once the collectives have written the views: stream-ordered behind them on CUDA,
        after the wait on the host"""
        cuda = bool(tensors) and tensors[0].is_cuda
        for r in reqs:
            if cuda:
                r.post_on_stream(wait_posted=wait_posted)   # returns once the kernel is in the current stream
                r.finalize_later = lambda r=r: self._pending.append(r)
            else:
                r.post()
        posted = None
        if cuda:
            if outs:
                _copy(outs, views)
            if wait_posted:   # every kernel is in the stream, a deferred zero-copy launch included: mark the stream behind them
                stream = torch.cuda.current_stream()
                posted = (stream, stream.record_event())
        self._reap()
        w = _Work(self, reqs, result, cuda, posted=posted)
        if outs and not cuda:
            w.wait()
            _copy(outs, views)
        return w

    def _reap(self):
        keep = []
        for r in self._pending:
            if r._graphed:          # owned by the graphed() cache, which finalizes it
                continue
            if r.test() == 0:
                r.finalize()
            else:
                keep.append(r)
        self._pending = keep
        if len(keep) > 256:
            for r in keep:
                r.wait(); r.finalize()
            self._pending = []

    # ---- collectives (list-of-tensors signatures of c10d)
    def allreduce(self, tensors, opts=None):
        op = _reduce_op(opts, tensors)
        reqs = [self._comm.allreduce_init(t, t, op=op, overlap_gpu=self._overlap_gpu) for t in tensors]
        return self._run(reqs, tensors, tensors)

    def allreduce_coalesced(self, tensors, opts=None):
        return self.allreduce(tensors, opts)

    def broadcast(self, tensors, opts=None):
        root = opts.rootRank if opts is not None else 0
        reqs = [self._init("bcast", t, None, root=root) for t in tensors]
        return self._run(reqs, tensors, tensors)

    def reduce(self, tensors, opts=None):
        root = opts.rootRank if opts is not None else 0
        op = _reduce_op(opts, tensors)
        me = self.rank()
        reqs = [self._init("reduce", None if me == root else t, t if me == root else None, op=op, root=root, inplace=me == root) for t in tensors]
        return self._run(reqs, tensors, tensors)

    # The list forms of allgather and reduce_scatter hold one block per rank, and every rank passes the whole list, so every rank
    # sees every block size.  Blocks of one size post ALLGATHER / REDUCE_SCATTER, blocks of different sizes (zero included) post
    # ALLGATHERV / REDUCE_SCATTERV, and all ranks make the same choice.
    def allgather(self, output_lists, input_tensors, opts=None):
        reqs, outs, views = [], [], []
        for blocks, inp in zip(output_lists, input_tensors):
            counts = [t.numel() for t in blocks]
            if len(set(counts)) == 1:
                flat = torch.empty((len(blocks),) + tuple(inp.shape), dtype=inp.dtype, device=inp.device)
                reqs.append(self._init("allgather", inp.contiguous(), flat))
                views += list(flat)
            else:
                flat = _flat(sum(counts), inp)
                src = inp.contiguous() if inp.numel() else _pack([inp])
                reqs.append(self._init("allgatherv", src, flat, dst_counts=counts, dst_displs=_displs(counts)))
                views += _views(flat, blocks)
            outs += blocks
        return self._run(reqs, input_tensors, output_lists, outs=outs, views=views)

    def allgather_coalesced(self, output_lists, input_list, opts=None):
        # output_lists[r][i] receives input_list[i] of rank r: one allgather per input
        return self.allgather([list(blocks) for blocks in zip(*output_lists)], input_list, opts)

    def _allgather_base(self, output, input, opts=None):
        return self._run([self._init("allgather", input.contiguous(), output)], [input], output)

    def allgather_into_tensor_coalesced(self, outputs, inputs, opts=None):
        return self._run([self._init("allgather", i.contiguous(), o) for o, i in zip(outputs, inputs)], inputs, outputs)

    def _reduce_scatter_base(self, output, input, opts=None):
        op = _reduce_op(opts, [input])
        return self._run([self._init("reduce_scatter", input.contiguous(), output, op=op)], [input], output)

    def reduce_scatter_tensor_coalesced(self, outputs, inputs, opts=None):
        op = _reduce_op(opts, inputs)
        return self._run([self._init("reduce_scatter", i.contiguous(), o, op=op) for o, i in zip(outputs, inputs)], inputs, outputs)

    def reduce_scatter(self, outputs, input_lists, opts=None):
        op = _reduce_op(opts, outputs)
        reqs, keep = [], []
        for out, ins in zip(outputs, input_lists):
            counts = [t.numel() for t in ins]
            if len(set(counts)) == 1:
                flat = torch.cat([t.reshape(-1) for t in ins])
                reqs.append(self._init("reduce_scatter", flat, out, op=op))
            else:
                flat = _pack(ins)
                dst = out if out.numel() else _flat(0, out)
                reqs.append(self._init("reduce_scatterv", flat, dst, op=op, dst_counts=counts, dst_displs=_displs(counts)))
            keep.append(flat)
        w = self._run(reqs, outputs, outputs)
        w._keep = keep
        return w

    def alltoall_base(self, output, input, output_split_sizes, input_split_sizes, opts=None):
        # an output aliasing the input makes it an in-place request
        equal = not output_split_sizes and not input_split_sizes
        req = _alltoall_init(self._comm, output, input.contiguous(), None if equal else output_split_sizes, None if equal else input_split_sizes,
                             self._overlap_gpu)
        return self._run([req], [input], output)

    # A rank cannot see the block sizes of the others (a gather's non-roots do not even see the root's list), so deciding between a
    # collective and its V form by the local sizes could post ALLTOALL on one rank and ALLTOALLV on another - e.g. on a rank that
    # moves nothing in this step - and the two do not match.  The list forms of alltoall, gather and scatter therefore always post
    # the V form.
    # Inside graphed() requests are cached by their buffers, and every member must create a new request or re-post a cached one in
    # step with the others (tl/nvl matches the zero-copy exchange by post order).  The root's flat buffer of a gather or scatter is
    # new on every call, so inside graphed() the other ranks move their block through a new buffer, too.
    def alltoall(self, output_tensors, input_tensors, opts=None):
        dst = _flat(sum(t.numel() for t in output_tensors), output_tensors[0])
        req = _alltoall_init(self._comm, dst, _pack(input_tensors), [t.numel() for t in output_tensors], [t.numel() for t in input_tensors],
                             self._overlap_gpu)
        return self._run([req], input_tensors, output_tensors, outs=output_tensors, views=_views(dst, output_tensors))

    def gather(self, output_tensors, input_tensors, opts=None):
        """the root passes one list of N blocks per input, the other ranks pass []"""
        root = opts.rootRank if opts is not None else 0
        reqs, outs, views = [], [], []
        for i, inp in enumerate(input_tensors):
            src = inp.contiguous() if inp.numel() and not self._comm._graphing else _pack([inp])
            if self.rank() != root:
                reqs.append(self._init("gatherv", src, None, root=root))
                continue
            blocks = output_tensors[i]
            counts = [t.numel() for t in blocks]
            flat = _flat(sum(counts), inp)
            reqs.append(self._init("gatherv", src, flat, root=root, dst_counts=counts, dst_displs=_displs(counts)))
            outs += blocks
            views += _views(flat, blocks)
        return self._run(reqs, input_tensors, output_tensors, outs=outs, views=views)

    def scatter(self, output_tensors, input_tensors, opts=None):
        """the root passes one list of N blocks per output, the other ranks pass []"""
        root = opts.rootRank if opts is not None else 0
        reqs, outs, views = [], [], []
        for i, out in enumerate(output_tensors):
            dst = out
            if not out.numel() or self._comm._graphing:
                dst = _flat(out.numel(), out)
                outs.append(out)
                views.append(dst.view(out.shape))
            if self.rank() != root:
                reqs.append(self._init("scatterv", None, dst, root=root))
                continue
            counts = [t.numel() for t in input_tensors[i]]
            reqs.append(self._init("scatterv", _pack(input_tensors[i]), dst, root=root, src_counts=counts, src_displs=_displs(counts)))
        return self._run(reqs, output_tensors, output_tensors, outs=outs, views=views)

    # ---- coalescing (torch's _coalescing_manager with a device): one Work that completes every operation of the block
    def _start_coalescing(self, device):
        if self._coalesced is not None:
            raise RuntimeError("ucc_b200: _start_coalescing while a coalescing block is already open")
        self._coalesced = []

    def _end_coalescing(self, device):
        if self._coalesced is None:
            raise RuntimeError("ucc_b200: _end_coalescing without _start_coalescing")
        works, self._coalesced = self._coalesced, None
        return _Work(self, [], None, False, parts=works)

    # ---- point to point: a two-member active-set broadcast, exactly how ProcessGroupUCC maps send/recv onto UCC.
    # CUDA tensors travel over tl/nvl's heap channels: messages between an ordered pair of ranks are matched in POST ORDER (the NCCL
    # contract: the tag does not reorder them); host tensors go through tl/shm, which matches by tag.
    def _p2p(self, tensors, src, dst, tag):
        reqs = [self._comm.coll_init("bcast", t, None, root=src, active_set=(src, dst - src, 2), tag=int(tag) & 0x3fff) for t in tensors]
        # rendezvous: a large send enters the stream when the receiver has published its buffer, a receive is published when the
        # stream reaches it - both need progress, which Work.wait() provides (isend + irecv + wait, as with every backend)
        if not (tensors and tensors[0].is_cuda):
            return self._run(reqs, tensors, tensors, wait_posted=False)
        # CUDA: one internal stream per (peer, direction), as ProcessGroupNCCL keeps per-peer streams - a kernel of the eager ring
        # may wait for its peer (a receive posted before its send), and torch issues the ops of batch_isend_irecv one after the
        # other on the caller's stream: an irecv in front of an isend there would deadlock a ring of ranks
        peer, is_send = (dst, True) if src == self.rank() else (src, False)
        side = self._p2p_streams.get((peer, is_send))
        if side is None:
            side = self._p2p_streams[(peer, is_send)] = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        for r, t in zip(reqs, tensors):
            r.post_on_stream(side, wait_posted=False)
            r.finalize_later = lambda r=r: self._pending.append(r)
            t.record_stream(side)
        self._reap()
        return _Work(self, reqs, tensors, True, side_stream=side)

    def send(self, tensors, dstRank, tag=0):
        return self._p2p(tensors, self.rank(), dstRank, tag)

    def recv(self, tensors, srcRank, tag=0):
        return self._p2p(tensors, srcRank, self.rank(), tag)

    def recv_anysource(self, tensors, tag=0):
        raise RuntimeError("ucc_b200 does not support recv_anysource: send / recv pairs match in post order on CUDA tensors, so "
                           "every receive must name its source")

    def barrier(self, opts=None):
        self._comm.barrier()
        w = _Work(self, [], None, False)
        return w

    def monitored_barrier(self, *args, **kwargs):
        raise RuntimeError("ucc_b200 does not support monitored_barrier: use barrier")

    def split_group(self, *args, **kwargs):
        raise RuntimeError("ucc_b200 does not support split_group")

    def shutdown(self):
        for r in self._pending:
            if not r._graphed:
                r.wait(); r.finalize()
        self._pending = []
        self._comm.destroy()


def _create(store, rank, size, timeout):
    return ProcessGroupUCCB200(store, rank, size, timeout)


def register():
    if "UCC_B200" not in [b for b in dir(dist.Backend)]:
        dist.Backend.register_backend("ucc_b200", _create, devices=["cpu", "cuda"])


register()
