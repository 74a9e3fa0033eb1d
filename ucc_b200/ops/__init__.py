"""Functional collectives on torch tensors, executed by libucc (tl/nvl kernels for CUDA tensors, tl/shm for host).

The call shapes follow torch.distributed so a user of `torch.distributed` + ProcessGroupUCC (reference consumer:
pytorch/torch-ucc) can switch by changing the import.  Every function returns a `Work` whose `.wait()` blocks the
host; with `async_op=False` (default) the wait is done before returning.  CUDA tensors are posted stream-ordered
(ucc_collective_triggered_post) on the current stream.  float8 and complex32 tensors move byte for byte; of their reductions
only complex32 SUM / AVG exist, the others raise ValueError (ucc_b200.dist.op_of)."""
from __future__ import annotations

import torch

from ..dist import Communicator, op_of

_default = None


def init(group=None, **kw) -> Communicator:
    """Create (once) the default communicator over `group` (default: WORLD)."""
    global _default
    if _default is None:
        _default = Communicator(group, **kw)
    return _default


def default_comm() -> Communicator:
    return init()


def shutdown():
    global _default
    if _default is not None:
        _default.destroy()
        _default = None


class Work:
    def __init__(self, req, keep=()):
        self.req, self._keep = req, keep

    def is_completed(self):
        return self.req is None or self.req.test() == 0

    def wait(self):
        if self.req is not None:
            self.req.wait()
            self.req.finalize()
            self.req = None
        return True


def _launch(comm, req, tensor, async_op, keep=(), wait_posted=True):
    if tensor is not None and tensor.is_cuda:
        req.post_on_stream(wait_posted=wait_posted)
    else:
        req.post()
    w = Work(req, keep)
    if not async_op:
        w.wait()
    return w


def all_reduce(tensor, op="sum", comm=None, async_op=False, overlap_gpu=False):
    """`overlap_gpu` (every collective below has it): the request carries UCC_COLL_ARGS_HINT_OPTIMIZE_OVERLAP_GPU, so tl/nvl moves
    its data by the copy engines and leaves the SMs to the kernels that run next to it (docs/user_guide.md)"""
    comm = comm or default_comm()
    return _launch(comm, comm.allreduce_init(tensor, tensor, op=op, overlap_gpu=overlap_gpu), tensor, async_op)


_from_host_state = {"chunks": 1}


def last_from_host_chunks():
    """how many chunks the most recent all_reduce_from_host() pipelined"""
    return _from_host_state["chunks"]


def all_reduce_from_host(host, out, staging=None, op="sum", comm=None, chunks=None, stream=None):
    """All-reduce a vector that lives in (pinned) HOST memory into the CUDA tensor `out` - offloaded gradients / optimizer
    shards, data-loader statistics.  The host -> device copy runs on its own stream (copy engine) in `chunks` pieces; the
    NVLink allreduce kernel of piece c is enqueued behind the arrival of piece c only, so PCIe transfer and NVLink
    reduction overlap instead of adding up.  `staging` (CUDA, same shape) receives the local copy; allocated when omitted.
    Every member must call with the same sizes (the chunking is derived from them).  Returns when `out` is complete."""
    comm = comm or default_comm()
    op_of(op, out)             # a reduction the library cannot do is refused before any copy is queued
    stream = stream or torch.cuda.current_stream()
    n = host.numel()
    nbytes = n * host.element_size()
    if chunks is None:
        chunks = 8 if nbytes >= (64 << 20) else (2 if nbytes >= (8 << 20) else 1)
    align = max(1, 256 // host.element_size())
    per = (n + chunks - 1) // chunks
    per = (per + align - 1) // align * align
    bounds = [(o, min(o + per, n)) for o in range(0, n, per)] if n else []
    _from_host_state["chunks"] = len(bounds)
    staging = staging if staging is not None else torch.empty_like(out)
    st = getattr(comm, "_h2d_stream", None)
    if st is None:
        st = comm._h2d_stream = torch.cuda.Stream()
    hflat, sflat, oflat = host.view(-1), staging.view(-1), out.view(-1)
    st.wait_stream(stream)                                   # earlier readers of `staging` on the caller's stream
    evs = []
    with torch.cuda.stream(st):
        for lo, hi in bounds:
            sflat[lo:hi].copy_(hflat[lo:hi], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(st)
            evs.append(ev)
    reqs = []
    for (lo, hi), ev in zip(bounds, evs):
        stream.wait_event(ev)
        r = comm.allreduce_init(sflat[lo:hi], oflat[lo:hi], op=op)
        # wait until the kernel really is in the stream (a zero-copy collective launches once the members' buffers are known):
        # the wait for the NEXT piece must be enqueued behind this kernel, not in front of it
        r.post_on_stream(stream, wait_posted=True)
        reqs.append(r)
    for r in reqs:
        r.wait()
        r.finalize()
    return out


def reduce(tensor, dst=0, op="sum", comm=None, async_op=False, overlap_gpu=False):
    comm = comm or default_comm()
    req = comm.coll_init("reduce", None if comm.rank == dst else tensor, tensor if comm.rank == dst else None, op=op, root=dst, inplace=comm.rank == dst,
                         overlap_gpu=overlap_gpu)
    return _launch(comm, req, tensor, async_op)


def broadcast(tensor, src=0, comm=None, async_op=False, overlap_gpu=False):
    comm = comm or default_comm()
    return _launch(comm, comm.coll_init("bcast", tensor, None, root=src, overlap_gpu=overlap_gpu), tensor, async_op)


def all_gather_into_tensor(output, input, comm=None, async_op=False, overlap_gpu=False):
    comm = comm or default_comm()
    assert output.numel() == input.numel() * comm.size
    return _launch(comm, comm.coll_init("allgather", input, output, overlap_gpu=overlap_gpu), input, async_op)


def reduce_scatter_tensor(output, input, op="sum", comm=None, async_op=False, overlap_gpu=False):
    comm = comm or default_comm()
    assert input.numel() == output.numel() * comm.size
    return _launch(comm, comm.coll_init("reduce_scatter", input, output, op=op, overlap_gpu=overlap_gpu), input, async_op)


def all_to_all_single(output, input, output_split_sizes=None, input_split_sizes=None, comm=None, async_op=False, overlap_gpu=False):
    """Equal splits -> alltoall; explicit split sizes (in elements of dim 0 rows) -> alltoallv (MoE dispatch / combine)."""
    comm = comm or default_comm()
    return _launch(comm, _alltoall_init(comm, output, input, output_split_sizes, input_split_sizes, overlap_gpu), input, async_op)


def _alltoall_init(comm, output, input, output_split_sizes, input_split_sizes, overlap_gpu=False):
    """alltoall / alltoallv request; `output` and `input` being the same memory makes it an in-place request, whose counts and
    displacements are those of the output (an in-place alltoallv needs the same split sizes in both directions)"""
    inplace = output.data_ptr() == input.data_ptr()
    src = None if inplace else input
    if output_split_sizes is None and input_split_sizes is None:
        return comm.coll_init("alltoall", src, output, inplace=inplace, overlap_gpu=overlap_gpu)
    row = input[0].numel() if input.dim() > 1 else 1
    sc = [int(s) * row for s in input_split_sizes]
    rc = [int(s) * row for s in output_split_sizes]
    sd = [sum(sc[:i]) for i in range(len(sc))]
    rd = [sum(rc[:i]) for i in range(len(rc))]
    if inplace:
        if sc != rc:
            raise ValueError("in-place all_to_all_single needs input_split_sizes == output_split_sizes")
        return comm.coll_init("alltoallv", None, output, inplace=True, dst_counts=rc, dst_displs=rd, overlap_gpu=overlap_gpu)
    return comm.coll_init("alltoallv", input, output, src_counts=sc, src_displs=sd, dst_counts=rc, dst_displs=rd, overlap_gpu=overlap_gpu)


def all_gather_v(output, input, counts, comm=None, async_op=False, overlap_gpu=False):
    comm = comm or default_comm()
    displs = [sum(counts[:i]) for i in range(len(counts))]
    return _launch(comm, comm.coll_init("allgatherv", input, output, dst_counts=list(counts), dst_displs=displs, overlap_gpu=overlap_gpu), input, async_op)


def gather(output, input, dst=0, comm=None, async_op=False, overlap_gpu=False):
    comm = comm or default_comm()
    return _launch(comm, comm.coll_init("gather", input, output if comm.rank == dst else None, root=dst, overlap_gpu=overlap_gpu), input, async_op)


def scatter(output, input, src=0, comm=None, async_op=False, overlap_gpu=False):
    comm = comm or default_comm()
    return _launch(comm, comm.coll_init("scatter", input if comm.rank == src else None, output, root=src, overlap_gpu=overlap_gpu), output, async_op)


def barrier(comm=None):
    (comm or default_comm()).barrier()


# ---- point to point (pipeline / ring-attention shapes): a two-member active-set broadcast, the way ProcessGroupUCC does it
def _p2p(tensor, src, dst, tag, comm, async_op):
    req = comm.coll_init("bcast", tensor, None, root=src, active_set=(src, dst - src, 2), tag=int(tag) & 0x3fff)
    # a large send is launched only once the receiver has published its buffer (rendezvous): never block in the post, or two
    # ranks that both send first would wait for each other's receive forever; Work.wait() drives the progress
    return _launch(comm, req, tensor, async_op, wait_posted=False)


def send(tensor, dst, tag=0, comm=None, async_op=False):
    comm = comm or default_comm()
    return _p2p(tensor, comm.rank, dst, tag, comm, async_op)


def recv(tensor, src, tag=0, comm=None, async_op=False):
    comm = comm or default_comm()
    return _p2p(tensor, src, comm.rank, tag, comm, async_op)


def batch_p2p(batch, comm=None):
    """The role of torch.distributed.batch_isend_irecv / an NCCL group: `batch` is a list of ("send" | "recv", tensor, peer[, tag]).
    All sends are posted before all receives (each kind in list order): a kernel of the eager ring may wait for its peer, so a
    receive must never be queued in front of a send that another rank is waiting for.  Returns the Work objects in `batch` order."""
    comm = comm or default_comm()
    works = [None] * len(batch)
    for want in ("send", "recv"):
        for i, item in enumerate(batch):
            kind, tensor, peer = item[0], item[1], item[2]
            tag = item[3] if len(item) > 3 else 0
            if kind != want:
                continue
            works[i] = send(tensor, peer, tag, comm, async_op=True) if kind == "send" else recv(tensor, peer, tag, comm, async_op=True)
    assert all(w is not None for w in works), "batch entries are ('send' | 'recv', tensor, peer[, tag])"
    return works


def ring_exchange(send_tensor, recv_tensor, shift=1, tag=0, comm=None):
    """Every rank sends to (rank + shift) and receives from (rank - shift): one hop of ring attention / a pipeline bubble step
    (a batch: the send is posted before the receive on every rank)."""
    comm = comm or default_comm()
    n, r = comm.size, comm.rank
    to, frm = (r + shift) % n, (r - shift) % n
    if n == 1:
        recv_tensor.copy_(send_tensor)
        return
    for w in batch_p2p([("recv", recv_tensor, frm, tag), ("send", send_tensor, to, tag)], comm):
        w.wait()
