"""One process per GPU: library / context / team bootstrap on top of torch.distributed.

torch.distributed (gloo) only provides the out-of-band allgather used for wire-up, exactly the role
MPI plays for the reference's ucc_perftest (tools/perf/ucc_pt_bootstrap_mpi.cc).  All collectives
then run through libucc: tl/nvl kernels over NVLink for CUDA tensors, tl/shm for host tensors.
"""
import contextlib
import ctypes as C
import itertools
import os

import torch
import torch.distributed as dist

from . import capi as U

_TORCH_DT = {torch.int8: "int8", torch.int16: "int16", torch.int32: "int32", torch.int64: "int64", torch.uint8: "uint8",
             torch.float16: "float16", torch.float32: "float32", torch.float64: "float64", torch.bfloat16: "bfloat16",
             torch.complex64: "float32_complex", torch.complex128: "float64_complex", torch.bool: "uint8"}
for _n, _t in (("uint16", "uint16"), ("uint32", "uint32"), ("uint64", "uint64")):
    if hasattr(torch, _n):
        _TORCH_DT[getattr(torch, _n)] = _t

# torch dtypes the library has no datatype for travel as the unsigned integer of their element size, so every data-movement
# collective moves their bytes unchanged; counts and displacements stay in elements of the tensor
_CARRIERS = {torch.complex32: "uint32"}
for _n in ("float8_e4m3fn", "float8_e5m2", "float8_e4m3fnuz", "float8_e5m2fnuz", "float8_e8m0fnu"):
    if hasattr(torch, _n):
        _CARRIERS[getattr(torch, _n)] = "uint8"
_TORCH_DT.update(_CARRIERS)

# a torch.bool tensor goes to the library as uint8 holding 0 / 1: sum is logical or (max), product logical and (min), as in
# ProcessGroupNCCL; the bitwise and logical operators keep 0 / 1 as they are
_BOOL_OP = {"sum": "max", "prod": "min"}

# the collectives whose operator the library applies
REDUCTIONS = frozenset(("allreduce", "reduce", "reduce_scatter", "reduce_scatterv"))


def dt_of(t):
    return _TORCH_DT[t.dtype]


def op_of(op, t):
    """(library datatype, library operator, library elements per element of `t`) of the reduction `op` on `t`.

    A complex32 element is two interleaved float16 halves, so its SUM and AVG are the float16 SUM and AVG of twice as many
    elements.  Every other reduction of a carried dtype (float8, complex32) raises ValueError: the library has no arithmetic for
    them.  The dtype alone decides, and every member of a collective passes the same dtype, so all of them refuse before
    any request exists."""
    if t.dtype == torch.bool:
        if op == "avg":
            raise ValueError("AVG reduction is not defined for torch.bool tensors")
        return "uint8", _BOOL_OP.get(op, op), 1
    if t.dtype == torch.complex32 and op in ("sum", "avg"):
        return "float16", op, 2
    if t.dtype in _CARRIERS:
        raise ValueError(f"{op.upper()} reduction is not supported for {t.dtype} tensors: the library moves them as "
                         f"{_CARRIERS[t.dtype]} without arithmetic (complex32 has SUM and AVG, float8 no reduction)")
    return dt_of(t), op, 1


def mem_type_of(t):
    return U.UCC_MEMORY_TYPE_CUDA if t.is_cuda else U.UCC_MEMORY_TYPE_HOST


class _TorchOob:
    """ucc_oob_coll_t whose allgather is a (blocking) gloo all_gather."""
    _ids = itertools.count(1)

    def __init__(self, group, rank, size, perm=None):
        self.group, self.rank, self.size = group, rank, size

        def allgather(src, recv, nbytes, info, req_pp):
            mine = torch.frombuffer(bytearray(C.string_at(src, nbytes)), dtype=torch.uint8).clone()
            outs = [torch.empty(nbytes, dtype=torch.uint8) for _ in range(self.size)]
            dist.all_gather(outs, mine, group=self.group)
            if perm is not None:          # UCC rank perm[g] is played by group rank g
                by_ucc = [None] * self.size
                for g, o in enumerate(outs):
                    by_ucc[perm[g]] = o
                outs = by_ucc
            flat = torch.cat(outs).contiguous()
            C.memmove(recv, flat.data_ptr(), nbytes * self.size)
            req_pp[0] = next(_TorchOob._ids)
            return U.UCC_OK

        self._ag = U.OOB_ALLGATHER_FN(allgather)
        self._test = U.OOB_REQ_FN(lambda req: U.UCC_OK)
        self._free = U.OOB_REQ_FN(lambda req: U.UCC_OK)

    def allgather_bytes(self, blob):
        """every member's `blob` (same length everywhere), through the same OOB allgather the library uses"""
        n = len(blob)
        src = C.create_string_buffer(bytes(blob), n)
        recv = C.create_string_buffer(n * self.size)
        req = (C.c_void_p * 1)()
        U.check(self._ag(C.cast(src, C.c_void_p).value, C.cast(recv, C.c_void_p).value, n, None, req), "oob allgather")
        return [recv.raw[r * n:(r + 1) * n] for r in range(self.size)]

    def struct(self):
        o = U.ucc_oob_coll_t()
        o.allgather, o.req_test, o.req_free = self._ag, self._test, self._free
        o.coll_info = None
        o.n_oob_eps, o.oob_ep = self.size, self.rank
        return o


class _StoreOob(_TorchOob):
    """ucc_oob_coll_t over a c10d Store (TCPStore / FileStore): used when ucc_b200 itself is the torch.distributed
    backend and no other process group exists yet."""

    def __init__(self, store, rank, size, prefix="ucc_b200_oob"):
        self.group, self.rank, self.size = None, rank, size
        self._seq = 0

        def allgather(src, recv, nbytes, info, req_pp):
            seq = self._seq
            self._seq += 1
            store.set(f"{prefix}/{seq}/{rank}", bytes(C.string_at(src, nbytes)))
            for r in range(size):
                C.memmove(recv + r * nbytes, store.get(f"{prefix}/{seq}/{r}"), nbytes)
            req_pp[0] = next(_TorchOob._ids)
            return U.UCC_OK

        self._ag = U.OOB_ALLGATHER_FN(allgather)
        self._test = U.OOB_REQ_FN(lambda req: U.UCC_OK)
        self._free = U.OOB_REQ_FN(lambda req: U.UCC_OK)


class MemHandles:
    """A registered segment: the local ucc_mem_map(EXPORT) handle plus one imported handle per team member (what collectives take
    as `global_memh`).  Keep it alive while requests that use it exist; `close()` unmaps everything."""

    def __init__(self, comm, tensor, local, imported, blobs):
        self.comm, self.tensor, self._local, self._imported, self._blobs = comm, tensor, local, imported, blobs
        self.array = (C.c_void_p * len(imported))(*[h.value for h in imported])

    def close(self):
        for h in self._imported:
            U.lib.ucc_mem_unmap(C.byref(h))
        U.lib.ucc_mem_unmap(C.byref(self._local))
        self._imported, self._blobs = [], []


_cu_capture_mode = None


@contextlib.contextmanager
def _relaxed_capture():
    """While the current stream captures a CUDA graph, progress polls the completion events of eager collectives
    (cudaEventQuery), which a capture in the default global mode forbids on every thread: switch this thread to relaxed mode
    for the duration, as PyTorch's own NCCL watchdog does."""
    global _cu_capture_mode
    if not (torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()):
        yield
        return
    if _cu_capture_mode is None:
        _cu_capture_mode = C.CDLL("libcuda.so.1").cuThreadExchangeStreamCaptureMode
        _cu_capture_mode.argtypes = [C.POINTER(C.c_int)]
    mode = C.c_int(2)   # CU_STREAM_CAPTURE_MODE_RELAXED
    _cu_capture_mode(C.byref(mode))
    try:
        yield
    finally:
        _cu_capture_mode(C.byref(mode))


def _overlap(a, on):
    """mark a request with UCC_COLL_ARGS_HINT_OPTIMIZE_OVERLAP_GPU"""
    if on:
        a.mask |= U.UCC_COLL_ARGS_FIELD_FLAGS
        a.flags |= U.UCC_COLL_ARGS_HINT_OPTIMIZE_OVERLAP_GPU
    return a


class Request:
    def __init__(self, comm, req, keep):
        self.comm, self.req, self._keep = comm, req, keep
        self._graphed = False      # owned by the communicator's graphed() cache: finalize() leaves it alone

    def post(self):
        U.check(U.ucc_collective_post(self.req), "collective_post")
        return self

    def post_on_stream(self, stream=None, wait_posted=True):
        """Stream-ordered post: the collective kernel is enqueued on `stream` (default: current).

        With `wait_posted` the call returns once UCC_EVENT_COLLECTIVE_POST was delivered, i.e. the kernel really is
        in the stream (a zero-copy collective first learns the peers' buffer mappings, which takes a few host
        microseconds); work enqueued on the stream afterwards is ordered behind the collective.

        Inside `torch.cuda.graph` the kernel is captured, not run: the post returns as soon as it is in the graph and the
        request completes at once.  Every replay of the graph runs the collective again."""
        if self._graphed and self.req.contents.status == U.UCC_INPROGRESS:
            self.wait()            # a persistent request is posted again only once its previous post completed
        ev = U.ucc_ev_t()
        ev.ev_type = U.UCC_EVENT_COMPUTE_COMPLETE
        ev.req = C.cast(self.req, C.c_void_p)
        self._ee = self.comm.ee_for(stream)
        self._seen_posted = False
        U.check(U.ucc_collective_triggered_post(self._ee, C.byref(ev)), "triggered_post")
        self.comm._unposted.add(self)
        if wait_posted:
            self.wait_posted()
        return self

    def wait_posted(self):
        """idempotent: returns at once when this post was already seen in the stream"""
        if getattr(self, "_seen_posted", False):
            return
        key = C.cast(self.req, C.c_void_p).value
        with _relaxed_capture():
            while key not in self.comm._posted:
                st = self.req.contents.status
                if st < 0:
                    raise U.UccError(st, "collective")
                if not self.comm.collect_events(self._ee):
                    U.ucc_context_progress(self.comm.ctx)
        self.comm._posted.discard(key)
        self.comm._unposted.discard(self)
        self._seen_posted = True

    def test(self):
        return self.req.contents.status

    def wait(self):
        with _relaxed_capture():
            while True:
                st = self.req.contents.status
                if st == U.UCC_OK:
                    return
                if st < 0:
                    raise U.UccError(st, "collective")
                U.ucc_context_progress(self.comm.ctx)

    def finalize(self):
        if self._graphed:
            return
        self._release()

    def _release(self):
        self.comm.drain_events()
        self.comm._unposted.discard(self)
        U.check(U.ucc_collective_finalize(self.req), "collective_finalize")
        self.req = None


class Communicator:
    """lib + context + one team spanning `group` (default: all ranks)."""

    def __init__(self, group=None, thread_mode=U.UCC_THREAD_SINGLE, lib_modify=(), ctx_modify=(), store=None, rank=None, size=None, perm=None,
                 fake_ppn=None, symm_size=None):
        """`perm[g]` = UCC rank of group rank g (default identity): lets a team use any rank order (e.g. reversed).
        `fake_ppn` (or env UCC_B200_FAKE_PPN): pretend the ranks are spread over nodes of that many processes each - a
        single-box way to exercise the hierarchical (cl/hier) schedules with real processes.
        `symm_size` (e.g. "2G"): reserve a symmetric user region in the tl/nvl team heap (UCC_TL_NVL_USER_SIZE); tensors from
        `symm_empty()` live there and are all-reduced in place through the NVSwitch (no staging, no copy-out)."""
        if store is not None:
            self.rank, self.size = rank, size
            self.oob = _StoreOob(store, rank, size)
        else:
            if not dist.is_initialized():
                raise RuntimeError("torch.distributed must be initialised (gloo is enough)")
            grank = dist.get_rank(group)
            self.size = dist.get_world_size(group)
            self.rank = perm[grank] if perm is not None else grank
            self.oob = _TorchOob(group, self.rank, self.size, perm)
        cfg = U.handle()
        U.check(U.ucc_lib_config_read(None, None, C.byref(cfg)), "lib_config_read")
        for k, v in lib_modify:
            U.check(U.ucc_lib_config_modify(cfg, k.encode(), v.encode()), "lib_config_modify")
        p = U.ucc_lib_params_t()
        p.mask, p.thread_mode = U.UCC_LIB_PARAM_FIELD_THREAD_MODE, thread_mode
        self.lib = U.handle()
        st = U.ucc_init_version(U.UCC_API_MAJOR, U.UCC_API_MINOR, C.byref(p), cfg, C.byref(self.lib))
        U.ucc_lib_config_release(cfg)
        U.check(st, "ucc_init")
        ccfg = U.handle()
        U.check(U.ucc_context_config_read(self.lib, None, C.byref(ccfg)), "context_config_read")
        if symm_size:
            ctx_modify = tuple(ctx_modify) + (("tl/nvl", "USER_SIZE", str(symm_size)),)
        for comp, name, val in ctx_modify:
            U.check(U.ucc_context_config_modify(ccfg, comp.encode() if comp else None, name.encode(), val.encode()), "ctx_modify")
        cp = U.ucc_context_params_t()
        if self.size > 1:
            cp.mask = U.UCC_CONTEXT_PARAM_FIELD_OOB
            cp.oob = self.oob.struct()
        self.ctx = U.handle()
        fake_ppn = fake_ppn or int(os.environ.get("UCC_B200_FAKE_PPN", "0"))
        if fake_ppn:
            from .harness import fake_proc_info
            pi = fake_proc_info(self.rank, fake_ppn)
            st = U.ucc_context_create_proc_info(self.lib, C.byref(cp), ccfg, C.byref(self.ctx), C.byref(pi))
        else:
            st = U.ucc_context_create(self.lib, C.byref(cp), ccfg, C.byref(self.ctx))
        U.ucc_context_config_release(ccfg)
        U.check(st, "context_create")
        tp = U.ucc_team_params_t()
        tp.mask = U.UCC_TEAM_PARAM_FIELD_EP | U.UCC_TEAM_PARAM_FIELD_EP_RANGE | U.UCC_TEAM_PARAM_FIELD_OOB
        tp.ep, tp.ep_range = self.rank, U.UCC_COLLECTIVE_EP_RANGE_CONTIG
        tp.oob = self.oob.struct()
        self.team = U.handle()
        ctxs = (U.handle * 1)(self.ctx)
        U.check(U.ucc_team_create_post(ctxs, 1, C.byref(tp), C.byref(self.team)), "team_create_post")
        while True:
            st = U.ucc_team_create_test(self.team)
            if st == U.UCC_OK:
                break
            U.check(st, "team_create_test")
            U.ucc_context_progress(self.ctx)
        self._ees = {}
        self._posted = set()
        self._unposted = set()     # stream-ordered posts whose kernel may not be in its stream yet
        self._graphing = 0
        self._graph_reqs = {}

    # ------------------------------------------------------------------ CUDA graphs
    @contextlib.contextmanager
    def graphed(self):
        """Collectives for a CUDA graph: use it around the warm-up iterations AND the capture.

            with comm.graphed():
                for _ in range(3):                      # warm-up, eager (on a side stream, as torch.cuda.graph wants)
                    step()
                with torch.cuda.graph(g):
                    step()
            g.replay()                                 # any number of times, on every member, in the same order

        Inside, every collective of this communicator (and of `ops` / the torch backend on top of it) is a persistent request,
        cached by its arguments: collective, buffer addresses, counts, datatype, operator, root.  The warm-up posts of a
        request resolve the zero-copy tables of the members' buffers, and the captured post reuses them, so the graph runs
        large collectives in place instead of staging them through the team heap.  A collective first posted under capture
        runs staged.  The requests stay alive, and the graph valid, until release_graphed() or destroy().  On entry, the
        collectives already posted are waited into their streams: a capture must not begin while a launch is still queued."""
        for r in list(self._unposted):
            r.wait_posted()
        self._graphing += 1
        try:
            yield self
        finally:
            self._graphing -= 1

    def release_graphed(self):
        """finalize the requests cached by graphed(); graphs captured from them must not be replayed any more"""
        reqs, self._graph_reqs = list(self._graph_reqs.values()), {}
        for r in reqs:
            r.wait()
            r._release()

    def take_device_error(self):
        """True when a tl/nvl kernel of this team gave up a device-side wait (UCC_TL_NVL_TIMEOUT) since the last call.  A
        replayed collective has no request to carry the error: call this after synchronizing the replay stream."""
        fn = getattr(self, "_dev_err_fn", None)
        if fn is None:
            fn = self._dev_err_fn = C.CDLL(os.path.join(os.path.dirname(U.LIB_PATH), "ucc", "libucc_tl_nvl.so")).ucc_tl_nvl_take_device_error
            fn.restype, fn.argtypes = C.c_int, [U.handle]
        return fn(self.team) == 1

    # ------------------------------------------------------------------ symmetric user memory (tl/nvl)
    def symm_region(self):
        """(base pointer, bytes, nvls) of the symmetric user region of this team's tl/nvl heap, or None"""
        if getattr(self, "_symm", None) is None:
            self._symm = False
            path = os.path.join(os.path.dirname(U.LIB_PATH), "ucc", "libucc_tl_nvl.so")
            try:
                fn = C.CDLL(path).ucc_tl_nvl_symm_region
            except (OSError, AttributeError):
                return None
            fn.restype = C.c_int
            fn.argtypes = [U.handle, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.POINTER(C.c_int)]
            base, size, nvls = C.c_void_p(), C.c_size_t(), C.c_int()
            if fn(self.team, C.byref(base), C.byref(size), C.byref(nvls)) == U.UCC_OK and base.value:
                self._symm = (base.value, size.value, bool(nvls.value))
                self._symm_off = 0
        return self._symm or None

    def symm_empty(self, shape, dtype=torch.float32):
        """Tensor inside the symmetric region (bump allocator, 256-byte aligned).  COLLECTIVE in spirit: every member must make
        the same sequence of calls so that a tensor sits at the same offset everywhere."""
        reg = self.symm_region()
        if reg is None:
            raise RuntimeError("no symmetric region: create the Communicator with symm_size=... (needs tl/nvl on CUDA devices)")
        shape = (shape,) if isinstance(shape, int) else tuple(shape)
        numel = 1
        for d in shape:
            numel *= d
        nbytes = numel * torch.empty((), dtype=dtype).element_size()
        off = (self._symm_off + 255) // 256 * 256
        if off + nbytes > reg[1]:
            raise MemoryError(f"symmetric region exhausted ({reg[1]} bytes)")
        self._symm_off = off + nbytes

        class _Raw:   # zero-copy view of device memory for torch.as_tensor
            __cuda_array_interface__ = {"shape": (max(nbytes, 1),), "typestr": "|u1", "data": (reg[0] + off, False), "version": 2}
        raw = torch.as_tensor(_Raw(), device=torch.device("cuda", torch.cuda.current_device()))
        return raw[:nbytes].view(dtype).view(shape)

    def request_info_last(self):
        """name and launch geometry of the tl/nvl kernel this process launched last ("" when tl/nvl is not loaded)"""
        fn = getattr(self, "_last_info_fn", None)
        if fn is None:
            try:
                fn = C.CDLL(os.path.join(os.path.dirname(U.LIB_PATH), "ucc", "libucc_tl_nvl.so")).ucc_tl_nvl_last_launch_info
                fn.restype = C.c_char_p
            except (OSError, AttributeError):
                fn = False
            self._last_info_fn = fn
        return fn().decode() if fn else ""

    def symm_reset(self):
        """forget every symm_empty() allocation (the tensors must no longer be used)"""
        self._symm_off = 0

    # ------------------------------------------------------------------ streams
    def ee_for(self, stream=None):
        s = stream if stream is not None else torch.cuda.current_stream()
        key = s.cuda_stream
        if key not in self._ees:
            ep = U.ucc_ee_params_t()
            ep.ee_type, ep.ee_context, ep.ee_context_size = U.UCC_EE_CUDA_STREAM, key, C.sizeof(C.c_void_p)
            ee = U.handle()
            U.check(U.ucc_ee_create(self.team, C.byref(ep), C.byref(ee)), "ee_create")
            self._ees[key] = ee
        return self._ees[key]

    def collect_events(self, ee):
        """Move pending EE events into the bookkeeping sets; returns how many were seen."""
        n = 0
        ev = C.POINTER(U.ucc_ev_t)()
        while U.ucc_ee_get_event(ee, C.byref(ev)) == U.UCC_OK:
            if ev.contents.ev_type == U.UCC_EVENT_COLLECTIVE_POST and ev.contents.req:
                self._posted.add(ev.contents.req)
            U.ucc_ee_ack_event(ee, ev)
            n += 1
        return n

    def drain_events(self):
        for ee in self._ees.values():
            self.collect_events(ee)
        if len(self._posted) > 4096:
            self._posted.clear()

    def progress(self):
        U.ucc_context_progress(self.ctx)

    # ------------------------------------------------------------------ collectives
    def init(self, args, hold=()):
        r = C.POINTER(U.ucc_coll_req_t)()
        U.check(U.ucc_collective_init(C.byref(args), C.byref(r), self.team), "collective_init")
        return Request(self, r, (args, hold))   # `hold` keeps the tensors alive until the request is finalized

    def _init_cached(self, key, make_args, hold):
        """init() outside graphed(); inside, the persistent request cached under `key` (created on first use)"""
        if not self._graphing:
            return self.init(make_args(False), hold)
        req = self._graph_reqs.get(key)
        if req is None:
            req = self.init(make_args(True), hold)
            req._graphed = True
            self._graph_reqs[key] = req
        return req

    @staticmethod
    def _graph_key(coll, src, dst, kw):
        def desc(t):
            return None if t is None else (t.data_ptr(), t.numel(), t.dtype, str(t.device))
        return (coll, desc(src), desc(dst)) + tuple(sorted((k, tuple(v) if isinstance(v, (list, tuple)) else v) for k, v in kw.items()))

    def _args(self, coll, src=None, dst=None, op="sum", root=0, inplace=False, persistent=False, **kw):
        from .harness import coll_args
        ref = dst if dst is not None else src
        if ref is None:  # barrier / fanin / fanout
            return coll_args(coll, root=root, persistent=persistent)
        dt, op, width = op_of(op, ref) if coll in REDUCTIONS else (dt_of(ref), op, 1)
        if width != 1:   # counts and displacements in library elements
            kw = {k: [c * width for c in v] if k in ("src_counts", "src_displs", "dst_counts", "dst_displs") and v is not None else v
                  for k, v in kw.items()}
        return coll_args(coll, dt=dt, op=op, root=root, inplace=inplace, persistent=persistent,
                         src_ptr=src.data_ptr() if src is not None else None, dst_ptr=dst.data_ptr() if dst is not None else None,
                         count_src=src.numel() * width if src is not None else 0, count_dst=dst.numel() * width if dst is not None else 0,
                         mem_type=mem_type_of(ref), **kw)

    def register(self, tensor):
        """ucc_mem_map: register the memory of `tensor` (a whole segment; collectives may later use any part of it, at the same
        offset on every member) with every TL that supports registration - tl/nvl for CUDA memory (zero-copy kernels without
        the per-post buffer exchange), tl/shm for host memory (put-based one-sided alltoall) - exchange the relocatable handles
        over the team's OOB channel and import every member's.  Collective on the team.  Returns MemHandles for
        `coll_init(..., src_memh= / dst_memh=)`."""
        U.lib.ucc_mem_map.argtypes = [U.handle, C.c_int, C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_void_p)]
        U.lib.ucc_mem_map.restype = C.c_int
        U.lib.ucc_mem_unmap.argtypes = [C.POINTER(C.c_void_p)]
        U.lib.ucc_mem_unmap.restype = C.c_int
        seg = U.ucc_mem_map_t(tensor.data_ptr(), tensor.numel() * tensor.element_size())
        params = U.ucc_mem_map_params_t()
        params.segments, params.n_segments = C.pointer(seg), 1
        local, size = C.c_void_p(), C.c_size_t()
        U.check(U.lib.ucc_mem_map(self.ctx, 0, C.byref(params), C.byref(size), C.byref(local)), "ucc_mem_map export")
        mine = C.string_at(local.value, size.value)
        sizes = [int.from_bytes(b, "little") for b in self.oob.allgather_bytes(len(mine).to_bytes(8, "little"))]
        width = max(sizes)
        blobs = [C.create_string_buffer(b[:sizes[r]], sizes[r]) for r, b in enumerate(self.oob.allgather_bytes(mine.ljust(width, b"\0")))]
        imported = []
        for b in blobs:   # the imported handle lives inside the received buffer (kept in MemHandles)
            h = C.c_void_p(C.addressof(b))
            U.check(U.lib.ucc_mem_map(self.ctx, 1, None, None, C.byref(h)), "ucc_mem_map import")
            imported.append(h)
        return MemHandles(self, tensor, local, imported, blobs)

    def allreduce_init(self, src, dst, op="sum", persistent=False, overlap_gpu=False):
        inplace = src is None or src.data_ptr() == dst.data_ptr()
        s = None if inplace else src

        def make(p):
            return _overlap(self._args("allreduce", s, dst, op=op, inplace=inplace, persistent=persistent or p), overlap_gpu)
        return self._init_cached(self._graph_key("allreduce", s, dst, {"op": op, "overlap_gpu": bool(overlap_gpu)}), make, (src, dst))

    def coll_init(self, coll, src=None, dst=None, src_memh=None, dst_memh=None, overlap_gpu=False, **kw):
        """`src_memh` / `dst_memh`: MemHandles from register() - the buffers are parts of registered segments.
        `overlap_gpu`: the request carries UCC_COLL_ARGS_HINT_OPTIMIZE_OVERLAP_GPU - on tl/nvl, data crosses NVLink by the copy
        engines and the SMs stay free for kernels that run next to the collective (docs/user_guide.md)"""
        def make(persistent):
            a = _overlap(self._args(coll, src, dst, **dict(kw, persistent=kw.get("persistent", False) or persistent)), overlap_gpu)
            if src_memh is not None:
                a.mask |= U.UCC_COLL_ARGS_FIELD_MEM_MAP_SRC_MEMH | U.UCC_COLL_ARGS_FIELD_FLAGS
                a.flags |= U.UCC_COLL_ARGS_FLAG_SRC_MEMH_GLOBAL
                a.src_memh.global_memh = C.cast(src_memh.array, C.POINTER(C.c_void_p))
            if dst_memh is not None:
                a.mask |= U.UCC_COLL_ARGS_FIELD_MEM_MAP_DST_MEMH | U.UCC_COLL_ARGS_FIELD_FLAGS
                a.flags |= U.UCC_COLL_ARGS_FLAG_DST_MEMH_GLOBAL
                a.dst_memh.global_memh = C.cast(dst_memh.array, C.POINTER(C.c_void_p))
            return a
        key = self._graph_key(coll, src, dst, dict(kw, src_memh=id(src_memh), dst_memh=id(dst_memh), overlap_gpu=bool(overlap_gpu)))
        return self._init_cached(key, make, (src, dst, src_memh, dst_memh))

    def run(self, req, stream=None):
        """Convenience: post, wait (host), finalize."""
        (req.post_on_stream(stream) if stream is not None else req.post()).wait()
        req.finalize()

    def barrier(self):
        self.run(self.coll_init("barrier"))

    def destroy(self):
        self.release_graphed()
        for ee in self._ees.values():
            U.ucc_ee_destroy(ee)
        self._ees = {}
        self._posted = set()
        while True:
            st = U.ucc_team_destroy(self.team)
            if st != U.UCC_INPROGRESS:
                break
            U.ucc_context_progress(self.ctx)
        U.ucc_context_destroy(self.ctx)
        U.ucc_finalize(self.lib)


def init_distributed(backend="cpu:gloo,cuda:nccl"):
    """Initialise torch.distributed from the torchrun environment and bind this rank's GPU."""
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    lrank = int(os.environ.get("LOCAL_RANK", str(rank)))
    if torch.cuda.is_available():
        torch.cuda.set_device(lrank % torch.cuda.device_count())
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29555")
    if not dist.is_initialized():
        if not torch.cuda.is_available():
            backend = "gloo"
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, world, lrank
