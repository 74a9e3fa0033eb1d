"""UCC_COLL_ARGS_HINT_OPTIMIZE_OVERLAP_GPU on tl/nvl: the cases shared by the host-emulated worker (tests/hostemu_overlap_worker.py)
and the GPU test (tests/test_nvl_overlap_gpu.py).

With the hint, allreduce and reduce_scatter(v) take the copy-engine reduction (launch note `reduce_copy_engine`, a fixed grid of
NVL_LOCAL_CTAS CTAs), bcast / gather(v) / scatter(v) the copy-engine exchange (`exchange_copy_engine`), allgather(v) / alltoall(v)
the copy-engine push (`exchange_push_copy_engine`), a team of one cudaMemcpyAsync.  Where the members' buffers do not resolve
(managed memory, a captured post without cached tables) every member runs the ordinary staged kernel of the collective; reduce,
in-place alltoall(v) and send / recv keep their ordinary paths.

Every reduction runs twice on the same buffers: without the hint (the zero-copy two-shot kernel, UCC_TL_NVL_TUNE / ZCOPY from
nvl_numerics.path_env("zcopy")) and with it; the two must agree bit for bit, guard bands included, and the hinted result must meet
the contract of tests/nvl_numerics.py.  Data movement is checked byte for byte against numpy on int32 data.

`h` provides: mem.alloc(nbytes) -> uint8 buffer (.ptr, .write, .read); alloc(nelems, managed) -> int32 buffer; args(coll, s, d,
smt, dmt, **coll_args keywords); nargs(coll, src_ptr, dst_ptr, dt, **kw); run(team, args); last_launch(); sync()."""
import ctypes as C

import numpy as np

from ucc_b200 import capi as U
import nvl_managed as M
import nvl_numerics as V

CUDA, MANAGED = U.UCC_MEMORY_TYPE_CUDA, U.UCC_MEMORY_TYPE_CUDA_MANAGED
HINT = U.UCC_COLL_ARGS_HINT_OPTIMIZE_OVERLAP_GPU
RED_CE, XCHG_CE, PUSH_CE = "reduce_copy_engine", "exchange_copy_engine", "exchange_push_copy_engine"
LOCAL_CTAS = 8                                   # NVL_LOCAL_CTAS of kernels/nvl_kernels.h
# the environment of the reduction cases: TUNE twoshot with zero-copy from 0 bytes, so a request without the hint is the reference
ENV = dict(V.path_env("zcopy"), UCC_TL_NVL_SYMMETRIC_SIZE="8Mb")
SMALL, LARGE = 37, 70000                         # int32 elements per block: 148 B and 280 KB (a v-form of 4 members: > 1 MB)
CE_NOTE = {"allreduce": RED_CE, "reduce_scatter": RED_CE, "reduce_scatterv": RED_CE, "bcast": XCHG_CE, "gather": XCHG_CE,
           "gatherv": XCHG_CE, "scatter": XCHG_CE, "scatterv": XCHG_CE, "allgather": PUSH_CE, "allgatherv": PUSH_CE,
           "alltoall": PUSH_CE, "alltoallv": PUSH_CE}


def hint(a, on=True):
    if on:
        a.mask |= U.UCC_COLL_ARGS_FIELD_FLAGS
        a.flags |= HINT
    else:
        a.flags &= ~HINT
    return a


def check_ce_note(note, coll, what):
    want = CE_NOTE[coll]
    assert note.startswith(want + " "), (what, "not served by the copy-engine path", note)
    if want == RED_CE:
        assert note.split()[1].startswith(f"{LOCAL_CTAS}x"), (what, "the local reduction runs on a fixed grid", note)
    if want == XCHG_CE:
        assert note.split()[1] == "1x32", (what, "only the one-CTA barrier kernel runs on the SMs", note)


# ------------------------------------------------------------------ reductions: numerics and bitwise equality with twoshot_zcopy
class Twin:
    """nvl_numerics.Harness whose run() posts the request first WITHOUT the hint (the zero-copy two-shot reference), restores every
    buffer of the case, posts it WITH the hint and checks that both left every buffer bit for bit the same.  last_launch() is the
    hinted run's note as nvl_numerics expects it for the zero-copy path: the copy-engine direct form stands where twoshot_zcopy
    would, its staged form is twoshot_staged."""

    def __init__(self, h):
        self.h, self.bufs, self.note, self.ncases = h, [], None, 0
        self.mem = self
        self.args = h.nargs

    def alloc(self, nbytes):
        b = self.h.mem.alloc(nbytes)
        self.bufs.append(b)
        return b

    def run(self, team, args):
        snap = [b.read() for b in self.bufs]
        for a in args:
            hint(a, False)
        self.h.run(team, args)
        ref_note = self.h.last_launch()
        ref = [b.read() for b in self.bufs]
        for b, s in zip(self.bufs, snap):
            b.write(s)
        for a in args:
            hint(a, True)
        self.h.run(team, args)
        self.note = self.h.last_launch()
        for i, (b, want) in enumerate(zip(self.bufs, ref)):
            got = b.read()
            if not np.array_equal(got, want):
                d = np.flatnonzero(got != want)
                raise V.Violation(f"buffer {i}: {d.size} bytes differ from the run without the hint ({ref_note}) under `{self.note}`, "
                                  f"e.g. at {d[:4].tolist()}")
        self.bufs = []
        self.ncases += 1

    def last_launch(self):
        n = self.note
        if n.startswith("twoshot_zcopy"):
            return "the hint was ignored: " + n
        if n.startswith(RED_CE + " "):
            assert n.split()[1].startswith(f"{LOCAL_CTAS}x"), n
            return "twoshot_zcopy(direct) " + n.split()[1]
        return n


def run_numerics(h, team, n, dtypes, count=4097, seed=0):
    """allreduce, reduce_scatter and reduce_scatterv: every datatype of `dtypes` with every operator it has, the counts where
    vector kernels go wrong, one element off alignment (staged), in place and an empty block; returns the number of cases"""
    t = Twin(h)
    for coll in ("allreduce", "reduce_scatter", "reduce_scatterv"):
        blk = count if coll == "allreduce" else count // n + 1
        for dt in dtypes:
            sz, e = V.SIZE[dt], 16 // V.SIZE[dt]
            rsv = [e * (blk // e + 3 * r) for r in range(n)]       # unequal blocks, each starting 16-byte aligned: the direct form
            for op in V.ops_of(dt):
                seed += 1
                V.run_case(t, team, n, coll, "zcopy", dt, op, blk, seed, rs_counts=rsv)
            seed += 1
            if coll == "reduce_scatterv":      # an empty block (aligned: direct), odd blocks (staged), one element off alignment
                V.run_case(t, team, n, coll, "zcopy", dt, "sum", None, seed, rs_counts=[0 if r == n // 2 else 3 * e * (r + 1) for r in range(n)])
                V.run_case(t, team, n, coll, "zcopy", dt, "sum", None, seed + 2, rs_counts=[0 if r == n // 2 else e * r + 1 for r in range(n)])
                V.run_case(t, team, n, coll, "zcopy", dt, "sum", None, seed + 1, rs_counts=[e + r for r in range(n)], mis=sz % 16)
                continue
            for c in V.small_counts(dt, n):
                V.run_case(t, team, n, coll, "zcopy", dt, "sum", c, seed)
            if sz < 16:
                V.run_case(t, team, n, coll, "zcopy", dt, "sum", blk, seed + 1, mis=sz)
            V.run_case(t, team, n, coll, "zcopy", dt, V.ops_of(dt)[-1], blk, seed + 2, inplace=True)
    return t.ncases


def run_rounds(h, team, n, symm):
    """reductions larger than the data region of the heap (`symm` bytes): the copy-engine form runs in three or more rounds"""
    t = Twin(h)
    for coll in ("allreduce", "reduce_scatter", "reduce_scatterv"):
        for dt in ("float32", "bfloat16"):
            sz, e = V.SIZE[dt], 16 // V.SIZE[dt]
            # my slice / block: 3.5 times what one peer's part of the data region holds, blocks 16-byte aligned, a ragged allreduce
            blk = int(3.5 * (symm // (n - 1))) // sz // e * e
            V.run_case(t, team, n, coll, "zcopy", dt, "sum", blk * n + 7 if coll == "allreduce" else blk, 5000 + n,
                       rs_counts=[blk + e * r for r in range(n)], classes=(V.EXACT_T, V.EXACT_ACC, V.RANDOM))
            assert t.note.startswith(RED_CE), t.note
    return t.ncases


# ------------------------------------------------------------------ data movement and the hint's reach
def _hinted(h):
    class HH:
        mem = getattr(h, "mem", None)
        alloc = staticmethod(h.alloc)
        last_launch = staticmethod(h.last_launch)
        run = staticmethod(h.run)

        @staticmethod
        def args(*a, **kw):
            return hint(h.args(*a, **kw))
    return HH


MOVE = ("bcast", "gather", "gatherv", "scatter", "scatterv", "allgather", "allgatherv", "alltoall", "alltoallv")


def run_colls(h, team, n, seed=0):
    """every collective of the table, below and above 1 MB, in place where UCC defines it, on device buffers: the copy-engine
    direct form and the exact result; reduce and in-place alltoall(v) keep their ordinary paths"""
    hh, k = _hinted(h), 0
    for coll in MOVE + ("allreduce", "reduce_scatter", "reduce_scatterv", "reduce"):
        for blk in (SMALL, LARGE):
            for ip in (False, True) if M.inplace_ok(coll) else (False,):
                c = M.Case(hh, n, coll, blk, ("d", "d"), ip, seed + 1000 * k, root=(k % n)).build()
                h.run(team, c.args)
                note, what = h.last_launch(), (coll, n, blk, "inplace" if ip else "")
                if coll == "reduce":
                    assert "copy_engine" not in note, (what, "reduce has no copy-engine form", note)
                elif ip and coll in ("alltoall", "alltoallv"):
                    assert note.startswith(("exchange_swap", "exchange_pull_staged_inplace")), (what, note)
                elif coll.startswith("reduce_scatter") and any(4 * o % 16 for o in np.cumsum(
                        [blk + 3 * r if coll == "reduce_scatterv" else blk for r in range(n)])[:-1]):
                    # blocks that do not start 16-byte aligned: the staged kernel, as for twoshot_zcopy
                    assert note.startswith("twoshot_staged"), (what, note)
                else:
                    check_ce_note(note, coll, what)
                c.check()
                k += 1
    return k


def _v_case(h, n, coll, counts, root, seed):
    """a v-form with zero-length and odd blocks; returns (args, [(dst buffer, expected)], every buffer: keep them alive)"""
    g = np.random.default_rng(seed)
    displs = [int(x) for x in np.concatenate([[0], np.cumsum(counts)[:-1]])]
    tot = sum(counts)
    args, check, keep = [], [], []
    if coll in ("allgatherv", "gatherv"):
        blocks = [g.integers(-99, 99, counts[r]).astype(np.int32) for r in range(n)]
        for r in range(n):
            s = h.alloc(max(counts[r], 1), False)
            s.write(blocks[r])
            has = coll == "allgatherv" or r == root
            d = h.alloc(tot + 8, False) if has else None
            keep += [s, d]
            if d is not None:
                d.write(np.full(tot + 8, 7, np.int32))
                check.append((d, np.concatenate(blocks + [np.full(8, 7, np.int32)])))
            kw = dict(dst_counts=counts, dst_displs=displs) if has else {}
            args.append(h.args(coll, s, d, CUDA, CUDA, count_src=counts[r], count_dst=tot if has else 0, root=root, **kw))
    elif coll == "scatterv":
        whole = g.integers(-99, 99, tot).astype(np.int32)
        for r in range(n):
            s = None
            if r == root:
                s = h.alloc(tot, False)
                s.write(whole)
            d = h.alloc(counts[r] + 8, False)
            d.write(np.full(counts[r] + 8, 7, np.int32))
            keep += [s, d]
            check.append((d, np.concatenate([whole[displs[r]:displs[r] + counts[r]], np.full(8, 7, np.int32)])))
            kw = dict(src_counts=counts, src_displs=displs) if r == root else {}
            args.append(h.args(coll, s, d, CUDA, CUDA, count_src=tot if r == root else 0, count_dst=counts[r], root=root, **kw))
    return args, check, keep


def run_vforms(h, team, n):
    """allgatherv / gatherv / scatterv with zero-length and odd blocks, every root"""
    hh, k = _hinted(h), 0
    for coll in ("allgatherv", "gatherv", "scatterv"):
        for root in range(n):
            counts = [0 if r == (root + 1) % n else 2 * r + 1 + (LARGE if r == root else 0) for r in range(n)]
            args, check, _keep = _v_case(hh, n, coll, counts, root, 40 + k)
            h.run(team, args)
            check_ce_note(h.last_launch(), coll, (coll, n, root, counts))
            for i, (d, want) in enumerate(check):
                got = d.read()[:len(want)]
                bad = np.flatnonzero(got != want)
                assert not bad.size, (coll, n, root, counts, "buffer", i, "differs at", bad[:4].tolist(), "of", bad.size, got[bad[:4]].tolist(), want[bad[:4]].tolist())
            k += 1
    return k


def run_persistent(h, team, n):
    """persistent requests posted three times with new inputs: the first post resolves the tables, the others reuse them"""
    hh, k = _hinted(h), 0
    for coll in ("allreduce", "reduce_scatter", "bcast", "gatherv", "scatter", "allgather"):
        c = M.Case(hh, n, coll, LARGE, ("d", "d"), False, 300 + k, 0).build()
        for a in c.args:
            a.flags |= U.UCC_COLL_ARGS_FLAG_PERSISTENT
        q = team.coll(c.args)
        for it in range(3):
            for r in range(n):
                if c.src[r] is not None:
                    cur = c.src[r].read()
                    c.src[r].write(cur + np.int32(it + 1))
            h.sync()
            assert q.run() == U.UCC_OK
            h.sync()
            check_ce_note(h.last_launch(), coll, (coll, "persistent", it))
            _check_shift(c, coll, n, it)
        q.finalize()
        k += 1
    return k


def _check_shift(c, coll, n, it):
    """after post `it` every source element grew by 1 + 2 + ... + (it + 1): the expected results shift accordingly"""
    s = (it + 1) * (it + 2) // 2
    for r, e in c.exp.items():
        e = e[1] if isinstance(e, tuple) else e
        add = s * n if coll in ("allreduce", "reduce_scatter") else s
        got = c.src[r].read() if coll == "bcast" else c.dst[r].read()
        assert np.array_equal(got[:len(e)], e + np.int32(add)), (coll, "persistent", it, r)


def run_fallbacks(h, team, n):
    """managed buffers make every member run the ordinary staged kernel, with the exact result"""
    hh, k = _hinted(h), 0
    for coll in ("allreduce", "reduce_scatter", "bcast", "gather", "scatter", "allgather", "alltoall"):
        c = M.Case(hh, n, coll, LARGE, ("m", "m"), False, 600 + k, 0).build()
        h.run(team, c.args)
        note = h.last_launch()
        assert note.startswith(("twoshot_staged", "exchange_pull_staged")), (coll, "managed source", note)
        c.check()
        k += 1
    return k


def run_registered(h, team, n, ctxs):
    """allreduce and bcast on registered segments (ucc_mem_map GLOBAL handles): the tables come from the registrations at init,
    three posts of a persistent request run the copy-engine form"""
    lib = U.lib
    lib.ucc_mem_map.argtypes = [U.handle, C.c_int, C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_void_p)]
    lib.ucc_mem_map.restype = C.c_int
    cnt = LARGE
    keep = []

    def register(bufs):
        blobs = []
        for r in range(n):
            seg = U.ucc_mem_map_t(bufs[r].ptr, 2 * cnt * 4)
            p = U.ucc_mem_map_params_t()
            p.segments, p.n_segments = C.pointer(seg), 1
            memh, size = C.c_void_p(), C.c_size_t()
            assert lib.ucc_mem_map(ctxs[r], 0, C.byref(p), C.byref(size), C.byref(memh)) == U.UCC_OK
            blobs.append(C.string_at(memh.value, size.value))
        glob = []
        for r in range(n):
            arr = (C.c_void_p * n)()
            for p in range(n):
                b = C.create_string_buffer(blobs[p], len(blobs[p]))
                keep.append(b)
                hd = C.c_void_p(C.addressof(b))
                assert lib.ucc_mem_map(ctxs[r], 1, None, None, C.byref(hd)) == U.UCC_OK
                arr[p] = hd.value
            keep.append(arr)
            glob.append(arr)
        return glob

    src = [h.alloc(2 * cnt, False) for _ in range(n)]
    dst = [h.alloc(2 * cnt, False) for _ in range(n)]
    gs, gd = register(src), register(dst)
    g = np.random.default_rng(77)
    args = []
    for r in range(n):
        dst[r].write(np.zeros(2 * cnt, np.int32))
        a = h.args("allreduce", src[r], dst[r], CUDA, CUDA, count_src=cnt, count_dst=cnt)
        a.src.info.buffer, a.dst.info.buffer = src[r].ptr + cnt * 4, dst[r].ptr + cnt * 4
        a.mask |= U.UCC_COLL_ARGS_FIELD_MEM_MAP_SRC_MEMH | U.UCC_COLL_ARGS_FIELD_MEM_MAP_DST_MEMH | U.UCC_COLL_ARGS_FIELD_FLAGS
        a.flags |= U.UCC_COLL_ARGS_FLAG_SRC_MEMH_GLOBAL | U.UCC_COLL_ARGS_FLAG_DST_MEMH_GLOBAL | U.UCC_COLL_ARGS_FLAG_PERSISTENT
        a.src_memh.global_memh = C.cast(gs[r], C.POINTER(C.c_void_p))
        a.dst_memh.global_memh = C.cast(gd[r], C.POINTER(C.c_void_p))
        args.append(hint(a))
    q = team.coll(args)
    for it in range(3):
        ins = [g.integers(-50, 50, 2 * cnt).astype(np.int32) for _ in range(n)]
        for r in range(n):
            src[r].write(ins[r])
        h.sync()
        assert q.run() == U.UCC_OK
        h.sync()
        check_ce_note(h.last_launch(), "allreduce", ("registered", it))
        exp = sum(x[cnt:].astype(np.int64) for x in ins).astype(np.int32)
        for r in range(n):
            got = dst[r].read()
            assert np.array_equal(got[cnt:], exp) and not got[:cnt].any(), ("registered allreduce", it, r)
    q.finalize()
    return 3


def run_self(h, team):
    """a team of one: device buffers take cudaMemcpyAsync at every size, a managed side the thread copy"""
    hh, k = _hinted(h), 0
    for blk in (SMALL, LARGE):
        for mix, want in ((("d", "d"), "self_copy(cudaMemcpyAsync)"), (("m", "d"), "self_copy "), (("d", "m"), "self_copy ")):
            for coll in ("allreduce", "allgather", "alltoall"):
                c = M.Case(hh, 1, coll, blk, mix, False, 900 + k, 0).build()
                h.run(team, c.args)
                assert h.last_launch().startswith(want), (coll, blk, mix, h.last_launch())
                c.check()
                k += 1
    return k
