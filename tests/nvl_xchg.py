"""The byte contract of the tl/nvl data-movement collectives (allgather(v), alltoall(v), bcast, gather(v), scatter(v)) with a plain
numpy reference and seeded layouts.  Shared by the GPU test (tests/test_nvl_xchg_gpu.py) and the host-emulation worker
(tests/hostemu_xchg_worker.py); the contract is written down in tests/README.md.

Every buffer a case touches - sources, destinations, root-only buffers and the buffers a non-root passes but may not use - is a
`Placed` buffer: its data region sits at a chosen distance from 16-byte alignment between two 64-byte guard bands, and all of it
starts as seeded random bytes.  The reference is the image every such buffer must have afterwards: the initial bytes with exactly
the blocks the caller has to receive copied in.  A case fails on the first byte that differs, naming the buffer, the byte range
and what lies there (a block of some rank, a gap between blocks, a guard band)."""
import ctypes as C

import numpy as np

from nvl_numerics import Harness, Placed, Violation  # noqa: F401  (Harness: what the test files build a case's surroundings with)

# one datatype per element size: the movers ignore the type, the displacement scale does not
ELEM = {"uint8": 1, "bfloat16": 2, "int32": 4, "float64": 8, "float64_complex": 16}
DTYPES = list(ELEM)
MIS = (0, 1, 4, 8)              # distance of every data region from 16-byte alignment
LAYOUTS = ("contiguous", "permuted", "gapped", "zeros", "skewed", "tail")
FIXED_LAYOUTS = ("contiguous", "tail")    # allgather / alltoall / bcast / gather / scatter: one block size, rank order
TMA_STAGE = 24 * 1024           # kernels/nvl_bulk.cuh NVL_BULK_STAGE_BYTES
TABLE_BYTES = 256               # kernels/nvl_kernels.h NVL_XCHG_TABLE_BYTES: the heap's offset table in front of the staged payload
VCOLLS = ("allgatherv", "alltoallv", "gatherv", "scatterv")
ROOTED = ("bcast", "gather", "gatherv", "scatter", "scatterv")
FAMILIES = {"allgather": ("allgather", "allgatherv"), "alltoall": ("alltoall", "alltoallv"), "bcast": ("bcast",),
            "gather": ("gather", "gatherv"), "scatter": ("scatter", "scatterv")}

# path -> (TUNE algorithm, collective families it serves, environment)
_ZC = {"UCC_TL_NVL_ZCOPY": "y", "UCC_TL_NVL_ZCOPY_THRESH": "0"}
PATHS = {
    "staged": ("pull", tuple(FAMILIES), {"UCC_TL_NVL_ZCOPY": "n"}),
    "zcopy": ("pull", tuple(FAMILIES), _ZC),
    "push": ("push", ("allgather", "alltoall"), dict(_ZC, UCC_TL_NVL_BULK="n")),
    "push_bulk": ("push", ("allgather", "alltoall"), dict(_ZC, UCC_TL_NVL_BULK="y", UCC_TL_NVL_BULK_THRESH="0", UCC_TL_NVL_BULK_CTAS="3")),
    "ce": ("ce", ("allgather", "alltoall"), _ZC),
    "ring": ("ring", ("allgather",), {"UCC_TL_NVL_ZCOPY": "n"}),
    "self": ("pull", tuple(FAMILIES), {"UCC_TL_NVL_ZCOPY": "n"}),
}


def path_env(path):
    alg, fams, extra = PATHS[path]
    tune = "#".join(f"{c}:cuda:inf:@{alg}" for f in fams for c in FAMILIES[f])
    return dict(extra, UCC_TL_NVL_TUNE=tune, UCC_TLS="nvl")


def inplace_allowed(path, coll):
    """in place where UCC defines it and the path serves it: allgather(v) and gather(v) / scatter(v) at the root everywhere;
    alltoall(v) on the pull paths (staged: the staged in-place kernel, zero-copy: the pairwise swap)"""
    if path in ("push", "push_bulk", "ce"):
        return False
    if coll in ("alltoall", "alltoallv"):
        return path in ("staged", "zcopy", "self")
    return coll != "bcast"


def want_note(path, coll, inplace):
    """the kernel that must serve (path, coll): the launch notes of tests/golden/nvl_launch_paths.txt.  In these single-process
    jobs every buffer resolves for the zero-copy kernels (the heap and the buffers live in one address space), so a staged note on a
    zero-copy path is a silent fallback and fails; a team of one copies with the self-copy kernel"""
    a2a_ip = inplace and coll in ("alltoall", "alltoallv")
    return {"staged": "exchange_pull_staged_inplace" if a2a_ip else "exchange_pull_staged",
            "zcopy": "exchange_swap" if a2a_ip else "exchange_pull_zcopy",
            "push": "exchange_push", "push_bulk": "exchange_push_bulk(tma)", "ce": "exchange_push_copy_engine",
            "ring": "exchange_ring", "self": "self_copy"}[path]


# ------------------------------------------------------------------ layouts
def big_count(sz, g, ragged):
    """a block of more than 3 TMA stages whose last stage is short; ragged: its byte length is also no multiple of 16"""
    nbytes = 3 * TMA_STAGE + 16 * int(g.integers(1, TMA_STAGE // 16))
    c = nbytes // sz
    return c + 1 if ragged and sz < 16 else c


def _small(e, g, k):
    return g.integers(1, 3 * e + 40, k)


def block_counts(layout, n, sz, g, rep, own=None):
    """counts (elements) of the n blocks of one side of a v-collective.  own: the caller's rank where the blocks are private to it
    (alltoallv rows), None where every rank sees the same counts"""
    e = 16 // sz
    c = _small(e, g, n)
    if layout == "zeros":
        if rep == 0:           # zero-count blocks first, last and at the caller's own rank (or at a middle rank)
            z = {0, n - 1, own if own is not None else n // 2}
            if len(z) == n:
                z.discard(n - 1 if n > 1 else 0)
            c[sorted(z)] = 0
        else:                  # all but one
            keep = int(g.integers(n))
            c[:] = 0
            c[keep] = _small(e, g, 1)[0]
    elif layout == "skewed":   # one hot receiver (the MoE shape)
        c = g.integers(0, e + 3, n)
        c[int(g.integers(n))] = 40 * e + int(g.integers(0, 5 * e))
    elif layout == "tail":     # E-1, E, E+1 of the 16-byte vector, and blocks of more than 3 TMA stages
        c = g.choice([e - 1, e, e + 1], n)
        hot = 0 if rep == 0 else int(g.integers(n))    # (first run: the whole-vector block at displacement 0, where TMA takes it)
        c[hot] = big_count(sz, g, ragged=False)
        if n > 2:
            c[(hot + 1) % n] = big_count(sz, g, ragged=True)
    return c.astype(np.int64)


def place(layout, counts, g):
    """displacements (elements) of blocks with these counts, and the extent of the buffer: rank order, another order (`permuted`)
    or holes of 1..40 elements between the blocks and after the last one (`gapped`)"""
    n = len(counts)
    order = list(range(n))
    if layout == "permuted" and n > 1:
        while order == sorted(order):
            order = [int(x) for x in g.permutation(n)]
    gaps = g.integers(1, 41, n) if layout == "gapped" else np.zeros(n, np.int64)
    displ = np.zeros(n, np.int64)
    off = 0
    for p in order:
        displ[p] = off
        off += int(counts[p]) + int(gaps[p])
    return displ, off


def fixed_count(layout, n, sz, g, rep):
    """the block count of a collective without v-arguments"""
    e = 16 // sz
    if layout == "tail":       # first run: whole vectors over more than 3 TMA stages, the last one short; then a vector-sized tail
        return big_count(sz, g, ragged=False) if rep == 0 else [max(e - 1, 1), e, e + 1, big_count(sz, g, ragged=True)][int(g.integers(4))]
    return int(_small(e, g, 1)[0])


# ------------------------------------------------------------------ arguments
def make_args(h, coll, sp, dp, dt, width, n, **kw):
    """the harness's arguments; width 32: the counts and displacements as 32-bit arrays, without the 64-bit flags"""
    a = h.args(coll, sp, dp, dt, **kw)
    if width == 32:
        from ucc_b200 import capi as U
        keep = []
        for side in ("src", "dst"):
            if kw.get(f"{side}_counts") is None:
                continue
            iv = getattr(a, side).info_v
            for field, k in (("counts", "counts"), ("displacements", "displs")):
                arr = np.ascontiguousarray(kw[f"{side}_{k}"], np.uint32)
                keep.append(arr)
                setattr(iv, field, arr.ctypes.data)
        if keep:
            a.flags &= ~(U.UCC_COLL_ARGS_FLAG_COUNT_64BIT | U.UCC_COLL_ARGS_FLAG_DISPLACEMENTS_64BIT)
            a._keep = a._keep + keep
    return a


# ------------------------------------------------------------------ one collective
class _Buf:
    """a Placed buffer, the image it must have afterwards and the labelled byte ranges of its data region"""

    def __init__(self, h, nbytes, mis, g, name):
        self.p = Placed(h.mem, nbytes, mis, g)
        self.name, self.regions = name, []
        self.exp = None

    def start(self, data=None, at=0):
        """initial content: random, with `data` at byte `at` of the data region"""
        if data is not None:
            b = self.p.init[self.p.off:self.p.off + self.p.nbytes].copy()
            b[at:at + len(data)] = data
            self.p.fill(b)
        else:
            self.p.fill()
        self.exp = self.p.init.copy()

    def expect(self, at, data, label):
        """bytes [at, at + len(data)) of the data region must come back as `data`"""
        self.exp[self.p.off + at:self.p.off + at + len(data)] = data
        if len(data):
            self.regions.append((at, at + len(data), label))

    def where(self, i):
        k = i - self.p.off
        if k < 0:
            return f"the leading guard band (byte {k})"
        if k >= self.p.nbytes:
            return f"past the end of the buffer (byte {k - self.p.nbytes} after it)"
        for lo, hi, label in self.regions:
            if lo <= k < hi:
                return f"{label} (bytes [{lo},{hi}))"
        return "bytes no block covers (a gap, or a region the caller must not have written)"

    def check(self, what):
        got, _ = self.p.read()
        bad = np.flatnonzero(got != self.exp)
        if bad.size:
            i = int(bad[0])
            j = i
            while j + 1 < got.size and got[j + 1] != self.exp[j + 1]:
                j += 1
            lo, hi = i - self.p.off, j + 1 - self.p.off
            raise Violation(f"{what}: {self.name}: {bad.size} bytes differ, first run [{lo},{hi}) of the data region in "
                            f"{self.where(i)}: got {got[i:min(j + 1, i + 8)].tolist()} expected {self.exp[i:min(j + 1, i + 8)].tolist()}")


def _rand(g, nbytes):
    return g.integers(0, 256, nbytes, dtype=np.uint8)


def build(h, n, coll, layout, dt, seed, mis=0, inplace=False, root=0, width=64, rep=0):
    """buffers, per-rank arguments and the reference image of every buffer of one collective"""
    sz = ELEM[dt]
    g = np.random.default_rng(seed)
    bufs = []

    def buf(nbytes, name):
        b = _Buf(h, nbytes, mis, g, name)
        bufs.append(b)
        return b
    args = [None] * n
    A = lambda *x, **kw: make_args(h, coll, *x, dt, width, n, **kw)  # noqa: E731
    if coll in ("allgather", "allgatherv"):
        if coll == "allgather":
            blk = fixed_count(layout, n, sz, g, rep)
            cnt, dsp, ext = np.full(n, blk), np.arange(n) * blk, n * blk
        else:
            cnt = block_counts(layout, n, sz, g, rep)
            dsp, ext = place(layout, cnt, g)
        data = [_rand(g, int(cnt[r]) * sz) for r in range(n)]
        for r in range(n):
            d = buf(ext * sz, f"rank {r} dst")
            if inplace:
                d.start(data[r], int(dsp[r]) * sz)
            else:
                d.start()
                s = buf(len(data[r]), f"rank {r} src")
                s.start(data[r])
            for p in range(n):
                d.expect(int(dsp[p]) * sz, data[p], f"the block of rank {p}")
            kw = dict(dst_counts=cnt, dst_displs=dsp) if coll == "allgatherv" else dict(count_dst=ext)
            args[r] = A(None if inplace else s.p.ptr, d.p.ptr, inplace=inplace, count_src=0 if inplace else int(cnt[r]), **kw)
    elif coll in ("alltoall", "alltoallv"):
        if coll == "alltoall":
            blk = fixed_count(layout, n, sz, g, rep)
            M = np.full((n, n), blk, np.int64)
            sd = rd = [np.arange(n) * blk] * n
            sext = rext = [n * blk] * n
        else:
            M = np.stack([block_counts(layout, n, sz, g, rep, own=s) for s in range(n)])
            if layout == "zeros" and rep == 1:            # all but one: every receiver gets a block from one sender only
                keep = int(g.integers(n))
                M = np.where(np.arange(n)[:, None] == keep, _small(16 // sz, g, (n, n)), 0)
            if inplace:                                   # the same split in both directions
                M = np.triu(M) + np.triu(M, 1).T
            sd, sext = zip(*[place(layout, M[s], g) for s in range(n)])
            rd, rext = zip(*[place(layout, M[:, r], g) for r in range(n)])
            if inplace:
                sd, sext = rd, rext
        payload = [[_rand(g, int(M[s, d]) * sz) for d in range(n)] for s in range(n)]
        for r in range(n):
            d = buf(int(rext[r]) * sz, f"rank {r} dst")
            if inplace:                                   # my regions hold what I send, and receive in their place
                img = _rand(g, int(rext[r]) * sz)
                for p in range(n):
                    img[int(rd[r][p]) * sz:][:len(payload[r][p])] = payload[r][p]
                d.start(img)
            else:
                d.start()
                img = _rand(g, int(sext[r]) * sz)
                for p in range(n):
                    img[int(sd[r][p]) * sz:][:len(payload[r][p])] = payload[r][p]
                s = buf(len(img), f"rank {r} src")
                s.start(img)
            for p in range(n):
                d.expect(int(rd[r][p]) * sz, payload[p][r], f"the block from rank {p}")
            if coll == "alltoall":
                args[r] = A(None if inplace else s.p.ptr, d.p.ptr, inplace=inplace, count_src=0 if inplace else n * blk, count_dst=n * blk)
            elif inplace:
                args[r] = A(None, d.p.ptr, inplace=True, dst_counts=M[:, r], dst_displs=rd[r])
            else:
                args[r] = A(s.p.ptr, d.p.ptr, src_counts=M[r], src_displs=sd[r], dst_counts=M[:, r], dst_displs=rd[r])
    elif coll == "bcast":
        cnt = fixed_count(layout, n, sz, g, rep)
        data = _rand(g, cnt * sz)
        for r in range(n):
            b = buf(cnt * sz, f"rank {r} buffer")
            b.start(data if r == root else None)
            b.expect(0, data, "the root's data")
            args[r] = A(b.p.ptr, None, root=root, count_src=cnt, count_dst=0)
    elif coll in ("gather", "gatherv"):
        if coll == "gather":
            blk = fixed_count(layout, n, sz, g, rep)
            cnt, dsp, ext = np.full(n, blk), np.arange(n) * blk, n * blk
        else:
            cnt = block_counts(layout, n, sz, g, rep)
            dsp, ext = place(layout, cnt, g)
        data = [_rand(g, int(cnt[r]) * sz) for r in range(n)]
        for r in range(n):
            ip = inplace and r == root
            if not ip:
                s = buf(len(data[r]), f"rank {r} src")
                s.start(data[r])
            if r == root:
                d = buf(ext * sz, f"root {r} dst")
                d.start(data[r] if ip else None, int(dsp[r]) * sz)
                for p in range(n):
                    d.expect(int(dsp[p]) * sz, data[p], f"the block of rank {p}")
                kw = dict(dst_counts=cnt, dst_displs=dsp) if coll == "gatherv" else dict(count_dst=ext)
                args[r] = A(None if ip else s.p.ptr, d.p.ptr, root=root, inplace=ip, count_src=0 if ip else int(cnt[r]), **kw)
            else:                                         # a destination the non-root passes, which the collective must not touch
                x = buf(ext * sz, f"rank {r} dst (non-root: unused)")
                x.start()
                args[r] = A(s.p.ptr, x.p.ptr, root=root, count_src=int(cnt[r]), count_dst=0)
    elif coll in ("scatter", "scatterv"):
        if coll == "scatter":
            blk = fixed_count(layout, n, sz, g, rep)
            cnt, dsp, ext = np.full(n, blk), np.arange(n) * blk, n * blk
        else:
            cnt = block_counts(layout, n, sz, g, rep)
            dsp, ext = place(layout, cnt, g)
        img = _rand(g, ext * sz)
        for r in range(n):
            ip = inplace and r == root
            blkb = img[int(dsp[r]) * sz:][:int(cnt[r]) * sz]
            if r == root:
                s = buf(len(img), f"root {r} src")
                s.start(img)
                kw = dict(src_counts=cnt, src_displs=dsp) if coll == "scatterv" else dict(count_src=ext)
            else:                                         # a source the non-root passes, which the collective must not touch
                s = buf(ext * sz, f"rank {r} src (non-root: unused)")
                s.start()
                kw = dict(count_src=0)
            if ip:
                args[r] = A(s.p.ptr, None, root=root, inplace=True, count_dst=0, **kw)
                continue
            d = buf(len(blkb), f"rank {r} dst")
            d.start()
            d.expect(0, blkb, f"block {r} of the root's source")
            args[r] = A(s.p.ptr, d.p.ptr, root=root, count_dst=int(cnt[r]), **kw)
    else:
        raise ValueError(coll)
    return bufs, args


def run_case(h, team, n, coll, path, layout, dt, seed, mis=0, inplace=False, root=0, width=64):
    """one case of the contract: the collective twice in a row on the same team, with fresh data and another layout of the same
    kind (a stale offset table, epoch or exchange-board entry of the first run shows up in the second)"""
    notes = []
    for rep in (0, 1):
        what = (f"{coll} path={path} n={n} layout={layout}{'#2' if rep else ''} {dt} mis={mis} counts={width}-bit"
                f"{' inplace' if inplace else ''}{f' root={root}' if coll in ROOTED else ''} seed={seed + rep}")
        bufs, args = build(h, n, coll, layout, dt, seed + rep * 7919, mis, inplace, root, width, rep)
        h.run(team, args)
        note = h.last_launch()
        want = want_note(path, coll, inplace)
        if note.split(" ")[0] != want:
            raise Violation(f"{what}: served by `{note}`, not by {want}")
        for b in bufs:
            b.check(what)
        notes.append(note)
    return notes


def cases_of(path, family, n, k=0):
    """the cases of one (path, family, team size): every layout of every collective of the family with a rotating datatype,
    misalignment and count width, in place where allowed, and both roots of rooted collectives.  `tail` cases keep the buffers
    16-byte aligned, so the TMA mover of push_bulk sees whole stages (it hands a misaligned block to the thread copy)"""
    out = []
    i = k
    for coll in FAMILIES[family]:
        layouts = LAYOUTS if coll in VCOLLS else FIXED_LAYOUTS
        roots = (0, n - 1) if coll in ROOTED else (0,)
        for layout in layouts:
            for root in roots:
                i += 1
                dt = DTYPES[i % len(DTYPES)]
                mis = 0 if layout == "tail" else MIS[(i // 2) % len(MIS)]
                width = 32 if (coll in VCOLLS and i % 2) else 64
                out.append(dict(coll=coll, layout=layout, dt=dt, mis=mis, root=root, width=width, inplace=False))
        if inplace_allowed(path, coll):
            for j, layout in enumerate(LAYOUTS[1:4] if coll in VCOLLS else layouts):
                i += 1
                out.append(dict(coll=coll, layout=layout, dt=DTYPES[(i + j) % len(DTYPES)], mis=MIS[i % len(MIS)],
                                root=(n - 1) if (coll in ROOTED and i % 2) else 0, width=32 if coll in VCOLLS and i % 2 else 64,
                                inplace=True))
    return out


def run_cases(h, team, n, path, family, seed, k=0):
    cases = cases_of(path, family, n, k)
    for c in cases:
        seed += 1
        run_case(h, team, n, path=path, seed=seed, **c)
    return len(cases)


# ------------------------------------------------------------------ the heap bound
def _init(team, args):
    """ucc_collective_init on every member: (status, request or None) per rank; nothing is posted"""
    from ucc_b200 import capi as U
    out = []
    for r, a in enumerate(args):
        q = C.POINTER(U.ucc_coll_req_t)()
        st = U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team)
        out.append((st, q if st == U.UCC_OK else None))
    return out


def expect_refused(h, team, n, what, args, refuse):
    """init must fail with UCC_ERR_NOT_SUPPORTED on the ranks in `refuse` (and succeed elsewhere); the requests that did initialise
    are finalized without being posted, so an init that wrongly accepted never runs past the heap"""
    from ucc_b200 import capi as U
    res = _init(team, args)
    for r, (st, q) in enumerate(res):
        if q is not None:
            U.ucc_collective_finalize(q)
    got = [st for st, _ in res]
    bad = [r for r in range(n) if (r in refuse) != (got[r] == U.UCC_ERR_NOT_SUPPORTED) or (r not in refuse and got[r] != U.UCC_OK)]
    if bad:
        raise Violation(f"{what}: init status per rank {[U.status_str(s) for s in got]}, expected UCC_ERR_NOT_SUPPORTED exactly on ranks "
                        f"{sorted(refuse)} and UCC_OK elsewhere")


def heap_cases(n, symm):
    """(coll, per-case parameters) at the heap bound of a team of n: cap = SYMMETRIC_SIZE - the offset table.  uint8, so every
    byte count is reachable.  `fits` says whether the staged payload fits; `refuse`: the ranks that must decline it"""
    cap = symm - TABLE_BYTES
    blk_a2a = cap // n
    out = [("allgather", dict(blk=cap), True, ()), ("allgather", dict(blk=cap + 1), False, tuple(range(n))),
           ("alltoall", dict(blk=blk_a2a), True, ()), ("alltoall", dict(blk=blk_a2a + 1), False, tuple(range(n))),
           ("scatterv", dict(ext=cap), True, ()), ("scatterv", dict(ext=cap + 1), False, (n - 1,))]
    return cap, out


def _heap_args(h, n, coll, p, g, width=64):
    """buffers and arguments of one heap-bound case (uint8; scatterv: root n-1 whose source ends exactly at `ext`)"""
    bufs, args = [], []
    if coll == "allgather":
        blk = p["blk"]
        data = [_rand(g, blk) for _ in range(n)]
        for r in range(n):
            s, d = _Buf(h, blk, 0, g, f"rank {r} src"), _Buf(h, n * blk, 0, g, f"rank {r} dst")
            s.start(data[r])
            d.start()
            for q in range(n):
                d.expect(q * blk, data[q], f"the block of rank {q}")
            bufs += [s, d]
            args.append(make_args(h, "allgather", s.p.ptr, d.p.ptr, "uint8", width, n, count_src=blk, count_dst=n * blk))
    elif coll == "alltoall":
        blk = p["blk"]
        srcs = [_rand(g, n * blk) for _ in range(n)]
        for r in range(n):
            s, d = _Buf(h, n * blk, 0, g, f"rank {r} src"), _Buf(h, n * blk, 0, g, f"rank {r} dst")
            s.start(srcs[r])
            d.start()
            for q in range(n):
                d.expect(q * blk, srcs[q][r * blk:(r + 1) * blk], f"the block from rank {q}")
            bufs += [s, d]
            args.append(make_args(h, "alltoall", s.p.ptr, d.p.ptr, "uint8", width, n, count_src=n * blk, count_dst=n * blk))
    else:   # scatterv from root n-1: blocks in reverse rank order, so the root's source ends exactly at ext
        ext = p["ext"]
        root = n - 1
        cnt = np.full(n, ext // n, np.int64)
        cnt[0] += ext - cnt.sum()
        order = list(range(n))[::-1]
        dsp = np.zeros(n, np.int64)
        off = 0
        for q in order:
            dsp[q] = off
            off += int(cnt[q])
        img = _rand(g, ext)
        for r in range(n):
            d = _Buf(h, int(cnt[r]), 0, g, f"rank {r} dst")
            d.start()
            d.expect(0, img[int(dsp[r]):int(dsp[r] + cnt[r])], f"block {r} of the root's source")
            bufs.append(d)
            if r == root:
                s = _Buf(h, ext, 0, g, f"root {r} src")
                s.start(img)
                bufs.append(s)
                args.append(make_args(h, "scatterv", s.p.ptr, d.p.ptr, "uint8", width, n, root=root, src_counts=cnt, src_displs=dsp,
                                      count_dst=int(cnt[r])))
            else:
                args.append(make_args(h, "scatterv", None, d.p.ptr, "uint8", width, n, root=root, count_src=0, count_dst=int(cnt[r])))
    return bufs, args


def ring_bound_counts(n, cap, g):
    """allgatherv block counts (uint8) whose 16-byte aligned sum is exactly cap, all but block j no multiples of 16 (so their plain
    sum stays below cap); block j is one: one byte more there adds 16 to the aligned sum"""
    units = cap // 16
    k = np.full(n, units // n, np.int64)
    k[0] += units - k.sum()
    cnt = 16 * k - g.integers(1, 16, n)
    j = int(g.integers(n))
    cnt[j] = 16 * k[j]
    return cnt, j


def run_heap_bound(h, team, n, path, symm, seed):
    """the staged payload at its bound: exactly cap runs and is byte-exact; one element more is refused at init on the ranks whose
    payload exceeds it.  The ring allgatherv is bounded by the sum of its 16-byte aligned blocks: at the bound the ring kernel
    serves it, one byte past it the staged pull."""
    g = np.random.default_rng(seed)
    cap, cases = heap_cases(n, symm)
    ran = 0
    if path == "ring":
        cnt, j = ring_bound_counts(n, cap, g)
        for extra, fits in ((0, True), (1, False)):
            c = cnt.copy()
            c[j] += extra
            dsp = np.concatenate([[0], np.cumsum(c)[:-1]])
            data = [_rand(g, int(c[r])) for r in range(n)]
            bufs, args = [], []
            for r in range(n):
                s, d = _Buf(h, int(c[r]), 0, g, f"rank {r} src"), _Buf(h, int(c.sum()), 0, g, f"rank {r} dst")
                s.start(data[r])
                d.start()
                for q in range(n):
                    d.expect(int(dsp[q]), data[q], f"the block of rank {q}")
                bufs += [s, d]
                args.append(make_args(h, "allgatherv", s.p.ptr, d.p.ptr, "uint8", 64, n, count_src=int(c[r]), dst_counts=c, dst_displs=dsp))
            what = (f"allgatherv path=ring n={n} heap bound: sum of 16-byte aligned blocks {int(sum((int(x) + 15) // 16 * 16 for x in c))}"
                    f" against cap {cap}")
            # past its bound the ring declines at init and the request goes down the score fallback to the staged pull
            h.run(team, args)
            note, want = h.last_launch(), "exchange_ring" if fits else "exchange_pull_staged"
            if note.split(" ")[0] != want:
                raise Violation(f"{what}: served by `{note}`, not by {want}")
            for b in bufs:
                b.check(what)
            ran += 1
        return ran
    for coll, p, fits, refuse in cases:
        if not any(coll in FAMILIES[f] for f in PATHS[path][1]):
            continue
        bufs, args = _heap_args(h, n, coll, p, g)
        what = f"{coll} path={path} n={n} heap bound: staged payload {p} against cap {cap}"
        if fits:
            h.run(team, args)
            note = h.last_launch()
            want = want_note(path, coll, False)
            if note.split(" ")[0] != want:
                raise Violation(f"{what}: served by `{note}`, not by {want}")
            for b in bufs:
                b.check(what)
            ran += 1
        else:
            expect_refused(h, team, n, what, args, set(refuse))
    return ran
