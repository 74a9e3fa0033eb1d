"""The numerical contract of the 128-bit integer reductions (UCC_DT_INT128 / UINT128, tests/README.md), shared by the GPU test
(tests/test_nvl_int128_gpu.py) and the host-emulation worker (tests/hostemu_int128_worker.py).

numpy has no 128-bit integer, so values are Python integers: a case builds each rank's values, encodes them as little-endian pairs
of 64-bit words between the guard bands of tests/nvl_numerics.py, runs the collective and decodes what came back.  The reference is
exact: every operator is evaluated on Python integers and wrapped mod 2^128; for int128 the wrapped value is read back as two's
complement.  AVG is trunc(wrapped sum / N), the rule of the other tl/nvl integer types."""
import numpy as np

import nvl_numerics as V

DTYPES = ["int128", "uint128"]
OPS = V.INT_OPS
SIZE = 16
M = 1 << 128
M64 = (1 << 64) - 1
IMIN, IMAX = -(1 << 127), (1 << 127) - 1


def wrap(dt, v):
    """any integer -> the dt value its low 128 bits encode"""
    u = v % M
    return u - M if dt == "int128" and u >> 127 else u


def encode(dt, vals):
    """dt values -> raw bytes (16 per value, low word first)"""
    w = np.array([(u & M64, u >> 64) for u in (v % M for v in vals)], np.uint64).reshape(-1)
    return w.astype("<u8").view(np.uint8)


def decode(dt, b):
    w = np.ascontiguousarray(b).view("<u8").reshape(-1, 2)
    return [wrap(dt, int(lo) | int(hi) << 64) for lo, hi in w]


# ------------------------------------------------------------------ inputs
# lane classes: small integers; the limits; a low word of all ones or zero under a non-zero high word (carries and borrows between
# the halves); values that differ only in the high word (MAX / MIN); random 128-bit values
SMALL, LIMIT, CARRY, HIGH, RANDOM = range(5)
CLASSES = (SMALL, LIMIT, CARRY, HIGH, RANDOM)


LIMITS = [IMIN, IMAX, 0, -1, 1 << 127, M - 1, 1, IMIN + 1, IMAX - 1]


def make_inputs(dt, count, n_ranks, seed):
    """per-rank inputs of one case: list [n_ranks][count] of dt values, the classes interleaved lane by lane"""
    g = np.random.default_rng(seed)
    shape = (n_ranks, count)

    def words():
        return g.integers(0, 1 << 64, shape, dtype=np.uint64).tolist()

    small = (g.integers(-4, 5, shape) if dt == "int128" else g.integers(0, 9, shape)).tolist()
    lim = g.integers(0, len(LIMITS), shape).tolist()
    chi, clo, cneg = words(), g.integers(0, 2, shape).tolist(), g.integers(0, 2, shape).tolist()
    hlow, hhi = words()[0], g.integers(-3, 4, shape).tolist()      # HIGH: one low word per lane, shared by every rank
    rhi, rlo = words(), words()
    x = []
    for r in range(n_ranks):
        row = []
        for i in range(count):
            c = i % len(CLASSES)
            if c == SMALL:
                v = small[r][i]
            elif c == LIMIT:
                v = LIMITS[lim[r][i]]
            elif c == CARRY:
                v = (chi[r][i] | 1) << 64 | (M64 if clo[r][i] else 0)
                v = -v if cneg[r][i] else v
            elif c == HIGH:
                v = hhi[r][i] << 64 | hlow[i]
            else:
                v = rhi[r][i] << 64 | rlo[r][i]
            row.append(wrap(dt, v))
        x.append(row)
    return x


# ------------------------------------------------------------------ reference
def reference(dt, op, col):
    """exact result of reducing the values `col` (one per rank) with op, wrapped to dt"""
    n = len(col)
    if op == "max":
        return max(col)
    if op == "min":
        return min(col)
    if op == "land":
        return int(all(v != 0 for v in col))
    if op == "lor":
        return int(any(v != 0 for v in col))
    if op == "lxor":
        return sum(v != 0 for v in col) % 2
    r = col[0]
    for v in col[1:]:
        if op in ("sum", "avg"):
            r += v
        elif op == "prod":
            r *= v
        elif op == "band":
            r &= v
        elif op == "bor":
            r |= v
        elif op == "bxor":
            r ^= v
    r = wrap(dt, r)
    if op == "avg":
        q = abs(r) // n
        return -q if r < 0 else q
    return r


def check_values(dt, op, x, got, what):
    """got[i] must be bitwise the reference of lane i of x ([n_ranks][count])"""
    bad = [i for i in range(len(got)) if got[i] != reference(dt, op, [row[i] for row in x])]
    if bad:
        i = bad[0]
        raise V.Violation(f"{what}: not bitwise the wrapped 128-bit reference in {len(bad)} lanes, e.g. lane {i} got {got[i]:#x} "
                          f"expected {reference(dt, op, [row[i] for row in x]):#x} (inputs {[hex(row[i]) for row in x]})")


# ------------------------------------------------------------------ one collective
def run_case(h, team, n, coll, path, dt, op, count, seed, mis=0, inplace=False, root=0, rs_counts=None):
    """one collective on team (n members), checked as tests/nvl_numerics.run_case checks the other types: results, cross-rank
    identity, guard bands, sources, the rest of an in-place reduce_scatter buffer, and the kernel that ran (V.PATHS).  count:
    elements of the vector (allreduce / reduce), of every block (reduce_scatter) or None (reduce_scatterv with rs_counts)."""
    counts = list(rs_counts) if coll == "reduce_scatterv" else ([count] * n if coll == "reduce_scatter" else None)
    total = sum(counts) if counts else count
    offs = [sum(counts[:r]) for r in range(n)] if counts else None
    what = f"{coll} path={path} n={n} {dt} {op} count={counts if coll == 'reduce_scatterv' else count} mis={mis} " \
           f"{'inplace ' if inplace else ''}{f'root={root} ' if coll == 'reduce' else ''}seed={seed}"
    x = make_inputs(dt, total, n, seed)
    g = np.random.default_rng(seed + 7)
    srcs = [V.Placed(h.mem, total * SIZE, mis, g) for _ in range(n)]
    for r in range(n):
        srcs[r].fill(encode(dt, x[r]))
    dsts = [None] * n
    args = []
    for r in range(n):
        if inplace:
            dsts[r] = srcs[r]
            kw = dict(dst_counts=counts, dst_displs=offs) if coll == "reduce_scatterv" else dict(count_dst=total)
            args.append(h.args(coll, None, srcs[r].ptr, dt, op=op, inplace=True, count_src=0, **kw))
            continue
        if coll == "allreduce":
            dsts[r] = V.Placed(h.mem, total * SIZE, mis, g)
            kw = dict(count_src=total, count_dst=total)
        elif coll == "reduce":
            if r == root:
                dsts[r] = V.Placed(h.mem, total * SIZE, mis, g)
            kw = dict(count_src=total, count_dst=total if r == root else 0, root=root)
        elif coll == "reduce_scatter":
            dsts[r] = V.Placed(h.mem, count * SIZE, mis, g)
            kw = dict(count_src=total, count_dst=count)
        else:
            dsts[r] = V.Placed(h.mem, counts[r] * SIZE, mis, g)
            kw = dict(count_src=total, dst_counts=counts, dst_displs=offs)
        if dsts[r] is not None:
            dsts[r].fill()
        args.append(h.args(coll, srcs[r].ptr, dsts[r].ptr if dsts[r] is not None else None, dt, op=op, **kw))
    h.run(team, args)
    note = h.last_launch()
    want = V.PATHS[path][3 if coll.startswith("reduce_scatter") else 2]
    if path == "zcopy" and mis % 16:
        want = "twoshot_staged"      # zero-copy needs 16-byte aligned buffers
    if not note.startswith(want):
        raise V.Violation(f"{what}: served by `{note}`, not by the {want.strip()} kernel")
    outs = {}
    for r in range(n):
        if dsts[r] is None:
            continue
        b, data = dsts[r].read()
        lo, hi, keep = 0, total, None
        if coll.startswith("reduce_scatter"):
            lo, hi = offs[r], offs[r] + counts[r]
            if inplace:
                keep = [(0, lo * SIZE), (hi * SIZE, total * SIZE)]
                data = data[lo * SIZE:hi * SIZE]
        dsts[r].check_outside(b, f"{what} rank {r}", keep)
        check_values(dt, op, [row[lo:hi] for row in x], decode(dt, data), f"{what} rank {r}")
        outs[r] = data
    if coll == "allreduce":
        for r in range(1, n):
            if not np.array_equal(outs[r], outs[0]):
                raise V.Violation(f"{what}: rank {r} differs bitwise from rank 0")
    if not inplace:
        for r in range(n):
            if not np.array_equal(srcs[r].read()[0], srcs[r].init):
                raise V.Violation(f"{what}: source of rank {r} changed")
    return note
