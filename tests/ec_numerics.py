"""The numerical contract of the execution components' reduce tasks (ec/cpu and ec/cuda), with a bitwise reference and seeded
inputs.  Shared by tests/test_ec_numerics.py (ec/cpu, no GPU) and tests/test_ec_numerics_gpu.py (ec/cuda); the contract is written
down in tests/README.md.

An executor reduces in a fixed order - source 0, then 1, ... n-1 - so the reference replays that order in the kernel's accumulator
type (float32 for float16 / bfloat16, T otherwise) with numpy's IEEE arithmetic and is bitwise for every real type.  Inputs are
those of tests/nvl_numerics.py (four lane classes in every 16-byte vector, edge values included) and tests/nvl_int128.py."""
import ctypes as C

import numpy as np

import nvl_int128 as Q
import nvl_numerics as V
from ucc_b200 import capi as U
from ucc_b200 import internal as I

GUARD = V.GUARD
INT128 = Q.DTYPES
DTYPES = V.ALL_DTYPES + INT128           # the 16 datatypes ec/cuda reduces
SIZE = dict(V.SIZE, int128=16, uint128=16)
ACC = {"float16": np.float32, "bfloat16": np.float32, "float32": np.float32, "float64": np.float64}
EC_MAX_SRCS = 16


def ops_of(dt):
    return Q.OPS if dt in INT128 else V.ops_of(dt)


def avg_divisor(alpha):
    """n when alpha == 1.0 / n exactly for an integer n >= 1 (every AVG the library posts), else 0"""
    if not 0.0 < alpha <= 1.0:
        return 0
    n = int(round(1.0 / alpha))
    return n if 1.0 / n == alpha else 0


# ------------------------------------------------------------------ inputs
class Case:
    """the values of n sources of one reduction: x ([n][count]; numpy rows, Python integers for 128-bit types), lane classes"""

    def __init__(self, dt, op, count, n, seed):
        self.dt, self.op, self.count, self.n = dt, op, count, n
        if dt in INT128:
            self.x, self.cls, self.pat = Q.make_inputs(dt, count, n, seed), None, None
        else:
            # (the edge lanes of floats need two sources: x with -x)
            cl = (V.EXACT_T, V.EXACT_ACC, V.RANDOM) if n == 1 and dt in V.FLOATS else (V.EXACT_T, V.EXACT_ACC, V.RANDOM, V.EDGE)
            self.x, self.cls, self.pat = V.make_inputs(dt, op, count, n, seed, cl)

    def src_bytes(self, k):
        return (Q.encode if self.dt in INT128 else V.encode)(self.dt, self.x[k])


# ------------------------------------------------------------------ reference
def _int_avg(dt, s, alpha):
    """AVG of the wrapped sums s: trunc(s / n) for alpha = 1/n; otherwise trunc(double(s) * alpha), None where |s| > 2^53"""
    n = avg_divisor(alpha)
    signed = V.INTS[dt][1]
    if n:
        if not signed:
            return s // np.uint64(n)
        q = s // n
        return np.where((s < 0) & (q * n != s), q + 1, q)
    return np.trunc(s.astype(np.float64) * alpha).astype(s.dtype)


def reference(case, alpha=None):
    """the exact result of the executor, lane by lane (values in the representation of nvl_numerics.decode / nvl_int128.decode);
    None for complex PROD, which has a bound instead"""
    dt, op, x = case.dt, case.op, case.x
    if case.n == 1 and op != "avg" and (dt in V.INTS or dt in INT128):
        return list(x[0]) if dt in INT128 else x[0].copy()      # one source is copied: no logical operator turns it into 0 / 1
    if dt in INT128:
        n = avg_divisor(alpha) if op == "avg" else 0
        out = []
        for i in range(case.count):
            col = [row[i] for row in x]
            if op != "avg":
                out.append(Q.reference(dt, op, col))
                continue
            s = Q.reference(dt, "sum", col)
            out.append((-(-s // n) if s < 0 else s // n) if n else Q.wrap(dt, int(float(s) * alpha)))
        return out
    if dt in V.INTS:
        if op == "avg":
            with np.errstate(over="ignore"):
                return _int_avg(dt, V.int_reference(dt, "sum", x), alpha)
        return V.int_reference(dt, op, x)
    with np.errstate(all="ignore"):
        if dt in V.COMPLEX:
            if op == "prod":
                return None
            R = np.float32 if dt == "float32_complex" else np.float64
            re, im = x[0].real.astype(R), x[0].imag.astype(R)
            for k in range(1, case.n):
                re, im = re + x[k].real.astype(R), im + x[k].imag.astype(R)
            if alpha is not None:
                re, im = re * R(alpha), im * R(alpha)
            return re.astype(np.float64) + 1j * im.astype(np.float64)
        A = ACC[dt]
        acc = x[0].astype(A)
        for k in range(1, case.n):
            v = x[k].astype(A)
            if op in ("sum", "avg"):
                acc = acc + v
            elif op == "prod":
                acc = acc * v
            elif op == "max":
                acc = np.where(acc > v, acc, v)
            else:
                acc = np.where(acc < v, acc, v)
        if alpha is not None:
            acc = acc * A(alpha)
        return V.decode(dt, V.encode(dt, acc.astype(np.float64)))      # RNE to T


def check(case, got_bytes, what, alpha=None):
    """got_bytes (the destination's data) must be the reference bit for bit: NaN lanes only have to be NaN, complex PROD gets the
    bound of nvl_numerics.check_complex"""
    dt, op = case.dt, case.op
    exp = reference(case, alpha)
    if dt in INT128:
        got = Q.decode(dt, got_bytes)
        bad = [i for i in range(case.count) if got[i] != exp[i]]
        if bad:
            i = bad[0]
            raise V.Violation(f"{what}: {len(bad)} lanes differ, e.g. lane {i} got {got[i]:#x} expected {exp[i]:#x}")
        return
    got = V.decode(dt, got_bytes)
    if exp is None:
        V.check_complex(dt, op, case.x, got, case.cls, 0, what)
        return
    if dt in V.INTS:
        bad = got != exp
        if op == "avg" and not avg_divisor(alpha):
            s = V.int_reference(dt, "sum", case.x)
            bad &= np.abs(s.astype(np.float64)) <= 2.0 ** 53
    else:
        sz = SIZE[dt]
        enc = V.encode(dt, exp) if dt not in V.COMPLEX else np.ascontiguousarray(
            exp.astype(np.complex64 if dt == "float32_complex" else np.complex128)).view(np.uint8)
        with np.errstate(invalid="ignore"):
            nan = np.isnan(exp) & np.isnan(got)
        bad = np.any(np.asarray(got_bytes).reshape(-1, sz) != enc.reshape(-1, sz), 1) & ~nan
    if np.any(bad):
        V._fail(f"{what}: not bitwise the in-order reference", bad, got, exp)


# ------------------------------------------------------------------ executor tasks
def _keep(args, *objs):
    args._keep = getattr(args, "_keep", []) + list(objs)
    return args


def reduce_args(dst, srcs, count, dt, op, alpha=None):
    """a REDUCE task; more than 9 sources go through srcs_ext"""
    a = I.eee_task_args()
    a.task_type = I.EE_TASK_REDUCE
    r = a.reduce
    r.dst, r.n_srcs, r.count, r.dt, r.op = dst, len(srcs), count, U.DT[dt], U.OP[op]
    if len(srcs) > I.NUM_BUFS:
        ext = (C.c_void_p * len(srcs))(*srcs)
        a.flags |= I.EEE_FLAG_SRCS_EXT
        r.srcs[0] = C.addressof(ext)          # srcs_ext shares its place with srcs[0]
        _keep(a, ext)
    else:
        for i, s in enumerate(srcs):
            r.srcs[i] = s
    if alpha is not None:
        a.flags |= I.EEE_FLAG_ALPHA
        r.alpha = alpha
    return a


def strided_args(dst, src1, src2, stride, n_src2, count, dt, op, alpha=None):
    a = I.eee_task_args()
    a.task_type = I.EE_TASK_REDUCE_STRIDED
    rs = a.reduce_strided
    rs.dst, rs.src1, rs.src2, rs.stride, rs.count, rs.dt, rs.op, rs.n_src2 = dst, src1, src2, stride, count, U.DT[dt], U.OP[op], n_src2
    if alpha is not None:
        a.flags |= I.EEE_FLAG_ALPHA
        rs.alpha = alpha
    return a


def multi_dst_args(dsts, src1, src2, counts, dt, op):
    a = I.eee_task_args()
    a.task_type = I.EE_TASK_REDUCE_MULTI_DST
    m = a.reduce_multi_dst
    for j in range(len(dsts)):
        m.dst[j], m.src1[j], m.src2[j], m.counts[j] = dsts[j], src1[j], src2[j], counts[j]
    m.dt, m.op, m.n_bufs = U.DT[dt], U.OP[op], len(dsts)
    return a


def post_status(ex, args):
    """task_post's status; an accepted task is run to completion first"""
    t = C.c_void_p()
    st = I.lib.ucc_ee_executor_task_post(ex.h, C.byref(args), C.byref(t))
    if st == U.UCC_OK:
        while I.lib.ucc_ee_executor_task_test(t) == U.UCC_INPROGRESS:
            pass
        I.lib.ucc_ee_executor_task_finalize(t)
    return st


# ------------------------------------------------------------------ one task, checked
class HostBuf:
    """host memory for nvl_numerics.Placed"""

    def __init__(self, nbytes):
        self.a = np.zeros(nbytes, np.uint8)
        self.ptr = self.a.ctypes.data

    def write(self, b):
        self.a[:] = b

    def read(self):
        return self.a.copy()


class HostMem:
    @staticmethod
    def alloc(nbytes):
        return HostBuf(nbytes)


class Env:
    """what a case needs from its surroundings: mem.alloc(nbytes) (see nvl_numerics.Placed), run(args) -> runs one task to
    completion with its results readable, and the element offsets a buffer may take from 16-byte alignment"""

    def __init__(self, mem, run):
        self.mem, self.run = mem, run


def mis_of(dt, k):
    """the k-th byte offset from 16-byte alignment in steps of the element size (8 for 128-bit integers): 0..15 bytes"""
    step = 8 if dt in INT128 else SIZE[dt]
    return (k * step) % 16


def run_reduce(env, dt, op, count, n, seed, mis=(), inplace=None, alpha=None, what=""):
    """REDUCE of n sources: mis = byte offsets of (dst, src 0, src 1, ...) (missing ones: 0); inplace = k: dst is source k"""
    case = Case(dt, op, count, n, seed)
    sz = SIZE[dt]
    g = np.random.default_rng(seed + 11)
    mis = list(mis) + [0] * (n + 1 - len(mis))
    srcs = [V.Placed(env.mem, count * sz, mis[k + 1], g) for k in range(n)]
    for k in range(n):
        srcs[k].fill(case.src_bytes(k))
    dst = srcs[inplace] if inplace is not None else V.Placed(env.mem, count * sz, mis[0], g)
    if inplace is None:
        dst.fill()
    what = f"{what} reduce {dt} {op} count={count} n_srcs={n} mis={mis}{f' inplace={inplace}' if inplace is not None else ''} " \
           f"alpha={alpha} seed={seed}"
    env.run(reduce_args(dst.ptr, [s.ptr for s in srcs], count, dt, op, alpha))
    _check_dst(case, dst, what, alpha)
    _check_srcs([s for s in srcs if s is not dst], what)
    return case


def run_strided(env, dt, op, count, n_src2, pad, seed, mis=(0, 0, 0), alpha=None, what=""):
    """REDUCE_STRIDED: src1 and n_src2 vectors in one buffer, `pad` elements apart (an odd pad moves later vectors off alignment)"""
    case = Case(dt, op, count, n_src2 + 1, seed)
    sz = SIZE[dt]
    stride = (count + pad) * sz
    g = np.random.default_rng(seed + 13)
    s1 = V.Placed(env.mem, count * sz, mis[1], g)
    s1.fill(case.src_bytes(0))
    s2 = V.Placed(env.mem, max(stride * n_src2, 1), mis[2], g)
    b = s2.init[s2.off:s2.off + s2.nbytes].copy()
    for k in range(n_src2):
        b[k * stride:k * stride + count * sz] = case.src_bytes(k + 1)
    s2.fill(b)
    dst = V.Placed(env.mem, count * sz, mis[0], g)
    dst.fill()
    what = f"{what} reduce_strided {dt} {op} count={count} n_src2={n_src2} pad={pad} mis={list(mis)} alpha={alpha} seed={seed}"
    env.run(strided_args(dst.ptr, s1.ptr, s2.ptr, stride, n_src2, count, dt, op, alpha))
    _check_dst(case, dst, what, alpha)
    _check_srcs([s1, s2], what)
    return case


def run_multi_dst(env, dt, op, counts, seed, mis=mis_of, what=""):
    """REDUCE_MULTI_DST: len(counts) independent dst[j] = src1[j] op src2[j]; mis(dt, k): byte offsets of the buffers"""
    sz = SIZE[dt]
    g = np.random.default_rng(seed + 17)
    cases = [Case(dt, op, c, 2, seed + 100 * j) for j, c in enumerate(counts)]
    bufs = []
    for j, c in enumerate(counts):
        a, b, d = (V.Placed(env.mem, c * sz, mis(dt, j + i), g) for i in range(3))
        a.fill(cases[j].src_bytes(0))
        b.fill(cases[j].src_bytes(1))
        d.fill()
        bufs.append((a, b, d))
    what = f"{what} reduce_multi_dst {dt} {op} counts={list(counts)} seed={seed}"
    env.run(multi_dst_args([d.ptr for _, _, d in bufs], [a.ptr for a, _, _ in bufs], [b.ptr for _, b, _ in bufs], counts, dt, op))
    for j, (a, b, d) in enumerate(bufs):
        _check_dst(cases[j], d, f"{what} buffer {j}", None)
        _check_srcs([a, b], f"{what} buffer {j}")


def run_copy(env, sizes, seed, mis=None, multi=True, what=""):
    """COPY (one size) or COPY_MULTI: byte-exact, guards and sources unchanged"""
    g = np.random.default_rng(seed)
    pairs = []
    for j, n in enumerate(sizes):
        m = mis[j] if mis else (3 * j) % 16
        s, d = V.Placed(env.mem, n, m, g), V.Placed(env.mem, n, (m + 5 * j) % 16, g)
        s.fill(g.integers(0, 256, n, dtype=np.uint8))
        d.fill()
        pairs.append((s, d))
    a = I.eee_task_args()
    if multi:
        a.task_type = I.EE_TASK_COPY_MULTI
        for j, (s, d) in enumerate(pairs):
            a.copy_multi.src[j], a.copy_multi.dst[j], a.copy_multi.counts[j] = s.ptr, d.ptr, s.nbytes
        a.copy_multi.num_vectors = len(pairs)
    else:
        (s, d), = pairs
        a.task_type = I.EE_TASK_COPY
        a.copy.dst, a.copy.src, a.copy.len = d.ptr, s.ptr, s.nbytes
    env.run(a)
    what = f"{what} {'copy_multi' if multi else 'copy'} sizes={list(sizes)} seed={seed}"
    for j, (s, d) in enumerate(pairs):
        b, data = d.read()
        d.check_outside(b, f"{what} buffer {j}")
        if not np.array_equal(data, s.init[s.off:s.off + s.nbytes]):
            raise V.Violation(f"{what} buffer {j}: {int(np.count_nonzero(data != s.init[s.off:s.off + s.nbytes]))} bytes differ")
        _check_srcs([s], what)


def _check_dst(case, dst, what, alpha):
    b, data = dst.read()
    dst.check_outside(b, what)
    check(case, data, what, alpha)


def _check_srcs(srcs, what):
    for k, s in enumerate(srcs):
        b = s.buf.read()
        if not np.array_equal(b, s.init):
            raise V.Violation(f"{what}: source buffer {k} changed")
