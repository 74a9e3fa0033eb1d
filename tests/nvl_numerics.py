"""The numerical contract of the tl/nvl reduction kernels, with exact CPU references and seeded inputs.  Shared by the GPU test
(tests/test_nvl_numerics_gpu.py) and the host-emulation worker (tests/hostemu_numerics_worker.py); the contract is written down in
tests/README.md.

Buffers travel as raw bytes, so every datatype - bfloat16 and the unsigned ones included - goes the same way: a case encodes each
rank's values into bytes, places them between two 64-byte guard bands, runs the collective and decodes what came back.  References
are exact: integers wrap in uint64 and are masked to the type's width, floating-point sums are taken in float64 (exact for the
inputs of the `exact` classes; compensated for float64 itself), and rounding to float16 / bfloat16 / float32 goes through torch's
round-to-nearest-even casts."""
import math

import numpy as np
import torch

GUARD = 64
INTS = {"int8": (8, True), "int16": (16, True), "int32": (32, True), "int64": (64, True),
        "uint8": (8, False), "uint16": (16, False), "uint32": (32, False), "uint64": (64, False)}
# floating point: (mantissa bits p incl. the hidden one, minimum normal exponent, accumulator precision p_acc)
FLOATS = {"float16": (11, -14, 24), "bfloat16": (8, -126, 24), "float32": (24, -126, 24), "float64": (53, -1022, 53)}
COMPLEX = {"float32_complex": "float32", "float64_complex": "float64"}
SIZE = {"int8": 1, "int16": 2, "int32": 4, "int64": 8, "uint8": 1, "uint16": 2, "uint32": 4, "uint64": 8, "float16": 2,
        "bfloat16": 2, "float32": 4, "float64": 8, "float32_complex": 8, "float64_complex": 16}
ALL_DTYPES = list(SIZE)
INT_OPS = ["sum", "prod", "max", "min", "land", "lor", "lxor", "band", "bor", "bxor", "avg"]
FLOAT_OPS = ["sum", "prod", "max", "min", "avg"]
COMPLEX_OPS = ["sum", "prod", "avg"]
NP_FLOAT = {"float16": np.float16, "float32": np.float32, "float64": np.float64}
TORCH_FLOAT = {"float16": torch.float16, "bfloat16": torch.bfloat16, "float32": torch.float32}


def ops_of(dt):
    return INT_OPS if dt in INTS else (FLOAT_OPS if dt in FLOATS else COMPLEX_OPS)


# ------------------------------------------------------------------ values <-> bytes
def round_to(dt, x):
    """float64 values -> the nearest dt values (round to nearest even), returned as float64"""
    x = np.asarray(x, np.float64)
    if dt == "float64":
        return x.copy()
    t = torch.from_numpy(x).to(torch.float32)       # exact for every value that fits float32 (the exact class)
    if dt != "float32":
        t = t.to(TORCH_FLOAT[dt]).to(torch.float32)
    return t.numpy().astype(np.float64)


def encode(dt, v):
    """values (int64 / uint64, float64 or complex128 holding dt values) -> raw bytes"""
    if dt in INTS:
        bits, signed = INTS[dt]
        return (np.asarray(v).astype(np.uint64) & np.uint64((1 << bits) - 1) if bits < 64 else np.asarray(v).astype(np.uint64)) \
            .astype(f"<u{bits // 8}").view(np.uint8)
    if dt in COMPLEX:
        return np.ascontiguousarray(np.asarray(v).astype(np.complex64 if dt == "float32_complex" else np.complex128)).view(np.uint8)
    if dt == "bfloat16":
        t = torch.from_numpy(np.asarray(v, np.float64)).to(torch.float32).to(torch.bfloat16)
        return t.view(torch.int16).numpy().view(np.uint8).copy()
    return np.ascontiguousarray(np.asarray(v).astype(NP_FLOAT[dt])).view(np.uint8)


def decode(dt, b):
    b = np.ascontiguousarray(b)
    if dt in INTS:
        bits, signed = INTS[dt]
        return b.view(f"<{'i' if signed else 'u'}{bits // 8}").astype(np.int64 if signed else np.uint64)
    if dt in COMPLEX:
        return b.view(np.complex64 if dt == "float32_complex" else np.complex128).astype(np.complex128)
    if dt == "bfloat16":
        return (b.view(np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    return b.view(NP_FLOAT[dt]).astype(np.float64)


def wrap(dt, u):
    """uint64 (mod 2^64) -> the dt value those low bits encode (int64 for signed types, uint64 for unsigned)"""
    bits, signed = INTS[dt]
    u = np.asarray(u, np.uint64) & np.uint64((1 << bits) - 1 if bits < 64 else (1 << 64) - 1)
    if not signed:
        return u
    s = u.astype(np.int64)
    if bits < 64:
        s = np.where(s >= (1 << (bits - 1)), s - (1 << bits), s)
    return s


# ------------------------------------------------------------------ inputs
# lane classes: EXACT_T (every partial sum representable in T), EXACT_ACC (in the fp32 accumulator but not in T), RANDOM, EDGE
EXACT_T, EXACT_ACC, RANDOM, EDGE = 0, 1, 2, 3
CLASS_NAME = {EXACT_T: "exact(T)", EXACT_ACC: "exact(acc)", RANDOM: "random", EDGE: "edge"}
# edge patterns of floating-point lanes
Z_SIGNED_ZEROS, Z_INF, Z_NAN, Z_MAX, Z_SUBNORMAL, Z_CANCEL = range(6)


def lane_classes(dt, count, classes):
    """class of every lane: the requested classes interleaved, so every 16-byte vector holds several"""
    cl = np.array([c for c in classes if not (c == EXACT_ACC and (dt in INTS or dt in COMPLEX))], np.int64)
    return cl[np.arange(count) % len(cl)]


def _float_values(dt, op, kind, shape, g):
    """float64 values of float type dt (or of the components of complex dt) for lanes of one class"""
    r = _real(dt)
    p = FLOATS[r][0]
    sign = np.where(g.random(shape) < 0.5, -1.0, 1.0)
    if op == "prod":
        # exact classes: powers of two, exact in any order, in T and in every hop; random: magnitudes in [0.5, 2), far from overflow
        mag = g.uniform(0.5, 2.0, shape) if kind == "random" else 2.0 ** g.integers(-1, 2, shape)
        return round_to(r, sign * mag)
    if kind == "exact_t":
        return g.integers(-8, 9, shape).astype(np.float64)
    if kind == "exact_acc":
        # T-representable k * 2^e (k as wide as the significand of T, at most 11 bits; e in 0..8): the sums need up to 22 bits -
        # exact in fp32, mostly not representable in bf16 / f16.  float16 (largest value 65504): 8-bit k, e in 0..5
        kb, eb = (8, 5) if r == "float16" else (min(p, 11), 8)
        return sign * g.integers(1, 1 << kb, shape) * 2.0 ** g.integers(0, eb + 1, shape)
    return round_to(r, g.standard_normal(shape) * 2.0 ** g.uniform(-4, 4, shape))


def _real(dt):
    return COMPLEX.get(dt, dt)


def float_max(dt):
    p, emin, _ = FLOATS[dt]
    return (2.0 - 2.0 ** (1 - p)) * 2.0 ** (-emin + 1) if dt != "float16" else 65504.0


def _float_edge(dt, op, n_ranks, L, g):
    """edge lanes whose exact result does not depend on the order of the reduction; returns (values, pattern per lane)"""
    p, emin, _ = FLOATS[dt]
    pats = np.array([Z_SIGNED_ZEROS, Z_INF, Z_NAN, Z_MAX, Z_SUBNORMAL, Z_CANCEL])
    pat = pats[np.arange(L) % len(pats)]
    if op == "avg":       # the average of values at the top of the range overflows the sum; the contract leaves it out
        pat = np.where(pat == Z_MAX, Z_SUBNORMAL, pat)
    fin = round_to(dt, g.uniform(0.5, 4.0, (n_ranks, L)) * np.where(g.random((n_ranks, L)) < 0.5, -1, 1))
    zeros = np.where(g.random((n_ranks, L)) < 0.5, -0.0, 0.0)
    one = (g.integers(0, n_ranks, L), np.arange(L))          # one rank per lane
    v = zeros.copy()                                          # Z_SIGNED_ZEROS: +-0 everywhere
    inf = g.random((n_ranks, L)) < 0.5                        # Z_INF: finite non-zero values, +inf / -inf on some ranks (one at least)
    inf[one] = True
    m = pat == Z_INF
    v[:, m] = np.where(inf, np.where(g.random((n_ranks, L)) < 0.7, np.inf, -np.inf), fin)[:, m]
    nan = fin.copy()                                          # Z_NAN: finite values, NaN on one rank
    nan[one] = np.nan
    m = pat == Z_NAN
    v[:, m] = nan[:, m]
    v[:, pat == Z_MAX] = float_max(dt)                       # the sum / product overflows in any order
    m = pat == Z_SUBNORMAL                                    # small multiples of the smallest subnormal: exact sums
    v[:, m] = (g.integers(-16, 17, (n_ranks, L)) * 2.0 ** (emin - p + 1))[:, m]
    m = pat == Z_CANCEL                                       # x and -x, the others +-0: the sum is +0 whatever the order
    v[0, m], v[1, m] = fin[0, m], -fin[0, m]
    return v, pat


def _int_values(dt, op, kind, n_ranks, L, g):
    bits, signed = INTS[dt]
    lo, hi = (-(1 << (bits - 1)), (1 << (bits - 1)) - 1) if signed else (0, (1 << bits) - 1)
    if kind == "exact_t":
        return g.integers(-4, 5, (n_ranks, L)) if signed else g.integers(0, 9, (n_ranks, L)).astype(np.uint64)
    if kind == "random":    # full-width random bits
        r = g.integers(0, 1 << 32, (n_ranks, L), dtype=np.uint64) << np.uint64(32) | g.integers(0, 1 << 32, (n_ranks, L), dtype=np.uint64)
        return wrap(dt, r)
    # edge: the limits, 0 and -1 (all ones), the top half of the unsigned range, non-zero values with a zero low byte
    pool = [lo, hi, 0, -1 if signed else hi, 1, (1 << (bits - 1)) if not signed else lo + 1, (1 << (bits - 1)) + 5 if not signed else hi - 1]
    if bits > 8:
        pool += [256, 256 << (bits - 16)]
    pool = np.array([wrap(dt, np.uint64(x & ((1 << 64) - 1))) for x in pool])
    return pool[g.integers(0, len(pool), (n_ranks, L))]


def make_inputs(dt, op, count, n_ranks, seed, classes=(EXACT_T, EXACT_ACC, RANDOM, EDGE)):
    """per-rank inputs of one case: (values [n_ranks, count], lane class [count], edge pattern [count] or -1)"""
    g = np.random.default_rng(seed)
    cls = lane_classes(dt, count, classes)
    pat = np.full(count, -1)
    kinds = {EXACT_T: "exact_t", EXACT_ACC: "exact_acc", RANDOM: "random", EDGE: "edge"}
    if dt in INTS:
        v = np.zeros((n_ranks, count), np.int64 if INTS[dt][1] else np.uint64)
    else:
        v = np.zeros((n_ranks, count), np.complex128 if dt in COMPLEX else np.float64)
    for c in np.unique(cls):
        m = cls == c
        L = int(m.sum())
        if dt in INTS:
            v[:, m] = _int_values(dt, op, kinds[c], n_ranks, L, g)
        elif dt in COMPLEX:
            kind = "exact_t" if c == EDGE else kinds[c]    # complex lanes: Gaussian integers and random values
            re = _float_values(dt, op, kind, (n_ranks, L), g)
            im = _float_values(dt, op, kind, (n_ranks, L), g)
            if op == "prod" and kind == "exact_t":          # one component zero: |z| a power of two, the product exact
                im = np.where(g.random(im.shape) < 0.5, im, 0.0)
                re = np.where(im != 0, 0.0, re)
            v[:, m] = re + 1j * im
        elif c == EDGE:
            v[:, m], pat[m] = _float_edge(dt, op, n_ranks, L, g)
        else:
            v[:, m] = _float_values(dt, op, kinds[c], (n_ranks, L), g)
    return v, cls, pat


# ------------------------------------------------------------------ references
def int_reference(dt, op, x):
    """exact result of reducing the rows of x (int64 / uint64 dt values) with op, wrapped to dt"""
    bits, signed = INTS[dt]
    u = x.astype(np.uint64)
    n = x.shape[0]
    with np.errstate(over="ignore"):
        if op in ("sum", "avg"):
            r = u.sum(0, dtype=np.uint64)
        elif op == "prod":
            r = u[0].copy()
            for i in range(1, n):
                r = r * u[i]
        elif op == "max":
            return x.max(0)
        elif op == "min":
            return x.min(0)
        elif op == "land":
            return np.all(x != 0, 0).astype(x.dtype)
        elif op == "lor":
            return np.any(x != 0, 0).astype(x.dtype)
        elif op == "lxor":
            return ((x != 0).sum(0) % 2).astype(x.dtype)
        elif op == "band":
            r = np.bitwise_and.reduce(u, 0)
        elif op == "bor":
            r = np.bitwise_or.reduce(u, 0)
        elif op == "bxor":
            r = np.bitwise_xor.reduce(u, 0)
    s = wrap(dt, r)
    if op == "avg":    # truncating division of the wrapped sum, as tl/shm and ec/cuda
        if signed:
            q = s // n
            return np.where((s < 0) & (q * n != s), q + 1, q)
        return s // np.uint64(n)
    return s


def sum_rows(x):
    """column sums of float64 x, compensated (TwoSum at every step): within an ulp of the exact sum, far inside every bound below"""
    s, c = x[0].copy(), np.zeros(x.shape[1])
    for i in range(1, x.shape[0]):
        t = s + x[i]
        bp = t - s
        c += (s - (t - bp)) + (x[i] - bp)
        s = t
    return s + c


def ulp(dt, x):
    p, emin, _ = FLOATS[dt]
    ax = np.abs(np.asarray(x, np.float64))
    e = np.where(ax > 0, np.frexp(np.where(ax > 0, ax, 1.0))[1] - 1, emin)
    return np.ldexp(1.0, np.maximum(e, emin) - p + 1)


class Violation(AssertionError):
    pass


def _fail(what, lanes, got, exp, extra=""):
    idx = np.flatnonzero(lanes)[:4]
    raise Violation(f"{what}: {int(np.count_nonzero(lanes))} lanes, e.g. lane {idx.tolist()} got {np.asarray(got)[idx].tolist()} "
                    f"expected {np.asarray(exp)[idx].tolist()} {extra}")


def _bits_differ(dt, a, b):
    """per lane: dt values a and b (held as float64) differ bitwise"""
    sz = SIZE[dt]
    return np.any(encode(dt, a).reshape(-1, sz) != encode(dt, b).reshape(-1, sz), 1)


def check_real(dt, op, x, got, cls, pat, hops, what):
    """floating-point result `got` (float64 holding dt values) of reducing the rows of x, against the contract of tests/README.md.
    hops: roundings to T along the way (ring / rhd round every partial result to T), 0 for the paths that accumulate in fp32"""
    n = x.shape[0]
    p, emin, p_acc = FLOATS[dt]
    u_acc, u_t = 2.0 ** -p_acc, 2.0 ** -p
    if op == "prod" and hops:   # every product of the tree is rounded to T, not only one per level
        hops = n - 1
    exact_lanes = (cls == EXACT_T) | ((cls == EXACT_ACC) & (hops == 0))
    bound_lanes = ((cls == EXACT_ACC) & (hops > 0)) | (cls == RANDOM)
    edge = cls == EDGE
    fin = ~edge
    if op in ("max", "min"):
        exp = x.max(0) if op == "max" else x.min(0)
        diff = _bits_differ(dt, got, exp)
        bad = fin & diff
        if bad.any():
            _fail(f"{what}: {op} not bitwise the {op} of the inputs", bad, got, exp)
        nan_in = np.isnan(x).any(0)
        bad = edge & ~nan_in & ~(got == exp)           # +-0 compare equal; NaN inputs: identical across ranks only
        if bad.any():
            _fail(f"{what}: {op} of edge values", bad, got, exp)
        return
    with np.errstate(invalid="ignore", over="ignore", under="ignore"):
        s = x[0].copy()       # a fold in rank order (numpy's reductions start from +0 and lose the sign of a sum of -0s)
        for i in range(1, n):
            s = s * x[i] if op == "prod" else s + x[i]
    if op != "prod" and fin.any():
        s[fin] = sum_rows(x[:, fin]) if dt == "float64" else x[:, fin].sum(0)
    sabs = np.abs(x).sum(0) if op != "prod" else np.abs(s)
    if op == "avg":
        with np.errstate(invalid="ignore", over="ignore"):
            exp = round_to(dt, s / n)
        ok_exact = np.abs(got - exp) <= ulp(dt, np.minimum(np.abs(got), np.abs(exp)))
        ok_exact |= (got == exp) | (np.isnan(got) & np.isnan(exp))
        bad = (exact_lanes | edge) & ~ok_exact
        if bad.any():
            _fail(f"{what}: avg more than 1 ulp from the correctly rounded S/N", bad, got, exp)
        tol = ((n + 1) * u_acc + hops * u_t) * sabs / n + 0.5 * ulp(dt, np.maximum(np.abs(got), np.abs(s / n)))
        err = np.abs(got - s / n)
        bad = bound_lanes & ~(err <= tol * (1 + 2.0 ** -20))
        if bad.any():
            _fail(f"{what}: avg error above the bound", bad, got, s / n, f"err {err[bad][:4].tolist()} bound {tol[bad][:4].tolist()}")
        return
    with np.errstate(invalid="ignore", over="ignore"):
        exp = round_to(dt, s)
    diff = _bits_differ(dt, got, exp)
    both_nan = np.isnan(got) & np.isnan(exp)
    bad = (exact_lanes | edge) & diff & ~both_nan
    if bad.any():
        _fail(f"{what}: {op} not bitwise RNE_T of the exact result ({CLASS_NAME[int(cls[np.flatnonzero(bad)[0]])]} lanes)", bad, got, exp)
    # (+ (N-1) 2^-53 |s|: the float64 fold of a product is not exact itself)
    tol = ((n - 1) * (u_acc + 2.0 ** -53 * (op == "prod")) + hops * u_t) * sabs + 0.5 * ulp(dt, np.maximum(np.abs(got), np.abs(s)))
    err = np.abs(got - s)
    bad = bound_lanes & ~(err <= tol * (1 + 2.0 ** -20))
    if bad.any():
        _fail(f"{what}: {op} error above (N-1) u_acc sum|x| + hops u_T sum|x| + ulp/2", bad, got, s,
              f"err {err[bad][:4].tolist()} bound {tol[bad][:4].tolist()}")


def check_complex(dt, op, x, got, cls, hops, what):
    r = COMPLEX[dt]
    n = x.shape[0]
    p, emin, p_acc = FLOATS[r]
    u = 2.0 ** -p
    exact = cls != RANDOM
    if op in ("sum", "avg"):
        s = sum_rows(x.real) + 1j * sum_rows(x.imag)
        if op == "sum":
            bad = exact & ((got.real != s.real) | (got.imag != s.imag))
            if bad.any():
                _fail(f"{what}: complex sum of Gaussian integers not exact", bad, got, s)
            tol_re = (n - 1 + hops) * u * np.abs(x.real).sum(0) + 0.5 * ulp(r, np.maximum(np.abs(got.real), np.abs(s.real)))
            tol_im = (n - 1 + hops) * u * np.abs(x.imag).sum(0) + 0.5 * ulp(r, np.maximum(np.abs(got.imag), np.abs(s.imag)))
            bad = ~exact & ((np.abs(got.real - s.real) > tol_re * 1.000001) | (np.abs(got.imag - s.imag) > tol_im * 1.000001))
            if bad.any():
                _fail(f"{what}: complex sum error above the bound", bad, got, s)
            return
        q = s / n
        e_re, e_im = round_to(r, q.real), round_to(r, q.imag)
        ok = (np.abs(got.real - e_re) <= ulp(r, np.minimum(np.abs(got.real), np.abs(e_re)))) & \
             (np.abs(got.imag - e_im) <= ulp(r, np.minimum(np.abs(got.imag), np.abs(e_im))))
        bad = exact & ~ok
        if bad.any():
            _fail(f"{what}: complex avg more than 1 ulp from the correctly rounded S/N", bad, got, e_re + 1j * e_im)
        tol = (n + 1 + hops) * u * (np.abs(x.real).sum(0) + np.abs(x.imag).sum(0)) / n + ulp(r, np.abs(q))
        bad = ~exact & (np.abs(got - q) > tol)
        if bad.any():
            _fail(f"{what}: complex avg error above the bound", bad, got, q)
        return
    P = np.prod(x, 0)
    bad = exact & ((got.real != P.real) | (got.imag != P.imag))
    if bad.any():
        _fail(f"{what}: complex product of exact inputs not exact", bad, got, P)
    mag = np.prod(np.abs(x), 0)
    tol = (2 * (n - 1) if hops else n - 1) * 4 * u * mag + ulp(r, mag)    # (ring / rhd: every product of the tree rounded to T)
    bad = ~exact & ((np.abs(got.real - P.real) > tol) | (np.abs(got.imag - P.imag) > tol))
    if bad.any():
        _fail(f"{what}: complex product error above (N-1) 4u prod|z|", bad, got, P)


@np.errstate(all="ignore")     # NaN / inf lanes are expected
def check_values(dt, op, x, got, cls, pat, hops, what):
    if dt in INTS:
        exp = int_reference(dt, op, x)
        bad = got != exp
        if bad.any():
            _fail(f"{what}: not bitwise the wrapped integer reference", bad, got, exp)
    elif dt in COMPLEX:
        check_complex(dt, op, x, got, cls, hops, what)
    else:
        check_real(dt, op, x, got, cls, pat, hops, what)


# ------------------------------------------------------------------ one collective
class Placed:
    """a buffer of `nbytes` at offset `mis` (mod 16) from 16-byte alignment, between guard bands, filled with random bytes"""

    def __init__(self, mem, nbytes, mis, g):
        self.buf = mem.alloc(nbytes + 2 * GUARD + 16)
        base = self.buf.ptr
        self.off = GUARD + ((mis - (base + GUARD)) % 16)
        self.ptr, self.nbytes = base + self.off, nbytes
        self.init = g.integers(0, 256, nbytes + 2 * GUARD + 16, dtype=np.uint8)

    def fill(self, data=None):
        b = self.init.copy()
        if data is not None:
            b[self.off:self.off + self.nbytes] = data
            self.init = b
        self.buf.write(b)

    def read(self):
        b = self.buf.read()
        return b, b[self.off:self.off + self.nbytes]

    def check_outside(self, b, what, keep=None):
        """bytes outside [off, off + nbytes) are what they were (`keep`: also these byte ranges inside)"""
        lo, hi = self.off, self.off + self.nbytes
        if not np.array_equal(b[:lo], self.init[:lo]) or not np.array_equal(b[hi:], self.init[hi:]):
            raise Violation(f"{what}: wrote outside the destination (guard band changed)")
        for a, z in keep or ():
            if not np.array_equal(b[lo + a:lo + z], self.init[lo + a:lo + z]):
                raise Violation(f"{what}: changed bytes [{a},{z}) of the buffer that are not its result")


# path -> (TUNE algorithm, zero-copy, launch note of allreduce, of reduce_scatter(v))
PATHS = {"oneshot": ("oneshot", False, "oneshot ", "oneshot_rs "), "twoshot": ("twoshot", False, "twoshot_staged", "twoshot_staged"),
         "zcopy": ("twoshot", True, "twoshot_zcopy", "twoshot_zcopy"), "ring": ("ring", False, "ring ", "ring "),
         "rhd": ("rhd", False, "rhd ", "rhd ")}


def path_env(path):
    alg, zc, _, _ = PATHS[path]
    env = {"UCC_TL_NVL_TUNE": "#".join(f"{c}:cuda:inf:@{alg}" for c in ("allreduce", "reduce_scatter", "reduce_scatterv", "reduce")
                                       if not (c == "reduce" and alg != "twoshot")),
           "UCC_TL_NVL_ALLREDUCE_ONESHOT_THRESH": "1M" if path == "oneshot" else "0", "UCC_TLS": "nvl"}
    env.update({"UCC_TL_NVL_ZCOPY": "y", "UCC_TL_NVL_ZCOPY_THRESH": "0"} if zc else {"UCC_TL_NVL_ZCOPY": "n"})
    return env


def hops_of(path, n):
    return (n - 1) if path == "ring" else (int(math.log2(n)) if path == "rhd" else 0)


class Harness:
    """what a case needs from its surroundings: mem.alloc(nbytes) -> object with .ptr, .write(uint8 array), .read() -> uint8 array;
    run(team, per-rank args); last_launch() -> launch note; args(coll, src_ptr, dst_ptr, dt, **kw) -> ucc_coll_args_t"""

    def __init__(self, mem, run, last_launch, args):
        self.mem, self.run, self.last_launch, self.args = mem, run, last_launch, args


def run_case(h, team, n, coll, path, dt, op, count, seed, mis=0, inplace=False, root=0, rs_counts=None,
             classes=(EXACT_T, EXACT_ACC, RANDOM, EDGE)):
    """one collective on team (n members): builds the inputs, runs, checks results, cross-rank identity, guards, sources and the
    kernel that ran.  count: elements of the vector (allreduce / reduce), of every block (reduce_scatter) or None (reduce_scatterv
    with rs_counts)."""
    sz = SIZE[dt]
    if coll == "reduce_scatterv":
        counts = list(rs_counts)
    elif coll == "reduce_scatter":
        counts = [count] * n
    else:
        counts = None
    total = sum(counts) if counts else count
    offs = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(int) if counts else None
    what = f"{coll} path={path} n={n} {dt} {op} count={counts if coll == 'reduce_scatterv' else count} mis={mis} " \
           f"{'inplace ' if inplace else ''}{f'root={root} ' if coll == 'reduce' else ''}seed={seed}"
    x, cls, pat = make_inputs(dt, op, total, n, seed, classes)
    g = np.random.default_rng(seed + 7)
    srcs = [Placed(h.mem, total * sz, mis, g) for _ in range(n)]
    for r in range(n):
        srcs[r].fill(encode(dt, x[r]))
    dsts = [None] * n
    args = []
    for r in range(n):
        if inplace:
            dsts[r] = srcs[r]
            if coll == "reduce_scatterv":
                kw = dict(dst_counts=counts, dst_displs=offs)
            else:
                kw = dict(count_dst=total)
            args.append(h.args(coll, None, srcs[r].ptr, dt, op=op, inplace=True, count_src=0, **kw))
            continue
        if coll == "allreduce":
            dsts[r] = Placed(h.mem, total * sz, mis, g)
            kw = dict(count_src=total, count_dst=total)
        elif coll == "reduce":
            if r == root:
                dsts[r] = Placed(h.mem, total * sz, mis, g)
            kw = dict(count_src=total, count_dst=total if r == root else 0, root=root)
        elif coll == "reduce_scatter":
            dsts[r] = Placed(h.mem, count * sz, mis, g)
            kw = dict(count_src=total, count_dst=count)
        else:
            dsts[r] = Placed(h.mem, counts[r] * sz, mis, g)
            kw = dict(count_src=total, dst_counts=counts, dst_displs=offs)
        if dsts[r] is not None:
            dsts[r].fill()
        args.append(h.args(coll, srcs[r].ptr, dsts[r].ptr if dsts[r] is not None else None, dt, op=op, **kw))
    h.run(team, args)
    note = h.last_launch()
    aligned = all(b.ptr % 16 == 0 for b in srcs + [d for d in dsts if d is not None])
    if coll.startswith("reduce_scatter"):
        aligned &= all(o * sz % 16 == 0 for o in offs)
    want = PATHS[path][3 if coll.startswith("reduce_scatter") else 2]
    if path == "zcopy" and not aligned:
        want = "twoshot_staged"
    if not note.startswith(want):
        raise Violation(f"{what}: served by `{note}`, not by the {want.strip()} kernel")
    hops = hops_of(path, n)
    outs = {}
    for r in range(n):
        if dsts[r] is None:
            continue
        b, data = dsts[r].read()
        if coll == "allreduce" or coll == "reduce":
            lo, hi = 0, total
            keep = None
        else:
            lo, hi = int(offs[r]), int(offs[r]) + counts[r]
            keep = [(0, lo * sz), (hi * sz, total * sz)] if inplace else None
            if inplace:
                data = data[lo * sz:hi * sz]
        dsts[r].check_outside(b, f"{what} rank {r}", keep)
        got = decode(dt, data)
        check_values(dt, op, x[:, lo:hi], got, cls[lo:hi], pat[lo:hi], hops, f"{what} rank {r}")
        outs[r] = data
    if coll == "allreduce":
        for r in range(1, n):
            if not np.array_equal(outs[r], outs[0]):
                d = np.flatnonzero(np.any(outs[r].reshape(-1, sz) != outs[0].reshape(-1, sz), 1))
                raise Violation(f"{what}: rank {r} differs bitwise from rank 0 in {d.size} elements, e.g. {d[:4].tolist()}")
    if not inplace:
        for r in range(n):
            b, _ = srcs[r].read()
            if not np.array_equal(b, srcs[r].init):
                raise Violation(f"{what}: source of rank {r} changed")
    return note


def small_counts(dt, n):
    """counts where vector kernels go wrong: 1, E-1, E, E+1, N*E-1, N*E+1 (E = elements of a 16-byte vector)"""
    e = 16 // SIZE[dt]
    return sorted({c for c in (1, e - 1, e, e + 1, n * e - 1, n * e + 1) if c > 0})
