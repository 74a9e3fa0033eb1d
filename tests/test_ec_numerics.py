"""ec/cpu against the bitwise reference of tests/ec_numerics.py (the contract in tests/README.md): every datatype and operator,
1..16 sources, in place, REDUCE_STRIDED, REDUCE_MULTI_DST, copies, AVG on every type - floats scale by alpha rounded to the
accumulator's precision, integers divide the wrapped sum exactly by N up to the limits of int64 / uint64 - and the refusal of AVG
without alpha.  The same cases run on ec/cuda in tests/test_ec_numerics_gpu.py."""
import numpy as np
import pytest

from ucc_b200 import capi as U
from ucc_b200 import internal as I
from ucc_b200.harness import UccJob

import ec_numerics as E


@pytest.fixture(scope="module")
def env():
    job = UccJob(1)  # keeps mc/ec initialised
    ex = I.Executor(U.UCC_EE_CPU_THREAD)
    yield E.Env(E.HostMem, ex.run)
    ex.close()
    job.cleanup()


def host_mis(dt, k):
    # ec/cpu loads 128-bit integers with 16-byte vector instructions: those stay aligned on the host
    return 0 if dt in E.INT128 else E.mis_of(dt, k)


@pytest.mark.parametrize("dt", E.DTYPES)
def test_ec_cpu_reduce_every_op(env, dt):
    e = 16 // E.SIZE[dt]
    for i, op in enumerate(E.ops_of(dt)):
        for n in (1, 2, 3, 9, 10, 16):
            alpha = 1.0 / n if op == "avg" else None
            for count in (1, e - 1, e + 1, 1031):
                if count < 1:
                    continue
                mis = [host_mis(dt, count + n + k) for k in range(n + 1)]
                E.run_reduce(env, dt, op, count, n, 1000 * i + 10 * n + count, mis=mis, alpha=alpha, what="ec/cpu")


@pytest.mark.parametrize("dt", E.DTYPES)
def test_ec_cpu_reduce_inplace_strided_multi_dst(env, dt):
    for i, op in enumerate(E.ops_of(dt)):
        alpha = 1.0 / 4 if op == "avg" else None
        for k in (0, 2):
            E.run_reduce(env, dt, op, 517, 4, 50 + i, inplace=k, alpha=alpha, what="ec/cpu")
        for n_src2, pad in ((0, 0), (1, 0), (15, 1), (15, 0)):
            a = 1.0 / (n_src2 + 1) if op == "avg" else None
            E.run_strided(env, dt, op, 301, n_src2, pad, 70 + i, alpha=a, what="ec/cpu")
        if op != "avg":
            E.run_multi_dst(env, dt, op, [1, 0, 33, 16, 7, 200, 3][:4 + i % 4], 90 + i, mis=host_mis, what="ec/cpu")


def test_ec_cpu_copy(env):
    E.run_copy(env, [1000], 1, multi=False, what="ec/cpu")
    E.run_copy(env, [0, 1, 15, 16, 17, 4099, 100_003], 2, what="ec/cpu")


@pytest.mark.parametrize("dt", ["float32", "bfloat16", "float16", "float32_complex", "float64", "float64_complex"])
@pytest.mark.parametrize("n", [3, 5, 6, 7])
def test_ec_cpu_float_avg_scales_in_accumulator_precision(env, dt, n):
    """AVG = the in-order sum in the accumulator type times alpha rounded to that type (float for float32 / bfloat16 / float16 /
    float32 complex): the same bits ec/cuda and tl/nvl produce.  Scaling a float sum by the double alpha and rounding back differs
    in a fifth to a half of the lanes for these N."""
    for alpha in (1.0 / n, 0.3):
        E.run_reduce(env, dt, "avg", 4099, n, 7 * n, mis=[host_mis(dt, 1)], alpha=alpha, what="ec/cpu")


@pytest.mark.parametrize("dt", ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "int128", "uint128"])
def test_ec_cpu_int_avg_divides_exactly(env, dt):
    """integer AVG is trunc(wrapped sum / N) up to the limits of the type, where double(sum) * (1/N) is off (uint64 2^64-1 over 2
    gave 2^63); another alpha than 1/N scales in double and truncates"""
    for n in (1, 2, 3, 7, 16):
        E.run_reduce(env, dt, "avg", 1031, n, 300 + n, alpha=1.0 / n, what="ec/cpu")
    E.run_reduce(env, dt, "avg", 1031, 3, 399, alpha=0.3, what="ec/cpu")


@pytest.mark.parametrize("dt,vals,n,exp", [
    ("uint64", [2 ** 64 - 1, 0], 2, 2 ** 63 - 1), ("uint64", [2 ** 64 - 1, 2 ** 64 - 1, 1], 3, (2 ** 64 - 1) // 3),
    ("uint64", [2 ** 63 + 1, 2 ** 62, 1], 3, (2 ** 63 + 2 ** 62 + 2) // 3),
    ("int64", [2 ** 63 - 1, 0], 2, 2 ** 62 - 1), ("int64", [-2 ** 63, 0, 0], 3, -(2 ** 63 // 3)),
    ("int64", [2 ** 62 + 1, 2 ** 62 - 3, 0, 0, 0], 5, (2 ** 63 - 2) // 5), ("int64", [-2 ** 63 + 7, 0], 2, -(2 ** 62 - 4))])
def test_ec_cpu_int64_avg_at_the_limits(env, dt, vals, n, exp):
    src = [np.full(8, v if dt == "uint64" else np.int64(v), np.uint64 if dt == "uint64" else np.int64) for v in vals]
    src += [np.zeros(8, src[0].dtype) for _ in range(n - len(vals))]
    dst = np.zeros(8, src[0].dtype)
    env.run(E.reduce_args(dst.ctypes.data, [s.ctypes.data for s in src], 8, dt, "avg", 1.0 / n))
    assert all(int(v) == exp for v in dst), f"{dt} avg of {vals} over {n}: got {int(dst[0])}, expected {exp}"


def test_ec_avg_divisor():
    assert [E.avg_divisor(1.0 / n) for n in (1, 2, 3, 5, 7, 1000, 12345)] == [1, 2, 3, 5, 7, 1000, 12345]
    assert [E.avg_divisor(a) for a in (0.3, 0.0, 2.0, 1.0 / 3 + 2 ** -54, -0.5)] == [0, 0, 0, 0, 0]


@pytest.mark.parametrize("kind", ["reduce", "strided", "multi_dst"])
def test_ec_cpu_refuses_avg_without_alpha(env, kind):
    n = 16
    a, b, d = (np.ones(n, np.float32) for _ in range(3))
    if kind == "reduce":
        args = E.reduce_args(d.ctypes.data, [a.ctypes.data, b.ctypes.data], n, "float32", "avg")
    elif kind == "strided":
        args = E.strided_args(d.ctypes.data, a.ctypes.data, b.ctypes.data, n * 4, 1, n, "float32", "avg")
    else:
        args = E.multi_dst_args([d.ctypes.data], [a.ctypes.data], [b.ctypes.data], [n], "float32", "avg")
    ex = I.Executor(U.UCC_EE_CPU_THREAD)
    try:
        assert E.post_status(ex, args) != U.UCC_OK, f"{kind}: AVG without alpha accepted"
    finally:
        ex.close()
    assert np.array_equal(d, np.ones(n, np.float32))


def test_reference_replays_kernel_order():
    """the reference itself: bitwise for a fold that rounds (float32 sum of 1, 2^-24, 2^-24 is 1 in order, not 1 + 2^-23)"""
    case = E.Case("float32", "sum", 4, 3, 0)
    case.x = np.array([[1.0] * 4, [2.0 ** -24] * 4, [2.0 ** -24] * 4])
    assert list(E.reference(case)) == [1.0] * 4
    case.op = "max"
    case.x = np.array([[0.0, -0.0, np.nan, 1.0], [-0.0, 0.0, 1.0, np.nan]])
    case.n = 2
    r = E.reference(case)
    assert np.signbit(r[0]) and not np.signbit(r[1]) and r[2] == 1.0 and np.isnan(r[3])
