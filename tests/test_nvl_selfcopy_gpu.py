"""Copy of a single-member tl/nvl team on a real GPU, through the public API, at the sizes and alignments that choose between
its two movers: the thread-copy kernel below 16 MB, one cudaMemcpyAsync from 16 MB on.  Every result is compared bitwise."""
import ctypes as C
import os

import pytest

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from ucc_b200 import capi as U  # noqa: E402
from ucc_b200.harness import UccJob, coll_args  # noqa: E402

CUDA = U.UCC_MEMORY_TYPE_CUDA
CROSS = 16 << 20          # bytes from which the copy is a cudaMemcpyAsync
DT = {"float32": torch.float32, "uint8": torch.uint8}


@pytest.fixture(scope="module")
def team():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    with UccJob(1, env={"UCC_TL_NVL_TIMEOUT": "5s"}, with_ctx_oob=False) as j:
        t = j.create_team()
        yield t
        t.destroy()


def last_launch():
    f = C.CDLL(os.path.join(os.path.dirname(U.LIB_PATH), "ucc", "libucc_tl_nvl.so")).ucc_tl_nvl_last_launch_info
    f.restype = C.c_char_p
    return f().decode()


def run(team, coll, src, dst, dt, inplace=False):
    a = coll_args(coll, dt=dt, mem_type=CUDA, src_ptr=None if inplace else src.data_ptr(), dst_ptr=dst.data_ptr(),
                  count_src=0 if inplace else src.numel(), count_dst=dst.numel(), inplace=inplace)
    torch.cuda.synchronize()   # the buffers were filled on torch's stream, which the team's stream does not wait for
    req = team.coll([a])
    st = req.run()
    req.finalize()
    assert st == U.UCC_OK, U.status_str(st)
    torch.cuda.synchronize()


def data(dt, n, seed, pad=0):
    """n random elements at element offset `pad` of a fresh allocation (pad=1 of float32: 4 bytes past 16-byte alignment)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = torch.randint(0, 256, ((n + pad) * DT[dt].itemsize,), dtype=torch.uint8, device="cuda", generator=g).view(DT[dt])
    return buf[pad:]


def same_bits(a, b):
    return torch.equal(a.view(torch.uint8), b.view(torch.uint8))   # random bit patterns include NaNs: compare the bytes


def expect_mover(nbytes):
    info = last_launch()
    if nbytes >= CROSS:
        assert info == "self_copy(cudaMemcpyAsync)", info
    else:
        assert info.startswith("self_copy "), info


# (datatype, elements, src pad, dst pad): around the crossover, a size that is no multiple of the thread copy's grid stride,
# odd uint8 counts (byte tails), and pointers 4 bytes past 16-byte alignment on either side of the crossover
CASES = [
    ("float32", CROSS // 4 - 4, 0, 0), ("float32", CROSS // 4, 0, 0), ("float32", CROSS // 4 + 4, 0, 0),
    ("float32", (5 << 20) // 4 + 12345, 0, 0),
    ("uint8", 1000003, 0, 0), ("uint8", CROSS + 7, 0, 0),
    ("float32", 1000001, 1, 0), ("float32", 1000001, 0, 1), ("float32", CROSS // 4 + 3, 1, 1), ("float32", CROSS // 4 + 3, 1, 0),
]


@pytest.mark.parametrize("dt,n,spad,dpad", CASES)
def test_self_copy(team, dt, n, spad, dpad):
    src = data(dt, n, 11, spad)
    dst = data(dt, n, 12, dpad)
    coll = "allreduce" if dt == "float32" else "allgather"
    run(team, coll, src, dst, dt)
    assert same_bits(dst, src)
    expect_mover(n * DT[dt].itemsize)


def test_self_copy_1gib_plus_4(team):
    n = (1 << 28) + 1
    src = data("float32", n, 21)
    dst = torch.zeros(n, dtype=torch.float32, device="cuda")
    run(team, "allreduce", src, dst, "float32")
    assert same_bits(dst, src)
    expect_mover(n * 4)
    del src, dst
    torch.cuda.empty_cache()


def test_self_allgather_and_inplace_above_crossover(team):
    n = 3 * CROSS // 4 + 1
    src = data("float32", n, 31)
    dst = torch.zeros(n, dtype=torch.float32, device="cuda")
    run(team, "allgather", src, dst, "float32")
    assert same_bits(dst, src)
    expect_mover(n * 4)
    keep = dst.clone()
    run(team, "allreduce", None, dst, "float32", inplace=True)
    assert same_bits(dst, keep)
    assert last_launch().startswith("self_copy "), last_launch()   # in place: nothing is copied, no cudaMemcpyAsync
