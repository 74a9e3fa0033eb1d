"""ec/cuda against the bitwise reference of tests/ec_numerics.py (the contract in tests/README.md): every task kind, datatype and
operator, in the interruptible executor and the persistent one on a user stream; counts and alignments where vector kernels go
wrong; launch-size knobs; the persistent task ring when the worker count does not divide its size; one reduction past 2^31 bytes;
and the collectives of the host transport (tl/shm), which reduce through ec/cuda on device buffers, against the same collectives
on host buffers."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from ucc_b200 import capi as U  # noqa: E402
from ucc_b200 import internal as I  # noqa: E402
from ucc_b200.harness import UccJob, coll_args  # noqa: E402

import ec_numerics as E  # noqa: E402
import nvl_numerics as V  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COPY_THRESH = 1 << 20           # EXEC_COPY_LARGE_THRESH default: multi-buffer copies from 1 MB on go to the copy engines


class DevBuf:
    def __init__(self, nbytes):
        self.t = torch.empty(max(nbytes, 1), dtype=torch.uint8, device="cuda")
        self.ptr = self.t.data_ptr()

    def write(self, b):
        self.t.copy_(torch.from_numpy(np.ascontiguousarray(b)))

    def read(self):
        return self.t.cpu().numpy()


class DevMem:
    @staticmethod
    def alloc(nbytes):
        return DevBuf(nbytes)


def cuda_env(ex):
    """inputs are written on torch's stream, the executor runs on its own streams: wait for the writes (this stream only - a
    device-wide synchronize would wait for a persistent executor's resident kernel)"""
    def run(args):
        torch.cuda.current_stream().synchronize()
        ex.run(args)
    return E.Env(DevMem, run)


@pytest.fixture(scope="module")
def job():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    j = UccJob(1)  # keeps mc/ec initialised
    yield j
    j.cleanup()


@pytest.fixture(params=["interruptible", "persistent"])
def env(job, request):
    stream = torch.cuda.Stream() if request.param == "persistent" else None
    ex = I.Executor(U.UCC_EE_CUDA_STREAM, stream.cuda_stream if stream else None)
    yield cuda_env(ex)
    ex.close()


# ------------------------------------------------------------------ the sweep (also run in subprocesses with other knobs)
def sweep_ops(env, dt, counts=None, n_list=(1, 2, 3, 9, 10, 16)):
    """every operator of dt, n sources from 1 to EC_MAX_SRCS; aligned (the 16-byte vector path) and every buffer 0..15 bytes off"""
    e = 16 // E.SIZE[dt]
    counts = counts or [c for c in (1, e - 1, e, e + 1, 1031) if c > 0]
    for i, op in enumerate(E.ops_of(dt)):
        for n in n_list:
            alpha = 1.0 / n if op == "avg" else None
            for j, count in enumerate(counts):
                mis = [0] * (n + 1) if j % 2 == 0 else [E.mis_of(dt, count + n + k) for k in range(n + 1)]
                E.run_reduce(env, dt, op, count, n, 1000 * i + 10 * n + count, mis=mis, alpha=alpha, what="ec/cuda")


def sweep_shapes(env, dt, op):
    """counts 0, a prime near 10^4 and one past 592 blocks x 512 threads x 8 (the grid-stride loop runs more than once); one
    misaligned source sends the whole task down the scalar path; in place on source 0 and on a later source"""
    alpha = 1.0 / 3 if op == "avg" else None
    e = 16 // E.SIZE[dt]
    big = 592 * 512 * (e if dt in E.INT128 else max(e, 8)) + 977    # more 16-byte vectors (or elements) than the grid has threads
    for count in (0, 10007, big):
        E.run_reduce(env, dt, op, count, 3, count + 5, mis=(0, 0, 0, 0), alpha=alpha, what="ec/cuda")
    E.run_reduce(env, dt, op, 10007, 3, 6, mis=(0, 0, 0, E.mis_of(dt, 1)), alpha=alpha, what="ec/cuda")
    E.run_reduce(env, dt, op, 10007, 3, 7, mis=(E.mis_of(dt, 3), E.mis_of(dt, 1), E.mis_of(dt, 2), 0), alpha=alpha, what="ec/cuda")
    for k in (0, 2):
        E.run_reduce(env, dt, op, 10007, 3, 8 + k, inplace=k, alpha=alpha, what="ec/cuda")


def sweep_strided_multi(env, dt, op):
    for n_src2, pad in ((0, 0), (1, 0), (1, 1), (15, 0), (15, 3), (70, 1)):
        alpha = 1.0 / (n_src2 + 1) if op == "avg" else None
        E.run_strided(env, dt, op, 301, n_src2, pad, 70 + n_src2 + pad, alpha=alpha, what="ec/cuda")
    if op != "avg":
        for nb in range(1, 8):
            E.run_multi_dst(env, dt, op, [1, 0, 33, 16, 7, 2001, 3][:nb], 90 + nb, what="ec/cuda")


KNOB_CASES = [("float32", "sum"), ("bfloat16", "avg"), ("float16", "max"), ("int64", "avg"), ("uint8", "prod"),
              ("uint128", "sum"), ("float64_complex", "prod"), ("float32_complex", "avg")]


def knob_sweep(stream):
    """what a subprocess with other launch knobs runs"""
    job = UccJob(1)
    st = torch.cuda.Stream() if stream else None
    ex = I.Executor(U.UCC_EE_CUDA_STREAM, st.cuda_stream if st else None)
    env = cuda_env(ex)
    try:
        for dt, op in KNOB_CASES:
            sweep_shapes(env, dt, op)
            sweep_ops(env, dt, counts=[1, 16 // E.SIZE[dt] + 1, 1031], n_list=(1, 3, 16))
            sweep_strided_multi(env, dt, op)
        E.run_copy(env, [COPY_THRESH - 1, 5, 0], 3)
        E.run_copy(env, [COPY_THRESH + 1, 5], 4)
    finally:
        ex.close()
    job.cleanup()


def in_subprocess(code, env, timeout=170):
    prog = f"import sys; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n" + code + "\nprint('SUBPROCESS_OK')"
    out = subprocess.run([sys.executable, "-c", prog], env=dict(os.environ, PYTHONPATH=ROOT, **env), capture_output=True, text=True,
                         timeout=timeout)
    assert "SUBPROCESS_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-5000:]


# ------------------------------------------------------------------ tests
@pytest.mark.parametrize("dt", E.DTYPES)
def test_ec_cuda_every_op(env, dt):
    sweep_ops(env, dt)


@pytest.mark.parametrize("dt", E.DTYPES)
def test_ec_cuda_shapes_inplace_strided_multi_dst(env, dt):
    for op in E.ops_of(dt):
        if op in ("sum", "avg", "max", "bxor"):
            sweep_shapes(env, dt, op)
        sweep_strided_multi(env, dt, op)


def test_ec_cuda_copies(env):
    E.run_copy(env, [1000], 1, multi=False)
    E.run_copy(env, [0, 1, 15, 16, 17, 4099, COPY_THRESH - 1], 2)         # copy kernel
    E.run_copy(env, [COPY_THRESH, 1, 17, COPY_THRESH + 1], 3)              # copy engines
    E.run_copy(env, [3 * COPY_THRESH + 5], 4, mis=[7], multi=False)


def test_ec_cuda_refusals(job):
    """AVG without alpha is refused by every reduce kind (REDUCE_STRIDED and REDUCE_MULTI_DST used to return a plain SUM); 17
    sources and 8 multi-dst buffers are refused"""
    n = 64
    a, b, d = (torch.ones(n * 17, device="cuda") for _ in range(3))
    torch.cuda.current_stream().synchronize()
    ex_args = [E.reduce_args(d.data_ptr(), [a.data_ptr(), b.data_ptr()], n, "float32", "avg"),
               E.strided_args(d.data_ptr(), a.data_ptr(), b.data_ptr(), n * 4, 1, n, "float32", "avg"),
               E.multi_dst_args([d.data_ptr()], [a.data_ptr()], [b.data_ptr()], [n], "float32", "avg"),
               E.multi_dst_args([d.data_ptr()], [a.data_ptr()], [b.data_ptr()], [n], "float32", "avg"),
               E.reduce_args(d.data_ptr(), [a.data_ptr() + 4 * n * k for k in range(17)], n, "float32", "sum"),
               E.multi_dst_args([d.data_ptr()] * 7, [a.data_ptr()] * 7, [b.data_ptr()] * 7, [n] * 7, "float32", "sum")]
    ex_args[3].flags |= I.EEE_FLAG_ALPHA                 # multi-dst has no alpha to scale by: AVG is refused with the flag too
    ex_args[5].reduce_multi_dst.n_bufs = 8
    names = ["reduce avg", "strided avg", "multi_dst avg", "multi_dst avg+flag", "reduce 17 sources", "multi_dst 8 buffers"]
    ex = I.Executor(U.UCC_EE_CUDA_STREAM)
    try:
        accepted = [nm for nm, args in zip(names, ex_args) if E.post_status(ex, args) == U.UCC_OK]
    finally:
        ex.close()
    assert not accepted, f"accepted: {accepted}"
    assert torch.equal(d, torch.ones_like(d))


@pytest.mark.parametrize("knobs", [{"UCC_EC_CUDA_REDUCE_NUM_BLOCKS": "1"}, {"UCC_EC_CUDA_REDUCE_NUM_THREADS": "32"},
                                   {"UCC_EC_CUDA_REDUCE_NUM_THREADS": "1024"}], ids=["blocks1", "threads32", "threads1024"])
def test_ec_cuda_reduce_launch_knobs(job, knobs):
    in_subprocess("import test_ec_numerics_gpu as T; T.knob_sweep(stream=False)", knobs)


@pytest.mark.parametrize("knobs", [{"UCC_EC_CUDA_EXEC_NUM_THREADS": "64"}, {"UCC_EC_CUDA_EXEC_NUM_WORKERS": "4"}],
                         ids=["exec_threads64", "workers4"])
def test_ec_cuda_persistent_knobs(job, knobs):
    in_subprocess("import test_ec_numerics_gpu as T; T.knob_sweep(stream=True)", knobs)


RING = r'''
import ctypes as C, time, numpy as np, torch
from ucc_b200 import capi as U, internal as I
from ucc_b200.harness import UccJob
import ec_numerics as E
slots, big = %d, %d
job = UccJob(1)
st = torch.cuda.Stream()
g = torch.Generator(device="cuda").manual_seed(5)
def task(k):
    n = big if k == 1 else 1000 + 37 * k
    s = [torch.randint(-1000, 1000, (n,), device="cuda", dtype=torch.int32, generator=g) for _ in range(3)]
    return s, (s[0] + s[1] + s[2]).cpu(), n
tasks = [task(k) for k in range(4 * 8)]
torch.cuda.current_stream().synchronize()
ex = I.Executor(U.UCC_EE_CUDA_STREAM, st.cuda_stream)
posted, bad, t0 = [], [], time.monotonic()
def done(k, deadline=60.0):
    while I.lib.ucc_ee_executor_task_test(posted[k]) == U.UCC_INPROGRESS:
        if time.monotonic() - t0 > deadline:
            raise TimeoutError(f"task {k} not done after {deadline} s")
def wait(k):
    done(k)
    I.lib.ucc_ee_executor_task_finalize(posted[k])
def post(k):
    s, _, n = tasks[k]
    a = E.reduce_args(s[0].data_ptr(), [x.data_ptr() for x in s], n, "int32", "sum")   # in place on source 0
    t = C.c_void_p()
    rc = I.lib.ucc_ee_executor_task_post(ex.h, C.byref(a), C.byref(t))
    return rc, t
def check(ks):
    """results of tasks ks (in place on source 0), compared on the host: while the executor runs, this process only copies - a
    torch kernel launched for the first time loads its module lazily, which can wait for the resident executor kernel"""
    for k in ks:
        s, exp, n = tasks[k]
        got = s[0].cpu()
        if not torch.equal(got, exp):
            d = int((got != exp).nonzero().flatten()[0])
            twice = int(exp[d]) + int(s[1][d:d + 1].cpu()[0]) + int(s[2][d:d + 1].cpu()[0])
            bad.append(f"task {k}: {int((got != exp).sum())} of {n} elements wrong, e.g. [{d}] = {int(got[d])} expected {int(exp[d])} "
                       f"(twice the sources: {twice})")
    assert not bad, "\n".join(bad)
try:
    for k in range(slots):                  # one lap: a task run twice shows here, before any slot is reused
        rc, t = post(k)
        assert rc == U.UCC_OK, f"post {k}: {U.status_str(rc)}"
        posted.append(t)
    for k in range(slots):
        done(k)
    check(range(slots))
    for k in range(slots, len(tasks)):      # three more laps: the ring is full until the oldest task is finalized
        rc, _ = post(k)
        assert rc == U.UCC_ERR_NO_RESOURCE, f"post {k} into a full ring of {slots}: {U.status_str(rc)}"
        wait(k - slots)
        rc, t = post(k)
        assert rc == U.UCC_OK, f"post {k}: {U.status_str(rc)}"
        posted.append(t)
    for k in range(len(tasks) - slots, len(tasks)):
        wait(k)
finally:
    ex.close()      # the shutdown flag makes every worker return, also after a failure
st.synchronize()
check(range(slots, len(tasks)))
job.cleanup()
'''


@pytest.mark.parametrize("workers,slots", [(3, 8), (4, 2)])
def test_ec_cuda_persistent_ring_never_runs_a_task_twice(job, workers, slots):
    """worker w serves tasks w, w + W, ... in slot idx %% n_slots.  With W = 3 and 8 slots worker 0 reaches task 9 (slot 1) while
    worker 1 still runs task 1 there, a large in-place reduce: without the slot's task index it ran task 1 a second time - an
    in-place sum counted twice - and marked it done early.  One full lap, checked before any slot is reused, then three more laps that
    wait for the oldest task; a post into a full ring is refused until the oldest task is finalized.  W = 4 > 2 slots as well."""
    big = 96 << 20 if slots == 8 else 8 << 20                     # 384 MB of int32 per source for the long task
    in_subprocess(RING % (slots, big), {"UCC_EC_CUDA_EXEC_NUM_WORKERS": str(workers), "UCC_EC_CUDA_EXEC_MAX_TASKS": str(slots)})


def test_ec_cuda_reduce_past_2g_bytes(job):
    """int8 SUM of 2^31 + 17 elements: byte offsets past 2^31, reference computed on the device with torch's wrapping int8 add"""
    n = (1 << 31) + 17
    if torch.cuda.mem_get_info()[0] < 8 * (1 << 30):
        pytest.skip("needs 8 GB of free device memory")
    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.randint(-128, 128, (n,), dtype=torch.int8, device="cuda", generator=g)
    b = torch.randint(-128, 128, (n,), dtype=torch.int8, device="cuda", generator=g)
    d = torch.zeros(n, dtype=torch.int8, device="cuda")
    torch.cuda.current_stream().synchronize()
    ex = I.Executor(U.UCC_EE_CUDA_STREAM)
    try:
        ex.run(E.reduce_args(d.data_ptr(), [a.data_ptr(), b.data_ptr()], n, "int8", "sum"))
    finally:
        ex.close()
    a += b
    assert torch.equal(d, a), f"{int((d != a).sum())} elements differ, first at {int((d != a).nonzero()[0])}"


# ------------------------------------------------------------------ tl/shm on host and device buffers
SHM_ALGS = {"allreduce": ["knomial", "sra_knomial", "dbt", "ring", "sliding_window"], "reduce": ["knomial", "dbt", "srg"],
            "reduce_scatter": ["ring", "knomial"], "reduce_scatterv": [None]}
TWIN_DTS = ["float32", "bfloat16", "float16", "float64", "float32_complex", "float64_complex", "int8", "uint16", "int32", "int64",
            "uint64"]


def shm_collective(team, n, coll, mem, mt, dt, op, x, count, seed, root, rs_counts):
    """one collective, inputs x, on buffers of `mem`; returns per-rank result bytes, after checking guards and sources"""
    sz = V.SIZE[dt]
    g = np.random.default_rng(seed)
    total = x.shape[1]
    offs = np.concatenate([[0], np.cumsum(rs_counts)[:-1]]).astype(int) if rs_counts is not None else None
    srcs = [V.Placed(mem, total * sz, 0, g) for _ in range(n)]
    for r in range(n):
        srcs[r].fill(V.encode(dt, x[r]))
    dsts, args = [], []
    for r in range(n):
        kw = dict(count_src=total)
        if coll == "allreduce" or (coll == "reduce" and r == root):
            d = V.Placed(mem, total * sz, 0, g)
            kw.update(count_dst=total, root=root)
        elif coll == "reduce":
            d = None
            kw.update(count_dst=0, root=root)
        elif coll == "reduce_scatter":
            d = V.Placed(mem, count * sz, 0, g)
            kw.update(count_dst=count)
        else:
            d = V.Placed(mem, rs_counts[r] * sz, 0, g)
            kw.update(dst_counts=rs_counts, dst_displs=offs)
        if d is not None:
            d.fill()
        dsts.append(d)
        args.append(coll_args(coll, dt=dt, op=op, mem_type=mt, src_ptr=srcs[r].ptr, dst_ptr=d.ptr if d else None, **kw))
    if mt == U.UCC_MEMORY_TYPE_CUDA:
        torch.cuda.synchronize()
    req = team.coll(args)
    st = req.run()
    req.finalize()
    assert st == U.UCC_OK, U.status_str(st)
    if mt == U.UCC_MEMORY_TYPE_CUDA:
        torch.cuda.synchronize()
    outs = {}
    for r in range(n):
        b = srcs[r].buf.read()
        assert np.array_equal(b, srcs[r].init), f"source of rank {r} changed"
        if dsts[r] is not None:
            b, data = dsts[r].read()
            dsts[r].check_outside(b, f"rank {r}")
            outs[r] = data
    return outs


def same_bits(dt, a, b):
    """bitwise equal, lanes where both are NaN aside (x86 and the GPU make different NaN payloads)"""
    sz = V.SIZE[dt]
    diff = np.any(a.reshape(-1, sz) != b.reshape(-1, sz), 1)
    if dt in V.INTS:
        return ~diff
    va, vb = V.decode(dt, a), V.decode(dt, b)
    with np.errstate(invalid="ignore"):
        return ~diff | (np.isnan(va) & np.isnan(vb))


def shm_twin(team, n, coll, dt, op, seed, root=0):
    count = 1000 + 13 * n if coll != "reduce_scatterv" else None
    rs_counts = [37 * (r % 3) + (r == 1) for r in range(n)] if coll == "reduce_scatterv" else None
    total = count * n if coll == "reduce_scatter" else (sum(rs_counts) if rs_counts else count)
    x, cls, pat = V.make_inputs(dt, op, total, n, seed)
    what = f"tl/shm {coll} n={n} {dt} {op} root={root} seed={seed}"
    host = shm_collective(team, n, coll, E.HostMem, U.UCC_MEMORY_TYPE_HOST, dt, op, x, count, seed, root, rs_counts)
    dev = shm_collective(team, n, coll, DevMem, U.UCC_MEMORY_TYPE_CUDA, dt, op, x, count, seed, root, rs_counts)
    for r, hb in host.items():
        if coll in ("allreduce", "reduce"):
            lo, hi = 0, total
        elif coll == "reduce_scatter":
            lo, hi = r * count, (r + 1) * count
        else:
            lo = sum(rs_counts[:r])
            hi = lo + rs_counts[r]
        for side, b in (("host", hb), ("cuda", dev[r])):
            V.check_values(dt, op, x[:, lo:hi], V.decode(dt, b), cls[lo:hi], pat[lo:hi], n - 1, f"{what} {side} buffers rank {r}")
        if not (dt in V.COMPLEX and op == "prod"):
            ok = same_bits(dt, hb, dev[r])
            if not ok.all():
                V._fail(f"{what} rank {r}: CUDA buffers differ from host buffers", ~ok, V.decode(dt, dev[r]), V.decode(dt, hb))


@pytest.mark.parametrize("n", [4, 5])
@pytest.mark.parametrize("coll,alg", [(c, a) for c, algs in SHM_ALGS.items() for a in algs])
def test_shm_host_and_cuda_buffers_agree(job, coll, alg, n):
    """the same tl/shm collective on host buffers (ec/cpu) and on CUDA buffers (ec/cuda) gives the same bits, AVG included, and
    meets the contract of tests/README.md with hops = N-1"""
    if alg == "sliding_window":   # reads the peers' buffers in place (pointer / CMA): host memory only, CUDA buffers fall back
        pytest.skip("tl/shm allreduce @sliding_window refuses CUDA buffers")
    if coll == "reduce_scatter" and alg == "knomial" and n & (n - 1):   # (k^m ranks with k = REDUCE_SCATTER_KN_RADIX, or 2^m)
        pytest.skip(f"tl/shm reduce_scatter @knomial refuses a team of {n}: another algorithm would run under its name")
    env = {"UCC_TLS": "shm,self"}
    if alg:
        env["UCC_TL_SHM_TUNE"] = f"{coll}:inf:@{alg}"
    with UccJob(n, env=env) as j:
        team = j.create_team(range(n))
        for k, dt in enumerate(TWIN_DTS):
            for i, op in enumerate(V.ops_of(dt)):
                if dt in V.INTS and op not in ("sum", "prod", "max", "bxor", "avg"):
                    continue
                roots = (0, n - 1) if coll == "reduce" else (0,)
                for root in roots:
                    try:
                        shm_twin(team, n, coll, dt, op, 100 * k + 10 * i + root, root)
                    except U.UccError as e:
                        if e.status == U.UCC_ERR_NOT_SUPPORTED:
                            pytest.skip(f"tl/shm {coll} @{alg} refuses {dt} {op} on CUDA buffers")
                        raise
        team.destroy()


@pytest.mark.parametrize("n", [4, 5])
def test_int_avg_shm_matches_nvl(job, n):
    """integer AVG of CUDA buffers: tl/shm (ec/cuda, exact division by N) and tl/nvl give the same bits"""
    count = 4099
    res = {}
    dts = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64"]
    xs = {dt: V.make_inputs(dt, "avg", count, n, 7 + k)[0] for k, dt in enumerate(dts)}
    nvl = {"UCC_TLS": "nvl", "UCC_TL_NVL_MAX_BLOCKS": "4", "UCC_TL_NVL_TIMEOUT": "5s", "UCC_TL_NVL_SYMMETRIC_SIZE": "1Mb"}
    for tl, env in (("shm", {"UCC_TLS": "shm,self"}), ("nvl", nvl)):
        with UccJob(n, env=env) as j:
            team = j.create_team(range(n), team_id=7)      # (a job of tl/nvl alone has no service team to allocate the id)
            for dt in dts:
                res[tl, dt] = shm_collective(team, n, "allreduce", DevMem, U.UCC_MEMORY_TYPE_CUDA, dt, "avg", xs[dt], count, 3, 0, None)
            team.destroy()
    for dt in dts:
        exp = V.int_reference(dt, "avg", xs[dt])
        for r in range(n):
            for tl in ("shm", "nvl"):
                got = V.decode(dt, res[tl, dt][r])
                if not np.array_equal(got, exp):
                    V._fail(f"tl/{tl} allreduce {dt} avg n={n} rank {r}: not trunc(wrapped sum / N)", got != exp, got, exp)


def triggered_allreduce(n=4, count=30011):
    """what test_shm_triggered_allreduce_on_cuda_buffers runs in its own process: tl/shm allreduces of CUDA buffers posted with
    ucc_collective_triggered_post on one user stream per rank, so each rank's persistent executor serves the collective's reduce
    and copy tasks through tl/shm's own post / test / finalize loop; every result against the contract and bitwise against the
    same allreduce posted without a stream (interruptible executor)"""
    import time
    cases = [("float32", "avg"), ("bfloat16", "sum"), ("int64", "avg"), ("float64_complex", "sum"), ("uint8", "max")]
    with UccJob(n, env={"UCC_TLS": "shm,self"}) as j:
        team = j.create_team(range(n))
        streams, ees = [torch.cuda.Stream() for _ in range(n)], []
        for r in range(n):
            ep = U.ucc_ee_params_t()
            ep.ee_type, ep.ee_context, ep.ee_context_size = U.UCC_EE_CUDA_STREAM, streams[r].cuda_stream, C.sizeof(C.c_void_p)
            ee = U.handle()
            U.check(U.ucc_ee_create(team.members[r].team, C.byref(ep), C.byref(ee)), "ee_create")
            ees.append(ee)
        for k, (dt, op) in enumerate(cases):
            x, cls, pat = V.make_inputs(dt, op, count, n, 500 + k)
            ref = shm_collective(team, n, "allreduce", DevMem, U.UCC_MEMORY_TYPE_CUDA, dt, op, x, count, 9, 0, None)
            g = np.random.default_rng(k)
            srcs = [V.Placed(DevMem, count * V.SIZE[dt], 0, g) for _ in range(n)]
            dsts = [V.Placed(DevMem, count * V.SIZE[dt], 0, g) for _ in range(n)]
            for r in range(n):
                srcs[r].fill(V.encode(dt, x[r]))
                dsts[r].fill()
            torch.cuda.current_stream().synchronize()
            reqs = []
            for r in range(n):
                a = coll_args("allreduce", dt=dt, op=op, mem_type=U.UCC_MEMORY_TYPE_CUDA, src_ptr=srcs[r].ptr, dst_ptr=dsts[r].ptr,
                              count_src=count, count_dst=count)
                q = C.POINTER(U.ucc_coll_req_t)()
                U.check(U.ucc_collective_init(C.byref(a), C.byref(q), team.members[r].team), "init")
                ev = U.ucc_ev_t()
                ev.ev_type, ev.req = U.UCC_EVENT_COMPUTE_COMPLETE, C.cast(q, C.c_void_p)
                U.check(U.ucc_collective_triggered_post(ees[r], C.byref(ev)), "triggered_post")
                reqs.append((a, q))
            t0 = time.monotonic()
            while any(q.contents.status == U.UCC_INPROGRESS for _, q in reqs):
                for r in range(n):
                    U.ucc_context_progress(j.procs[r].ctx)
                    e = C.POINTER(U.ucc_ev_t)()
                    while U.ucc_ee_get_event(ees[r], C.byref(e)) == U.UCC_OK:
                        U.ucc_ee_ack_event(ees[r], e)
                if time.monotonic() - t0 > 60:
                    # the collective's executors stop only when it completes: this process exits with the failure, and its CUDA
                    # context - the resident executor kernels with it - ends there
                    raise TimeoutError(f"triggered {dt} {op} allreduce not complete after 60 s: {[q.contents.status for _, q in reqs]}")
            for r in range(n):       # completion stopped the executor: its kernel has left the stream
                streams[r].synchronize()
                assert reqs[r][1].contents.status == U.UCC_OK, U.status_str(reqs[r][1].contents.status)
                U.check(U.ucc_collective_finalize(reqs[r][1]), "finalize")
            what = f"triggered tl/shm allreduce n={n} {dt} {op}"
            for r in range(n):
                b, data = dsts[r].read()
                dsts[r].check_outside(b, f"{what} rank {r}")
                assert np.array_equal(srcs[r].buf.read(), srcs[r].init), f"{what}: source of rank {r} changed"
                V.check_values(dt, op, x, V.decode(dt, data), cls, pat, n - 1, f"{what} rank {r}")
                ok = same_bits(dt, ref[r], data)
                if not ok.all():
                    V._fail(f"{what} rank {r}: differs from the allreduce posted without a stream", ~ok, V.decode(dt, data),
                            V.decode(dt, ref[r]))
        for ee in ees:
            U.check(U.ucc_ee_destroy(ee), "ee_destroy")
        team.destroy()


@pytest.mark.parametrize("knobs", [{}, {"UCC_EC_CUDA_EXEC_NUM_WORKERS": "3", "UCC_EC_CUDA_EXEC_MAX_TASKS": "8"}],
                         ids=["default", "workers3_slots8"])
def test_shm_triggered_allreduce_on_cuda_buffers(job, knobs):
    """a real collective served by the persistent executor (the default ring, and 3 workers on 8 slots)"""
    in_subprocess("import test_ec_numerics_gpu as T; T.triggered_allreduce()", knobs)
