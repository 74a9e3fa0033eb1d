"""Multi-process, one process per GPU: VMM heap exchange, NVLS binding and the fused kernels over real NVLink."""
import os
import subprocess
import sys

import pytest

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _run(n, extra_env=None):
    port = 29700 + n
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "dist_worker.py"), "cuda"]
    env = dict(os.environ, PYTHONPATH=ROOT)
    env.update(extra_env or {})
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=150)
    assert "DIST_WORKER_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


def test_multiproc_all_gpus():
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    _run(n)


def test_multiproc_no_nvls():
    n = min(2, torch.cuda.device_count()) if torch.cuda.is_available() else 0   # validated on 2 GPUs
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    _run(n, {"UCC_TL_NVL_USE_NVLS": "n"})


def test_multiproc_ipc_heap():
    n = min(2, torch.cuda.device_count()) if torch.cuda.is_available() else 0   # validated on 2 GPUs
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    _run(n, {"UCC_TL_NVL_USE_VMM": "n"})


def test_multiproc_zcopy_forced():
    n = min(2, torch.cuda.device_count()) if torch.cuda.is_available() else 0   # validated on 2 GPUs
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    _run(n, {"UCC_TL_NVL_ZCOPY": "y", "UCC_TL_NVL_ZCOPY_THRESH": "0"})


def test_multiproc_no_zcopy():
    n = min(2, torch.cuda.device_count()) if torch.cuda.is_available() else 0   # validated on 2 GPUs
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    _run(n, {"UCC_TL_NVL_ZCOPY": "n"})


def test_parallel_helpers_cuda():
    """DDP buckets / tensor parallel / MoE alltoallv on CUDA tensors through the tl/nvl kernels."""
    n = min(2, torch.cuda.device_count()) if torch.cuda.is_available() else 0   # validated on 2 GPUs
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29790", os.path.join(ROOT, "tests", "parallel_worker.py"), "cuda"]
    out = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=150)
    assert "PARALLEL_WORKER_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


def test_multiproc_nvls_everything():
    """NVLS variants forced: in-switch allreduce / reduce_scatter (float and integer), multicast allgather / bcast."""
    n = min(2, torch.cuda.device_count()) if torch.cuda.is_available() else 0   # validated on 2 GPUs
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    _run(n, {"UCC_TL_NVL_TUNE": "allreduce:cuda:inf:@nvls#reduce_scatter:cuda:inf:@nvls#allgather:cuda:inf:@nvls#bcast:cuda:inf:@nvls", "UCC_TL_NVL_ALLREDUCE_ONESHOT_THRESH": "0"})


def test_multiproc_ring_rhd():
    n = min(2, torch.cuda.device_count()) if torch.cuda.is_available() else 0   # validated on 2 GPUs
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    _run(n, {"UCC_TL_NVL_TUNE": "allreduce:cuda:inf:@ring#reduce_scatter:cuda:inf:@rhd#allgather:cuda:inf:@ring", "UCC_TL_NVL_ZCOPY": "n"})


@pytest.mark.parametrize("alg", ["rab", "split_rail"])
def test_multiproc_hier_fake_nodes(alg):
    """cl/hier schedules on CUDA buffers with real processes: every GPU pretends to be its own node (UCC_B200_FAKE_PPN=1), so node
    sub-teams are single-member tl/nvl teams and the leaders / rail sub-teams cross "nodes" (host TL + mc/ec staging)."""
    n = min(2, torch.cuda.device_count()) if torch.cuda.is_available() else 0
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    _run(n, {"UCC_B200_FAKE_PPN": "1", "UCC_CLS": "hier,basic", "UCC_CL_HIER_TUNE": f"allreduce:0-inf:@{alg}"})


def test_multiproc_asymmetric_memory_at_root():
    """reference asym_mem tests with one process per GPU: root's src / dst in different memory types around tl/nvl collectives
    (in the one-device emulation this couples the ranks through device-wide synchronisation, see tests/test_nvl_gpu.py)"""
    n = min(2, torch.cuda.device_count()) if torch.cuda.is_available() else 0
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    _run(n, {"DW_ASYM": "1"})


def test_torch_backend_cuda():
    """init_process_group("ucc_b200"): c10d collectives and torch DDP on CUDA tensors run on the tl/nvl kernels."""
    n = min(2, torch.cuda.device_count()) if torch.cuda.is_available() else 0   # validated on 2 GPUs
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29795", os.path.join(ROOT, "tests", "pg_worker.py"), "cuda"]
    out = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=150)
    assert "PG_WORKER_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


@pytest.mark.skipif(os.environ.get("UCC_B200_EXPERIMENTAL_TESTS") != "1", reason="opt-in multi-GPU test of nvls_pipe: set UCC_B200_EXPERIMENTAL_TESTS=1")
@pytest.mark.parametrize("heap", ["128M", "24M"])
def test_multiproc_nvls_pipe(heap):
    """Pipelined staged NVLS allreduce (kernels/nvl_pipe.cuh); the small heap forces many chunks so the three buffers rotate."""
    n = min(2, torch.cuda.device_count()) if torch.cuda.is_available() else 0
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    _run(n, {"UCC_TL_NVL_TUNE": "allreduce:cuda:inf:@nvls_pipe", "UCC_TL_NVL_ALLREDUCE_ONESHOT_THRESH": "0", "UCC_TL_NVL_SYMMETRIC_SIZE": heap})


@pytest.mark.skipif(os.environ.get("UCC_B200_EXPERIMENTAL_TESTS") != "1", reason="opt-in multi-GPU test of the symmetric-memory allreduce: set UCC_B200_EXPERIMENTAL_TESTS=1")
def test_multiproc_symm():
    """allreduce on tensors inside the symmetric user region: in-place multimem.ld_reduce / multimem.st (kernels/nvl_symm.cuh)"""
    n = min(2, torch.cuda.device_count()) if torch.cuda.is_available() else 0
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29741", os.path.join(ROOT, "tests", "symm_worker.py")]
    out = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT, SYMM_BENCH_BYTES=str(256 << 20)), capture_output=True, text=True, timeout=150)
    assert "SYMM_WORKER_OK" in out.stdout or "SYMM_WORKER_SKIP" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


@pytest.mark.skipif(os.environ.get("UCC_B200_EXPERIMENTAL_TESTS") != "1", reason="opt-in multi-GPU test of the push exchange: set UCC_B200_EXPERIMENTAL_TESTS=1")
def test_multiproc_push_exchange():
    """zero-copy push allgather / alltoall (kernels/nvl_push.cu) instead of the pull kernels"""
    n = min(2, torch.cuda.device_count()) if torch.cuda.is_available() else 0
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    _run(n, {"UCC_TL_NVL_TUNE": "allgather:cuda:inf:@push#alltoall:cuda:inf:@push#alltoallv:cuda:inf:@push"})
