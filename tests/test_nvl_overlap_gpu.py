"""UCC_COLL_ARGS_HINT_OPTIMIZE_OVERLAP_GPU on tl/nvl on a real GPU: the cases of tests/nvl_overlap.py with N emulated ranks on
cuda:0 (up to 8), and two processes on the same GPU, whose buffers cross the exchange board as CUDA IPC handles, through the torch
backend (tests/overlap_torch_worker.py).  With emulated ranks on one GPU the copy engines move data inside its HBM, not over NVLink;
what is checked is which path runs and what it computes."""
import os
import subprocess
import sys

import numpy as np
import pytest

# emulated ranks share one GPU: every rank's stream needs a hardware queue of its own, or a copy queued behind one rank's spinning
# barrier kernel can hold up another rank's barrier kernel in the same queue (as in tests/test_nvl_numerics_gpu.py)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from test_nvl_managed_gpu import H as ManagedH, need_cuda  # noqa: E402
from ucc_b200 import capi as U  # noqa: E402
from ucc_b200.harness import UccJob, coll_args  # noqa: E402

import nvl_numerics as V  # noqa: E402
import nvl_overlap as O  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENV = dict(O.ENV, UCC_TL_NVL_MAX_BLOCKS="4", UCC_TL_NVL_TIMEOUT="10s")


class Bytes:
    def __init__(self, nbytes):
        self.t = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        self.ptr = self.t.data_ptr()

    def write(self, b):
        self.t.copy_(torch.from_numpy(np.ascontiguousarray(b)))

    def read(self):
        return self.t.cpu().numpy()


class H(ManagedH):
    class mem:
        @staticmethod
        def alloc(nbytes):
            return Bytes(nbytes)

    @staticmethod
    def nargs(coll, sp, dp, dt, **kw):
        return coll_args(coll, dt=dt, mem_type=U.UCC_MEMORY_TYPE_CUDA, src_ptr=sp, dst_ptr=dp, **kw)


@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_overlap_numerics(n):
    need_cuda()
    with UccJob(n, env=ENV) as j:
        O.run_numerics(H(False), j.create_team(range(n), team_id=n), n, V.ALL_DTYPES, seed=1000 * n)


def test_overlap_rounds():
    need_cuda()
    with UccJob(4, env=dict(ENV, UCC_TL_NVL_SYMMETRIC_SIZE="256K")) as j:
        for n in (2, 3, 4):
            O.run_rounds(H(False), j.create_team(range(n), team_id=n), n, 256 << 10)


def test_overlap_collectives():
    need_cuda()
    h = H(False)
    with UccJob(8, env=ENV) as j:
        for n in (2, 3, 4, 8):
            team = j.create_team(range(n), team_id=n)
            O.run_colls(h, team, n, seed=100 * n)
            O.run_vforms(h, team, n)
        h.free()


def test_overlap_persistent_registered_fallbacks():
    need_cuda()
    h = H(False)
    with UccJob(4, env=ENV) as j:
        for n in (2, 4):
            team = j.create_team(range(n), team_id=n)
            O.run_persistent(h, team, n)
            O.run_registered(h, team, n, [j.procs[r].ctx for r in range(n)])
            O.run_fallbacks(h, team, n)
        h.free()
    with UccJob(1, env=ENV, with_ctx_oob=False) as j:
        O.run_self(h, j.create_team(team_id=1))
        h.free()


def test_overlap_torch_two_processes():
    need_cuda()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29917", os.path.join(ROOT, "tests", "overlap_torch_worker.py")]
    env = {k: v for k, v in os.environ.items() if k not in ("UCC_TLS", "UCC_TL_NVL_TUNE")}   # (the backend's service team needs tl/shm)
    out = subprocess.run(cmd, env=dict(env, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=300)
    assert "OVERLAP_TORCH_OK" in out.stdout, out.stdout[-4000:] + out.stderr[-4000:]
