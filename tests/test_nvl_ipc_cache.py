"""The per-peer CUDA IPC cache of tl/nvl (tl_nvl_direct.c) against the emulated CUDA runtime, from a compiled C driver.

Teams inside one process publish raw pointers and never map anything, so the driver plays both members of a two-member team
itself: two team objects share their exchange boards, and every buffer goes through the emulated cudaIpcGetMemHandle /
cudaIpcOpenMemHandle of tests/emu/cudart_emu.cpp.  A persistent allreduce resolves the zero-copy (direct) tables on its first post; then more distinct peer
allocations than the cache holds are mapped, and the persistent request's tables are launched again.  The mappings those tables
point into must still be open: the emulated launcher refuses a kernel whose tables reach into a closed mapping."""
import os
import subprocess

from test_nvl_hostemu import emu_build  # noqa: F401  (module fixture: builds the host-emulated runtime and plugin)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r'''
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "components/tl/nvl/tl_nvl.h"
#define CHECK(c) do { if (!(c)) { printf("FAIL line %d: %s\n", __LINE__, #c); exit(1); } } while (0)
long emu_ipc_count(int what);

enum { N = 2, COUNT = 4096, FILLERS = 3 * NVL_IPC_CACHE_MAX / 2 };
static ucc_base_lib_t lib;
static ucc_tl_nvl_context_t ctx;
static ucc_tl_nvl_team_t team[N];
static char *heap[N];
static uint32_t host_err;
static cudaStream_t stream[N];

static float *dev_floats(size_t n) { void *p = NULL; CHECK(cudaMalloc(&p, n * sizeof(float)) == cudaSuccess); return (float *)p; }

/* both members launch the zero-copy allreduce with the tables of their plans; 0: both ran */
static int launch_direct(nvl_zc_t *zc, float **src, float **dst)
{
    int rc = 0;
    for (int r = 0; r < N; r++) {
        nvl_red_args_t a;
        memset(&a, 0, sizeof(a));
        a.team.rank = r; a.team.size = N; a.team.data_size = 1 << 20; a.team.timeout_ns = 30000000000ull; a.team.host_err = &host_err;
        for (int p = 0; p < N; p++) a.team.heap[p] = heap[p];
        a.src = src[r]; a.dst = dst[r]; a.count = COUNT; a.dt = NVL_DT_F32; a.op = NVL_OP_SUM; a.kind = NVL_RED_ALLREDUCE;
        a.direct = NVL_DIRECT_FULL; a.d = zc[r].d;
        if (nvl_launch_reduce_direct(&a, 1, 32, stream[r]) != cudaSuccess) rc = -1;
    }
    for (int r = 0; r < N; r++) cudaStreamSynchronize(stream[r]);
    return rc;
}

int main(void)
{
    nvl_xb_seg_t *seg[N];
    nvl_zc_t zc[N];
    float *src[N], *dst[N];
    lib.log_component.log_level = UCC_LOG_LEVEL_WARN;
    ctx.super.super.lib = &lib;
    for (int r = 0; r < N; r++) { seg[r] = calloc(1, sizeof(nvl_xb_seg_t)); CHECK(seg[r]); }
    for (int r = 0; r < N; r++) {
        ucc_tl_nvl_team_t *t = &team[r];
        t->super.super.context = &ctx.super.super; t->super.super.params.rank = r; t->super.super.params.size = N;
        t->heap_kind = NVL_HEAP_IPC; t->zcopy = 1; t->xb_mine = seg[r];
        for (int p = 0; p < N; p++) t->xb[p] = seg[p];
        CHECK(cudaMalloc((void **)&heap[r], NVL_DATA_OFFSET + (1 << 20)) == cudaSuccess);
        memset(heap[r], 0, NVL_DATA_OFFSET + (1 << 20));
        CHECK(cudaStreamCreate(&stream[r]) == cudaSuccess);
        src[r] = dev_floats(COUNT); dst[r] = dev_floats(COUNT);
        for (int i = 0; i < COUNT; i++) { src[r][i] = (float)(i % 97 + 10 * r); dst[r][i] = -1.f; }
    }
    /* first post of a persistent allreduce: both members publish, both map the other's src and dst */
    for (int r = 0; r < N; r++) ucc_tl_nvl_zc_init(&team[r], &zc[r], NVL_ZC_SRC | NVL_ZC_DST | NVL_ZC_ALIGN, src[r], COUNT * 4, dst[r], COUNT * 4, NULL);
    for (int r = 0; r < N; r++) ucc_tl_nvl_zc_post(&team[r], &zc[r], 0, NULL);
    for (int r = 0; r < N; r++) {
        int direct = 0;
        CHECK(ucc_tl_nvl_zc_ready(&team[r], &zc[r], 1, NULL, NULL, &direct) == UCC_OK);
        CHECK(direct && zc[r].cache == NVL_ZC_DIRECT);
        CHECK(zc[r].d.src[1 - r] == (const char *)src[1 - r]);   /* the emulated mapping of an allocation is the allocation */
    }
    CHECK(launch_direct(zc, src, dst) == 0);
    for (int i = 0; i < COUNT; i++) CHECK(dst[0][i] == (float)(2 * (i % 97) + 10) && dst[1][i] == dst[0][i]);
    /* more distinct peer allocations than the cache holds, each mapped for one launch */
    for (int k = 0; k < FILLERS; k++) {
        for (int r = 0; r < N; r++) {
            nvl_xb_buf_t b;
            float *peer = dev_floats(256);
            ucc_tl_nvl_xb_export(&team[1 - r], peer, 256 * sizeof(float), &b);
            CHECK(b.kind == NVL_XB_IPC);
            CHECK(ucc_tl_nvl_xb_import(&team[r], (ucc_rank_t)(1 - r), &b) == (char *)peer);
        }
    }
    /* the persistent request posts again: its cached tables must still be mapped */
    for (int r = 0; r < N; r++) for (int i = 0; i < COUNT; i++) { src[r][i] = (float)(i % 13 + 3 * r); dst[r][i] = -1.f; }
    CHECK(launch_direct(zc, src, dst) == 0);
    for (int i = 0; i < COUNT; i++) CHECK(dst[0][i] == (float)(2 * (i % 13) + 3) && dst[1][i] == dst[0][i]);
    /* the cache evicted the idle fillers instead of growing without bound */
    CHECK(emu_ipc_count(1) > 0 && emu_ipc_count(2) <= 2 * NVL_IPC_CACHE_MAX);
    printf("IPC_CACHE_OK opens %ld closes %ld open now %ld\n", emu_ipc_count(0), emu_ipc_count(1), emu_ipc_count(2));
    return 0;
}
'''


def test_persistent_tables_survive_a_full_ipc_cache(emu_build, tmp_path):  # noqa: F811
    src = tmp_path / "ipc_cache.c"
    src.write_text(SRC)
    exe = tmp_path / "ipc_cache"
    emu = os.path.join(ROOT, "build-emu", "lib")
    core = os.path.join(ROOT, "ucc_b200", "lib")
    cc = subprocess.run(["gcc", "-O1", "-g", "-std=gnu11", "-D_GNU_SOURCE", f"-I{ROOT}/src", f"-I{ROOT}/include", "-I/usr/local/cuda/include", str(src), "-o", str(exe),
                         os.path.join(emu, "ucc", "libucc_tl_nvl.so"), f"-L{emu}", "-lcudart_emu", f"-L{core}", "-lucc",
                         f"-Wl,-rpath,{emu}:{emu}/ucc:{core}", "-Wl,--allow-shlib-undefined", "-lpthread"], capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-4000:]
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "IPC_CACHE_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
    assert "closed IPC mapping" not in out.stderr, out.stderr[-2000:]
