// Launchers of the tl/nvl kernels for the host-emulated build of the plugin: same C interface as kernels/nvl_kernels.h, but a
// launch enqueues a closure on the emulated stream (cudart_emu.cpp) that runs the grid with one OS thread per CUDA thread.  The
// reduction entry points, their datatype predicates and the kernel selection are the kernel sources' own (NVL_EMU_LAUNCHERS).
// A kernel whose pointer tables reach into a CUDA IPC mapping that was closed (cudart_emu.cpp, emu_range_dead) is not run and its
// launch fails, as the kernel would fault on a GPU.
#define NVL_EMU_LAUNCHERS 1
#include "nvl_emu_prelude.h"
#include <initializer_list>

extern "C" void emu_stream_enqueue(cudaStream_t s, std::function<void()> *f);
extern "C" int emu_range_dead(const void *p, size_t n);

template <typename F> static cudaError_t enqueue_grid(cudaStream_t s, int nb, int nt, F body)
{
    if (nb < 1 || nt < 1) return cudaErrorInvalidValue;
    std::function<void()> f = [nb, nt, body]() {
        std::vector<pthread_barrier_t> bars((size_t)nb);
        for (auto &b : bars) pthread_barrier_init(&b, nullptr, (unsigned)nt);
        std::vector<std::thread> th;
        th.reserve((size_t)nb * nt);
        for (int b = 0; b < nb; b++) for (int t = 0; t < nt; t++)
            th.emplace_back([=, &bars]() {
                threadIdx = {(unsigned)t, 0, 0}; blockIdx = {(unsigned)b, 0, 0}; blockDim = {(unsigned)nt, 1, 1}; gridDim = {(unsigned)nb, 1, 1};
                emu_cta_barrier = &bars[(size_t)b];
                body();
            });
        for (auto &x : th) x.join();
        for (auto &b : bars) pthread_barrier_destroy(&b);
    };
    emu_stream_enqueue(s, &f);
    return cudaSuccess;
}

static bool tables_dead(const char *what, std::initializer_list<const void *> ptrs)
{
    for (const void *p : ptrs) if (p && emu_range_dead(p, 1)) { fprintf(stderr, "EMU: %s kernel table references a closed IPC mapping (%p)\n", what, p); return true; }
    return false;
}
template <typename P> static bool peers_dead(const char *what, const P *tab, int n, int skip)
{
    for (int i = 0; i < n; i++) if (i != skip && tables_dead(what, {(const void *)tab[i]})) return true;
    return false;
}

static cudaError_t nvl_red_run(nvl_red_kernel_t k, const nvl_red_args_t &a, int nb, int nt, cudaStream_t s)
{
    /* the direct form's tables are rotated: entry 0 is mine */
    if (a.direct && (peers_dead("reduction", a.d.src, a.team.size, 0) || peers_dead("reduction", a.d.dst, a.team.size, 0))) return cudaErrorIllegalAddress;
    return enqueue_grid(s, nb, nt, [k, a]() { k(a); });
}

/* a representative subset of the datatypes (eight, plus INT128 / UINT128) keeps the build of this test-only plugin short; the others
 * are not supported */
const nvl_dt_row *const nvl_rows[NVL_DT_LAST] = {nullptr, nullptr, &nvl_row_of<int32_t>, &nvl_row_of<int64_t>, &nvl_row_of<uint8_t>, nullptr, nullptr,
    nullptr, nullptr, &nvl_row_of<float>, &nvl_row_of<double>, &nvl_row_of<__nv_bfloat16>, &nvl_row_of<nvl_c64>, &nvl_row_of<nvl_c128>, nullptr,
    &nvl_row_of<nvl_i128>, &nvl_row_of<nvl_u128>};
static_assert(NVL_DT_F128 == 14 && NVL_DT_U128 + 1 == NVL_DT_LAST, "the table above lists every datatype of nvl_kernels.h");

extern "C" {
cudaError_t nvl_launch_allgather_symm(const nvl_xchg_args_t *, int, int, cudaStream_t) { return cudaErrorInvalidValue; }
cudaError_t nvl_launch_exchange(const nvl_xchg_args_t *ap, int nb, int nt, cudaStream_t s)
{
    nvl_xchg_args_t a = *ap;
    if (a.direct && peers_dead("exchange", a.d.src, a.team.size, a.team.rank)) return cudaErrorIllegalAddress;
    return enqueue_grid(s, nb, nt, [a]() { nvl_exchange_kernel(a); });
}
cudaError_t nvl_launch_exchange_push(const nvl_push_args_t *ap, int nb, int nt, cudaStream_t s)
{
    nvl_push_args_t a = *ap;
    if (peers_dead("push", a.dst_of, a.team.size, a.team.rank)) return cudaErrorIllegalAddress;
    return enqueue_grid(s, nb, nt, [a]() { nvl_exchange_push_kernel(a); });
}
int nvl_p2p_lanes(size_t bytes) { size_t n = (bytes + NVL_P2P_LANE_BYTES - 1) / NVL_P2P_LANE_BYTES; return n < 1 ? 1 : (n > NVL_P2P_MAX_CTAS ? NVL_P2P_MAX_CTAS : (int)n); }
int nvl_p2p_push_ctas(size_t bytes) { size_t n = bytes / (64 * 1024); return n < 1 ? 1 : (n > 4 ? 4 : (int)n); }
cudaError_t nvl_launch_p2p(const nvl_p2p_args_t *ap, int nt, cudaStream_t s)
{
    nvl_p2p_args_t a = *ap;
    if (a.mode == NVL_P2P_PUSH && tables_dead("p2p push", {a.remote})) return cudaErrorIllegalAddress;
    if (a.mode == NVL_P2P_PUSH) return enqueue_grid(s, nvl_p2p_push_ctas(a.bytes), nt > 64 ? 64 : nt, [a]() { nvl_p2p_push_kernel(a); });
    if (a.mode == NVL_P2P_WAIT) return enqueue_grid(s, 1, 32, [a]() { nvl_p2p_wait_kernel(a); });
    return enqueue_grid(s, nvl_p2p_lanes(a.bytes), nt > 64 ? 64 : nt, [a]() { nvl_p2p_kernel(a); });
}
cudaError_t nvl_launch_exchange_push_bulk(const nvl_push_args_t *ap, int nb, cudaStream_t s) { return nvl_launch_exchange_push(ap, nb, 32, s); }   /* no TMA here: the thread-copy kernel */
cudaError_t nvl_launch_exchange_swap(const nvl_swap_args_t *ap, int nb, int nt, cudaStream_t s)
{
    nvl_swap_args_t a = *ap;
    if (peers_dead("swap", a.dst_of, a.team.size, a.team.rank)) return cudaErrorIllegalAddress;
    return enqueue_grid(s, nb, nt, [a]() { nvl_exchange_swap_kernel(a); });
}
cudaError_t nvl_launch_barrier(const nvl_team_dev_t *tp, cudaStream_t s) { nvl_team_dev_t t = *tp; return enqueue_grid(s, 1, 32, [t]() { nvl_barrier_kernel(t); }); }
cudaError_t nvl_launch_self_copy(void *dst, const void *src, size_t bytes, int, int, cudaStream_t s)
{ return enqueue_grid(s, 1, 1, [=]() { memmove(dst, src, bytes); }); }
cudaError_t nvl_launch_ctrl_init(void *heap_base, cudaStream_t s) { return enqueue_grid(s, 1, 1, [=]() { memset(heap_base, 0, sizeof(nvl_ctrl_t)); }); }
}
