// The emulated launchers of nvl_emu_launch.cpp for the graph tests (tests/emu/build_hostemu_graph.sh): a kernel whose pointer
// tables reach into a CUDA IPC mapping that was closed (cudart_emu_graph.cpp, emu_range_dead) is not run and its launch fails, as
// the kernel would fault on a GPU.  The prelude is included first, so the kernel sources call the checking launchers below, and
// nvl_emu_launch.cpp's launchers are compiled under other names.
#define NVL_EMU_LAUNCHERS 1
#include "nvl_emu_prelude.h"
#include <initializer_list>

#define nvl_red_run nvl_red_run_unchecked
#define nvl_launch_exchange nvl_launch_exchange_unchecked
#define nvl_launch_exchange_push nvl_launch_exchange_push_unchecked
#define nvl_launch_exchange_push_bulk nvl_launch_exchange_push_bulk_unchecked
#define nvl_launch_exchange_swap nvl_launch_exchange_swap_unchecked
#define nvl_launch_p2p nvl_launch_p2p_unchecked
#include "nvl_emu_launch.cpp"
#undef nvl_red_run
#undef nvl_launch_exchange
#undef nvl_launch_exchange_push
#undef nvl_launch_exchange_push_bulk
#undef nvl_launch_exchange_swap
#undef nvl_launch_p2p

extern "C" int emu_range_dead(const void *p, size_t n);

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
    return nvl_red_run_unchecked(k, a, nb, nt, s);
}

extern "C" {
cudaError_t nvl_launch_exchange(const nvl_xchg_args_t *a, int nb, int nt, cudaStream_t s)
{
    if (a->direct && peers_dead("exchange", a->d.src, a->team.size, a->team.rank)) return cudaErrorIllegalAddress;
    return nvl_launch_exchange_unchecked(a, nb, nt, s);
}
cudaError_t nvl_launch_exchange_push(const nvl_push_args_t *a, int nb, int nt, cudaStream_t s)
{
    if (peers_dead("push", a->dst_of, a->team.size, a->team.rank)) return cudaErrorIllegalAddress;
    return nvl_launch_exchange_push_unchecked(a, nb, nt, s);
}
cudaError_t nvl_launch_exchange_push_bulk(const nvl_push_args_t *a, int nb, cudaStream_t s)
{
    if (peers_dead("push", a->dst_of, a->team.size, a->team.rank)) return cudaErrorIllegalAddress;
    return nvl_launch_exchange_push_bulk_unchecked(a, nb, s);
}
cudaError_t nvl_launch_exchange_swap(const nvl_swap_args_t *a, int nb, int nt, cudaStream_t s)
{
    if (peers_dead("swap", a->dst_of, a->team.size, a->team.rank)) return cudaErrorIllegalAddress;
    return nvl_launch_exchange_swap_unchecked(a, nb, nt, s);
}
cudaError_t nvl_launch_p2p(const nvl_p2p_args_t *a, int nt, cudaStream_t s)
{
    if (a->mode == NVL_P2P_PUSH && tables_dead("p2p push", {a->remote})) return cudaErrorIllegalAddress;
    return nvl_launch_p2p_unchecked(a, nt, s);
}
}
