// Launchers of the host-emulated tl/nvl plugin with the in-place alltoall(v) swap kernel (kernels/nvl_swap.cu) added to those of
// nvl_emu_launch.cpp.
#include "nvl_emu_launch.cpp"
#include "nvl_swap.cu"

extern "C" cudaError_t nvl_launch_exchange_swap(const nvl_swap_args_t *ap, int nb, int nt, cudaStream_t s)
{
    nvl_swap_args_t a = *ap;
    return enqueue_grid(s, nb, nt, [a]() { nvl_exchange_swap_kernel(a); });
}
