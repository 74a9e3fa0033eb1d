// Launchers of the host-emulated tl/nvl plugin with the complex datatypes added: the launchers of nvl_emu_launch.cpp (which builds a
// representative subset of the real datatypes) under other names, and in front of them the entry points of kernels/nvl_kernels.h
// that route complex float / double to the emulated kernels and everything else to those launchers.
#define nvl_dt_size nvl_emu_base_dt_size
#define nvl_dt_supports_op nvl_emu_base_dt_supports_op
#define nvl_launch_allreduce_oneshot nvl_emu_base_launch_allreduce_oneshot
#define nvl_launch_reduce_staged nvl_emu_base_launch_reduce_staged
#define nvl_launch_reduce_direct nvl_emu_base_launch_reduce_direct
#define nvl_launch_reduce_steps nvl_emu_base_launch_reduce_steps
#define nvl_launch_reduce_scatter_oneshot nvl_emu_base_launch_reduce_scatter_oneshot
#include "nvl_emu_launch.cpp"
#undef nvl_dt_size
#undef nvl_dt_supports_op
#undef nvl_launch_allreduce_oneshot
#undef nvl_launch_reduce_staged
#undef nvl_launch_reduce_direct
#undef nvl_launch_reduce_steps
#undef nvl_launch_reduce_scatter_oneshot

static bool is_complex(int dt) { return dt == NVL_DT_C64 || dt == NVL_DT_C128; }

#define BY_COMPLEX_DT(_ap, _K, _base)                                                                    \
    {                                                                                                    \
        nvl_red_args_t a = *(_ap);                                                                       \
        if (a.dt == NVL_DT_C64) return enqueue_grid(s, nb, nt, [a]() { _K<nvl_c64>(a); });              \
        if (a.dt == NVL_DT_C128) return enqueue_grid(s, nb, nt, [a]() { _K<nvl_c128>(a); });            \
        return _base(_ap, nb, nt, s);                                                                    \
    }

extern "C" {
size_t nvl_dt_size(int dt) { return dt == NVL_DT_C64 ? 8 : (dt == NVL_DT_C128 ? 16 : nvl_emu_base_dt_size(dt)); }
int nvl_dt_supports_op(int dt, int op)
{
    if (is_complex(dt)) return op == NVL_OP_SUM || op == NVL_OP_PROD || op == NVL_OP_AVG;
    return nvl_emu_base_dt_supports_op(dt, op);
}
cudaError_t nvl_launch_allreduce_oneshot(const nvl_red_args_t *ap, int nb, int nt, cudaStream_t s)
BY_COMPLEX_DT(ap, nvl_allreduce_oneshot_kernel, nvl_emu_base_launch_allreduce_oneshot)
cudaError_t nvl_launch_reduce_staged(const nvl_red_args_t *ap, int nb, int nt, cudaStream_t s)
BY_COMPLEX_DT(ap, nvl_reduce_staged_kernel, nvl_emu_base_launch_reduce_staged)
cudaError_t nvl_launch_reduce_direct(const nvl_red_args_t *ap, int nb, int nt, cudaStream_t s)
BY_COMPLEX_DT(ap, direct_any, nvl_emu_base_launch_reduce_direct)
cudaError_t nvl_launch_reduce_steps(const nvl_red_args_t *ap, int nb, int nt, cudaStream_t s)
BY_COMPLEX_DT(ap, nvl_reduce_steps_kernel, nvl_emu_base_launch_reduce_steps)
cudaError_t nvl_launch_reduce_scatter_oneshot(const nvl_red_args_t *ap, int nb, int nt, cudaStream_t s)
BY_COMPLEX_DT(ap, nvl_reduce_scatter_oneshot_kernel, nvl_emu_base_launch_reduce_scatter_oneshot)
}
