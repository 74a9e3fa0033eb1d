/* Entry point of the one-shot reduce_scatter(v) (kernel: nvl_oneshot_rs.cuh); the host-emulated plugin compiles it too. */
#include "nvl_reduce_impl.cuh"

#if !defined(NVL_HOST_EMU) || defined(NVL_EMU_LAUNCHERS)
extern "C" cudaError_t nvl_launch_reduce_scatter_oneshot(const nvl_red_args_t *a, int nblocks, int nthreads, cudaStream_t s)
{
    if (a->kind != NVL_RED_REDUCE_SCATTER) return cudaErrorInvalidValue;
    return nvl_red_launch(NVL_FAM_ONESHOT_RS, a, nblocks, nthreads, s);
}
#endif
