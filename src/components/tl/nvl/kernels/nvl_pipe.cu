/* Entry point of the pipelined staged NVLS allreduce (kernel: nvl_pipe.cuh); the host-emulated plugin compiles it too. */
#include "nvl_reduce_impl.cuh"

#if !defined(NVL_HOST_EMU) || defined(NVL_EMU_LAUNCHERS)
extern "C" cudaError_t nvl_launch_reduce_pipe(const nvl_red_args_t *a, int nblocks, int nthreads, cudaStream_t s)
{
    if (nthreads > NVL_THREADS_MAX) nthreads = NVL_THREADS_MAX;
    if (nthreads < 128 || (nthreads & 127)) return cudaErrorInvalidValue; /* three roles need at least four warps */
    if (a->kind != NVL_RED_ALLREDUCE || !a->use_nvls || !a->team.mc_heap) return cudaErrorInvalidValue;
    return nvl_red_launch(NVL_FAM_PIPE, a, nblocks, nthreads, s);
}
#endif
