/* Symmetric user memory (UCC_TL_NVL_USER_SIZE > 0): the entry point of the in-place NVLS reduction (kernel: nvl_symm.cuh), which
 * the host-emulated plugin compiles too, and the allgather into a symmetric destination. */
#include "nvl_reduce_impl.cuh"

#if !defined(NVL_HOST_EMU) || defined(NVL_EMU_LAUNCHERS)
extern "C" cudaError_t nvl_launch_reduce_symm(const nvl_red_args_t *a, int nblocks, int nthreads, cudaStream_t s)
{
    if ((a->kind != NVL_RED_ALLREDUCE && a->kind != NVL_RED_REDUCE_SCATTER) || !a->team.mc_heap || !a->d.src[0]) return cudaErrorInvalidValue;
    if (a->kind == NVL_RED_ALLREDUCE && !a->d.dst[0]) return cudaErrorInvalidValue;
    return nvl_red_launch(NVL_FAM_SYMM, a, nblocks, nthreads, s);
}
#endif

/* ------------------------------------------------------------------ */
/* allgather INTO a symmetric destination: every member multicasts its */
/* block to the same offset of everybody's dst with multimem.st - no   */
/* staging, no pull, no copy-out; the block is read once from local    */
/* memory and crosses each link once.                                  */
/*   a.src / a.src_bytes = my block (any local memory, 16-byte aligned)*/
/*   a.dst = LOCAL address of the gathered buffer inside my heap       */
/*   a.push_off = byte offset of my block inside it (multiple of 16)   */
/* ------------------------------------------------------------------ */
__global__ void __launch_bounds__(NVL_THREADS_MAX, 2) nvl_allgather_symm_kernel(const __grid_constant__ nvl_xchg_args_t a)
{
    const nvl_team_dev_t &t = a.team;
    const int N = t.size, me = t.rank;
    BlockSync bs; bs.init(t);
    const size_t dof = (size_t)(static_cast<char *>(a.dst) - t.heap[me]) + a.push_off;
    const char *src = static_cast<const char *>(a.src);
    char *mc = t.mc_heap + dof;
    const size_t nfull = a.src_bytes / 16, per = (nfull + gridDim.x - 1) / gridDim.x;
    const size_t j0 = dmin((size_t)blockIdx.x * per, nfull), j1 = dmin(j0 + per, nfull), nt = blockDim.x;
    constexpr int U = 8;

    bs.barrier(t, 1);                       /* every member's kernel runs: its dst may be written */
    size_t j = j0 + threadIdx.x;
    for (; j + (size_t)(U - 1) * nt < j1; j += (size_t)U * nt) {
        uint4 x[U];
#pragma unroll
        for (int u = 0; u < U; u++) x[u] = ld_src_v4(src + (j + (size_t)u * nt) * 16);
#pragma unroll
        for (int u = 0; u < U; u++) mc_st_v4(mc + (j + (size_t)u * nt) * 16, x[u]);
    }
    for (; j < j1; j += nt) mc_st_v4(mc + j * 16, ld_src_v4(src + j * 16));
    /* trailing bytes (block size not a multiple of 16): plain byte stores to every member's unicast mapping */
    if (blockIdx.x == 0 && threadIdx.x < (a.src_bytes & 15))
        for (int p = 0; p < N; p++) t.heap[p][dof + nfull * 16 + threadIdx.x] = src[nfull * 16 + threadIdx.x];
    bs.barrier(t, 2);                       /* every block has landed everywhere */
    bs.finish(2);
}

#ifndef NVL_HOST_EMU /* the host emulation calls the kernels directly */
extern "C" cudaError_t nvl_launch_allgather_symm(const nvl_xchg_args_t *a, int nblocks, int nthreads, cudaStream_t s)
{
    if (nthreads > NVL_THREADS_MAX) nthreads = NVL_THREADS_MAX;
    if (!a->team.mc_heap || !a->dst || !a->src || (a->push_off & 15) || ((uintptr_t)a->src & 15) || ((uintptr_t)a->dst & 15)) return cudaErrorInvalidValue;
    nvl_allgather_symm_kernel<<<nblocks, nthreads, 0, s>>>(*a);
    return cudaGetLastError();
}
#endif
