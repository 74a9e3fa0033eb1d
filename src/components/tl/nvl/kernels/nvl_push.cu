/* Zero-copy PUSH exchange for allgather(v) / alltoall(v) (algorithm "push", opt-in): the members' DESTINATION buffers are mapped
 * through the buffer-exchange board (tl_nvl_direct.c) and every rank stores its blocks straight into them.
 *
 *     barrier (per block: peer kernels are running => their dst may be written)
 *     for every peer p: my block for p  --st-->  p's dst          (fire-and-forget NVLink writes; own block: local copy)
 *     signal + wait for ALL blocks of ALL peers (their stores into my dst have landed)
 *
 * The pull kernels (nvl_exchange_kernel) issue loads over NVLink: each 16-byte vector costs a request and a response crossing
 * the switch, and a thread stalls a full round trip (~2 us) before it can retire the dependent store.  Stores need no response:
 * in the 1-64 MB range, where a thread owns only a few vectors per block, that is what NCCL's copy-based allgather / alltoall
 * exploit, and where the pull variants pay the round trip for every vector.  The host emulation (tests/emu) checks the logic. */
#include "nvl_reduce_impl.cuh"
#include "nvl_bulk.cuh"

/* grid-strided copy local memory -> (possibly peer) memory, any alignment */
static __device__ __forceinline__ void push_bytes_grid(char *dst, const char *src, size_t n)
{
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nt = (size_t)gridDim.x * blockDim.x;
    const uintptr_t mis = ((uintptr_t)dst | (uintptr_t)src);
    if ((mis & 15) == 0) {
        const size_t nv = n / 16;
        size_t v = tid;
        for (; v + 7 * nt < nv; v += 8 * nt) {
            uint4 x[8];
#pragma unroll
            for (int u = 0; u < 8; u++) x[u] = ld_src_v4(src + (v + u * nt) * 16);
#pragma unroll
            for (int u = 0; u < 8; u++) st_v4(dst + (v + u * nt) * 16, x[u]);
        }
        for (; v < nv; v += nt) st_v4(dst + v * 16, ld_src_v4(src + v * 16));
        for (size_t i = nv * 16 + tid; i < n; i += nt) dst[i] = src[i];
    } else if ((mis & 3) == 0) {
        const size_t nw = n / 4;
        for (size_t v = tid; v < nw; v += nt) ((uint32_t *)dst)[v] = ((const uint32_t *)src)[v];
        for (size_t i = nw * 4 + tid; i < n; i += nt) dst[i] = src[i];
    } else {
        for (size_t i = tid; i < n; i += nt) dst[i] = src[i];
    }
}

__global__ void __launch_bounds__(NVL_THREADS_MAX, 2) nvl_exchange_push_kernel(nvl_push_args_t a)
{
    const nvl_team_dev_t &t = a.team;
    const int N = t.size, me = t.rank;
    BlockSync bs; bs.init(t);
    const char *src = static_cast<const char *>(a.src);
    /* alltoallv: publish where every source's block lands in my dst.  Every block keeps its own copy of the table (block b of
     * a peer reads copy b), so the per-block barrier below orders exactly the accesses that touch it */
    const size_t tbl = (size_t)blockIdx.x * NVL_MAX_PEERS * sizeof(uint64_t);
    if (a.lookup && (int)threadIdx.x < N) reinterpret_cast<volatile uint64_t *>(data_of(t, me) + tbl)[threadIdx.x] = (uint64_t)a.recv_off[threadIdx.x];
    bs.barrier(t, 1);
    for (int i = 1; i < N; i++) {   /* start at my right neighbour so the N senders do not converge on one receiver */
        int p = me + i; if (p >= N) p -= N;
        if (!a.send_bytes[p]) continue;
        const size_t land = a.lookup ? (size_t) * reinterpret_cast<volatile const uint64_t *>(data_of(t, p) + tbl + (size_t)me * 8) : a.land_off[p];
        push_bytes_grid(a.dst_of[p] + land, src + a.send_off[p], a.send_bytes[p]);
    }
    if (a.send_bytes[me] && a.dst_of[me] + a.land_off[me] != src + a.send_off[me]) push_bytes_grid(a.dst_of[me] + a.land_off[me], src + a.send_off[me], a.send_bytes[me]);
    bs.signal(t, 2);
    bs.wait_all_blocks(t, 2);
    bs.finish(2);
}

#ifndef NVL_HOST_EMU
/* The same exchange with the TMA engine as the data mover (nvl_bulk.cuh): one-warp CTAs, thread 0 of each drives a ring of
 * shared-memory stages - bulk load of a chunk of my block from local HBM, bulk store of it into the member's destination over
 * NVLink.  A block whose addresses are not 16-byte aligned (only known on the device for alltoallv, where the receiver
 * publishes the landing offset) is copied by the warp's threads instead; the barrier protocol is identical either way. */
static __device__ __forceinline__ void push_job(BulkPipe &pp, char *dst, const char *src, size_t n, int rot)
{
    const bool aligned = ((((uintptr_t)dst | (uintptr_t)src) & 15) == 0) && (n & 15) == 0;   /* uniform across the CTA */
    if (aligned) { if (threadIdx.x == 0) bulk_copy_range(pp, dst, src, n, blockIdx.x, gridDim.x, rot); }
    else push_bytes_grid(dst, src, n);
}
__global__ void __launch_bounds__(32) nvl_exchange_push_bulk_kernel(const __grid_constant__ nvl_push_args_t a)
{
    extern __shared__ __align__(128) char bulk_smem[];
    const nvl_team_dev_t &t = a.team;
    const int N = t.size, me = t.rank;
    BlockSync bs; bs.init(t);
    BulkPipe pp;
    const char *src = static_cast<const char *>(a.src);
    const size_t tbl = (size_t)blockIdx.x * NVL_MAX_PEERS * sizeof(uint64_t);
    if (threadIdx.x == 0) pp.init(bulk_smem);
    if (a.lookup && (int)threadIdx.x < N) reinterpret_cast<volatile uint64_t *>(data_of(t, me) + tbl)[threadIdx.x] = (uint64_t)a.recv_off[threadIdx.x];
    bs.barrier(t, 1);
    for (int i = 1; i < N; i++) {
        int p = me + i; if (p >= N) p -= N;
        if (!a.send_bytes[p]) continue;
        const size_t land = a.lookup ? (size_t) * reinterpret_cast<volatile const uint64_t *>(data_of(t, p) + tbl + (size_t)me * 8) : a.land_off[p];
        push_job(pp, a.dst_of[p] + land, src + a.send_off[p], a.send_bytes[p], i);
    }
    if (a.send_bytes[me] && a.dst_of[me] + a.land_off[me] != src + a.send_off[me]) push_job(pp, a.dst_of[me] + a.land_off[me], src + a.send_off[me], a.send_bytes[me], 0);
    if (threadIdx.x == 0) { bulk_wait_all(); fence_proxy_async(); fence_sys(); }   /* my bulk stores have landed before anybody sees the flag */
    bs.signal(t, 2);
    bs.wait_all_blocks(t, 2);
    bs.finish(2);
}
extern "C" cudaError_t nvl_launch_exchange_push_bulk(const nvl_push_args_t *a, int nblocks, cudaStream_t s)
{
    static int attr_set = 0;
    if (!attr_set) { cudaError_t e = cudaFuncSetAttribute(nvl_exchange_push_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, NVL_BULK_SMEM); if (e != cudaSuccess) return e; attr_set = 1; }
    nvl_exchange_push_bulk_kernel<<<nblocks, 32, NVL_BULK_SMEM, s>>>(*a);
    return cudaGetLastError();
}
#endif

#ifndef NVL_HOST_EMU /* the host emulation calls the kernel directly */
extern "C" cudaError_t nvl_launch_exchange_push(const nvl_push_args_t *a, int nblocks, int nthreads, cudaStream_t s)
{
    if (nthreads > NVL_THREADS_MAX) nthreads = NVL_THREADS_MAX;
    nvl_exchange_push_kernel<<<nblocks, nthreads, 0, s>>>(*a);
    return cudaGetLastError();
}
#endif
