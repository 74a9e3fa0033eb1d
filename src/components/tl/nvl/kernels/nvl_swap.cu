/* In-place alltoall(v) as pairwise swaps (algorithm "swap"): the members' buffers are mapped through the buffer-exchange board
 * (tl_nvl_direct.c), and my region for member p trades contents with p's region for me, straight between the two buffers.
 *
 *     publish (offset, length) of my region for every member   (alltoallv: only I know them)
 *     barrier (per block: peer kernels are running => their buffers may be read and written)
 *     for every peer p: my region for p  <--swap-->  p's region for me   (the lower rank moves the first half, the higher the rest)
 *     signal + wait for ALL blocks of ALL peers (their stores into my buffer have landed)
 *
 * Nothing is staged: each byte crosses NVLink once per direction, as in the out-of-place exchange, and no scratch copy of the
 * buffer exists anywhere.  Both sides of a pair derive the same split from the same two lengths, so every byte of the two
 * regions is loaded and stored by exactly one thread of one of the two GPUs.  The host emulation (tests/emu) checks the logic. */
#include "nvl_reduce_impl.cuh"

/* grid-strided swap of two n-byte ranges, any alignment; b is (possibly) peer memory */
static __device__ __forceinline__ void swap_bytes_grid(char *a, char *b, size_t n)
{
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nt = (size_t)gridDim.x * blockDim.x;
    const uintptr_t mis = ((uintptr_t)a | (uintptr_t)b);
    if ((mis & 15) == 0) {
        /* 2 KB chunks, one per group of 32 threads: lane l moves vectors l, l + 32, l + 64, l + 96 of the chunk, so each of the
         * 8 loads in flight (4 of mine, 4 of the peer's) is a coalesced 512-byte warp access at an immediate offset from one
         * base; eight separately computed addresses next to eight vectors would not fit the 64 registers of 2 x 512 threads */
        const size_t nv = n / 16, nchunk = nv / 128, groups = nt / 32, lane = tid % 32;
        for (size_t c = tid / 32; tid < groups * 32 && c < nchunk; c += groups) {   /* (a partial last group of the grid idles here) */
            char *pa = a + (c * 128 + lane) * 16, *pb = b + (c * 128 + lane) * 16;
            uint4 x[4], y[4];
#pragma unroll
            for (int u = 0; u < 4; u++) { x[u] = ld_peer_v4(pa + u * 512); y[u] = ld_peer_v4(pb + u * 512); }
#pragma unroll
            for (int u = 0; u < 4; u++) { st_v4(pa + u * 512, y[u]); st_v4(pb + u * 512, x[u]); }
        }
        for (size_t v = nchunk * 128 + tid; v < nv; v += nt) { const uint4 x = ld_peer_v4(a + v * 16), y = ld_peer_v4(b + v * 16); st_v4(a + v * 16, y); st_v4(b + v * 16, x); }
        for (size_t i = nv * 16 + tid; i < n; i += nt) { const char x = a[i], y = *(volatile const char *)(b + i); a[i] = y; b[i] = x; }
    } else if ((mis & 3) == 0) {
        const size_t nw = n / 4;
        uint32_t *aw = reinterpret_cast<uint32_t *>(a), *bw = reinterpret_cast<uint32_t *>(b);
        for (size_t v = tid; v < nw; v += nt) { const uint32_t x = aw[v], y = ((volatile const uint32_t *)bw)[v]; aw[v] = y; bw[v] = x; }
        for (size_t i = nw * 4 + tid; i < n; i += nt) { const char x = a[i], y = *(volatile const char *)(b + i); a[i] = y; b[i] = x; }
    } else {
        for (size_t i = tid; i < n; i += nt) { const char x = a[i], y = *(volatile const char *)(b + i); a[i] = y; b[i] = x; }
    }
}

__global__ void __launch_bounds__(NVL_THREADS_MAX, 2) nvl_exchange_swap_kernel(nvl_swap_args_t a)
{
    const nvl_team_dev_t &t = a.team;
    const int N = t.size, me = t.rank;
    BlockSync bs; bs.init(t);
    /* alltoallv: publish (offset, length) of my region for every member.  Every block keeps its own copy of the table (block b of
     * a peer reads copy b), so the per-block barrier below orders exactly the accesses that touch it */
    const size_t tbl = (size_t)blockIdx.x * NVL_SWAP_TABLE_BYTES;
    if (a.lookup && (int)threadIdx.x < N) {
        volatile uint64_t *e = reinterpret_cast<volatile uint64_t *>(data_of(t, me) + tbl) + 2 * threadIdx.x;
        e[0] = (uint64_t)a.off[threadIdx.x]; e[1] = (uint64_t)a.len[threadIdx.x];
    }
    bs.barrier(t, 1);
    for (int i = 1; i < N; i++) {   /* start at my right neighbour so the N swappers do not converge on one member */
        int p = me + i; if (p >= N) p -= N;
        size_t poff = a.off[me], plen = a.len[me];   /* alltoall: every member's region for me sits where mine for me does */
        if (a.lookup) { const volatile uint64_t *e = reinterpret_cast<const volatile uint64_t *>(data_of(t, p) + tbl) + 2 * me; poff = (size_t)e[0]; plen = (size_t)e[1]; }
        /* a mismatched alltoallv (a user error) swaps the common prefix only: nothing outside either region is written */
        const size_t L = a.len[p] < plen ? a.len[p] : plen, h = (L / 2) & ~(size_t)15;
        const size_t lo = me < p ? 0 : h, hi = me < p ? h : L;
        if (hi > lo) swap_bytes_grid(a.buf + a.off[p] + lo, a.dst_of[p] + poff + lo, hi - lo);
    }
    bs.signal(t, 2);
    bs.wait_all_blocks(t, 2);
    bs.finish(2);
}

#ifndef NVL_HOST_EMU /* the host emulation calls the kernel directly */
extern "C" cudaError_t nvl_launch_exchange_swap(const nvl_swap_args_t *a, int nblocks, int nthreads, cudaStream_t s)
{
    if (nthreads > NVL_THREADS_MAX) nthreads = NVL_THREADS_MAX;
    nvl_exchange_swap_kernel<<<nblocks, nthreads, 0, s>>>(*a);
    return cudaGetLastError();
}
#endif
