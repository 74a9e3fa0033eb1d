/* Candidate device-copy kernels for tools/selfcopy_study.py: the team-of-one copy of tl/nvl, parameterised so that one
 * process can time every variant side by side.  Not part of the library; the script builds it with
 *     nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -shared -Xcompiler -fPIC
 *
 * tma_copy:    one-warp CTAs, thread 0 drives a ring of STAGES shared-memory stages with cp.async.bulk (global -> shared
 *              completing on an mbarrier, shared -> global tracked by bulk groups), loads AHEAD chunks ahead of the stores.
 *              Runtime: stage size, grid (CTAs per SM = grid / SMs), chunk ownership (round-robin or one contiguous span
 *              per CTA).  HINT bit 0 / bit 1: an L2 evict_first cache policy on the loads / the stores.
 * thread_copy: every warp copies tiles of 32 x U 16-byte vectors (each load / store instruction of the warp covers 512
 *              contiguous bytes), tiles grid-strided over the warps.  LD 0: ld.global.nc.L1::no_allocate, 1: the same
 *              with .L2::256B.  ST 0: st.global, 1: st.global.cs, 2: st.global with an L2 evict_first cache policy.
 * Sizes must be multiples of 16 and pointers 16-byte aligned (the study only times such copies). */
#include <cuda_runtime.h>
#include <stdint.h>

static __device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
static __device__ __forceinline__ uint64_t evict_first_policy()
{ uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }

template <int STAGES, int AHEAD, int HINT>
__global__ void __launch_bounds__(32) tma_copy(char *dst, const char *src, size_t n, uint32_t stage_bytes, int contig)
{
    static_assert(AHEAD > 0 && AHEAD < STAGES, "a load may only reuse a stage whose store has been issued");
    extern __shared__ __align__(128) char smem[];
    if (threadIdx.x != 0) return;
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem + (size_t)STAGES * stage_bytes);
    for (int s = 0; s < STAGES; s++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bar[s])) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    const uint64_t pol = HINT ? evict_first_policy() : 0;
    const size_t nchunks = (n + stage_bytes - 1) / stage_bytes, cta = blockIdx.x, nctas = gridDim.x;
    size_t first, stride, mine;
    if (contig) { first = cta * nchunks / nctas; mine = (cta + 1) * nchunks / nctas - first; stride = 1; }
    else { first = cta; mine = cta < nchunks ? (nchunks - cta + nctas - 1) / nctas : 0; stride = nctas; }
    for (size_t i = 0; i < mine + AHEAD; i++) {
        if (i < mine) {
            const size_t o = (first + i * stride) * stage_bytes;
            const uint32_t nb = (uint32_t)(n - o < stage_bytes ? n - o : stage_bytes), s = (uint32_t)(i % STAGES);
            asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(STAGES - AHEAD - 1) : "memory");
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar[s])), "r"(nb) : "memory");
            if (HINT & 1)
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                             ::"r"(smem_u32(smem + (size_t)s * stage_bytes)), "l"(src + o), "r"(nb), "r"(smem_u32(&bar[s])), "l"(pol) : "memory");
            else
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(smem_u32(smem + (size_t)s * stage_bytes)), "l"(src + o), "r"(nb), "r"(smem_u32(&bar[s])) : "memory");
        }
        if (i >= AHEAD) {
            const size_t k = i - AHEAD, o = (first + k * stride) * stage_bytes;
            const uint32_t nb = (uint32_t)(n - o < stage_bytes ? n - o : stage_bytes), s = (uint32_t)(k % STAGES), par = (uint32_t)(k / STAGES) & 1;
            asm volatile("{\n .reg .pred p;\n W_%=:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n @!p bra W_%=;\n}"
                         ::"r"(smem_u32(&bar[s])), "r"(par) : "memory");
            if (HINT & 2)
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;"
                             ::"l"(dst + o), "r"(smem_u32(smem + (size_t)s * stage_bytes)), "r"(nb), "l"(pol) : "memory");
            else
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst + o), "r"(smem_u32(smem + (size_t)s * stage_bytes)), "r"(nb) : "memory");
        }
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");   /* one group per iteration, empty or not */
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

template <int LD> static __device__ __forceinline__ uint4 ld_v4(const uint4 *p)
{
    uint4 v;
    if (LD == 1) asm volatile("ld.global.nc.L1::no_allocate.L2::256B.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    else asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
template <int ST> static __device__ __forceinline__ void st_v4(uint4 *p, uint4 v, uint64_t pol)
{
    if (ST == 1) asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
    else if (ST == 2) asm volatile("st.global.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "l"(pol) : "memory");
    else asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

template <int U, int LD, int ST>
__global__ void __launch_bounds__(1024) thread_copy(uint4 *dst, const uint4 *src, size_t n)
{
    const uint64_t pol = ST == 2 ? evict_first_policy() : 0;
    const size_t nv = n / 16, lane = threadIdx.x & 31, tile = 32 * U;
    const size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / 32, nw = (size_t)gridDim.x * blockDim.x / 32;
    const size_t full = nv / tile;
    for (size_t t = w; t < full; t += nw) {
        const size_t b = t * tile + lane;
        uint4 x[U];
#pragma unroll
        for (int u = 0; u < U; u++) x[u] = ld_v4<LD>(src + b + u * 32);
#pragma unroll
        for (int u = 0; u < U; u++) st_v4<ST>(dst + b + u * 32, x[u], pol);
    }
    for (size_t v = full * tile + (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += (size_t)gridDim.x * blockDim.x) st_v4<ST>(dst + v, ld_v4<LD>(src + v), pol);
}

/* non-persistent: block b copies the b-th run of blockDim x U vectors (warp tiles of 32 x U inside it), so the blocks in flight
 * cover one narrow window that moves through memory in launch order */
template <int U, int LD, int ST>
__global__ void __launch_bounds__(1024) thread_copy_flat(uint4 *dst, const uint4 *src, size_t n)
{
    const uint64_t pol = ST == 2 ? evict_first_policy() : 0;
    const size_t nv = n / 16, b = ((size_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u)) * U + (threadIdx.x & 31);
    if (b + 32 * (U - 1) < nv) {
        uint4 x[U];
#pragma unroll
        for (int u = 0; u < U; u++) x[u] = ld_v4<LD>(src + b + u * 32);
#pragma unroll
        for (int u = 0; u < U; u++) st_v4<ST>(dst + b + u * 32, x[u], pol);
    } else {
        for (int u = 0; u < U; u++) if (b + u * 32 < nv) st_v4<ST>(dst + b + u * 32, ld_v4<LD>(src + b + u * 32), pol);
    }
}

/* (STAGES, AHEAD) pairs the study may ask for, each with the four HINT values */
#define TMA_RINGS(X) X(12, 6) X(12, 9) X(8, 4) X(8, 6) X(8, 2) X(6, 3) X(6, 4) X(4, 2) X(4, 3) X(3, 2) X(2, 1)
#define TMA_CASE(S, A)                                                                                                      \
    if (stages == S && ahead == A) {                                                                                        \
        void (*k)(char *, const char *, size_t, uint32_t, int) = hint == 0 ? tma_copy<S, A, 0> : hint == 1 ? tma_copy<S, A, 1> \
                                                                : hint == 2 ? tma_copy<S, A, 2> : tma_copy<S, A, 3>;        \
        const size_t smem = (size_t)S * stage_bytes + 128;                                                                  \
        cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);                    \
        if (e != cudaSuccess) return e;                                                                                     \
        k<<<nctas, 32, smem, s>>>(static_cast<char *>(dst), static_cast<const char *>(src), n, stage_bytes, contig);        \
        return cudaGetLastError();                                                                                          \
    }

extern "C" int study_tma(void *dst, const void *src, size_t n, int stages, int ahead, int hint, int contig, unsigned stage_bytes, int nctas, cudaStream_t s)
{
    if (hint < 0 || hint > 3) return cudaErrorInvalidValue;
    TMA_RINGS(TMA_CASE)
    return cudaErrorInvalidValue;
}

#define THR_CASE(U_, L_, S_) \
    if (u == U_ && ld == L_ && st == S_) { thread_copy<U_, L_, S_><<<nblocks, nthreads, 0, s>>>(static_cast<uint4 *>(dst), static_cast<const uint4 *>(src), n); return cudaGetLastError(); }
#define THR_ST(U_, L_) THR_CASE(U_, L_, 0) THR_CASE(U_, L_, 1) THR_CASE(U_, L_, 2)
extern "C" int study_thread(void *dst, const void *src, size_t n, int u, int ld, int st, int nblocks, int nthreads, cudaStream_t s)
{
    THR_ST(4, 0) THR_ST(4, 1) THR_ST(8, 0) THR_ST(8, 1)
    return cudaErrorInvalidValue;
}

#define FLAT_CASE(U_, L_, S_) \
    if (u == U_ && ld == L_ && st == S_) { thread_copy_flat<U_, L_, S_><<<(unsigned)((n / 16 + (size_t)nthreads * U_ - 1) / ((size_t)nthreads * U_)), nthreads, 0, s>>>(static_cast<uint4 *>(dst), static_cast<const uint4 *>(src), n); return cudaGetLastError(); }
#define FLAT_U(U_) FLAT_CASE(U_, 0, 0) FLAT_CASE(U_, 1, 1) FLAT_CASE(U_, 0, 1)
extern "C" int study_thread_flat(void *dst, const void *src, size_t n, int u, int ld, int st, int nthreads, cudaStream_t s)
{
    FLAT_U(1) FLAT_U(2) FLAT_U(4) FLAT_U(8)
    return cudaErrorInvalidValue;
}

extern "C" int study_memcpy(void *dst, const void *src, size_t n, cudaStream_t s)
{ return cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToDevice, s); }

extern "C" int study_max_blocks_per_sm(int u, int ld, int st, int nthreads)
{
    int nb = -1;
#define THR_OCC(U_, L_, S_) if (u == U_ && ld == L_ && st == S_) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, thread_copy<U_, L_, S_>, nthreads, 0);
    THR_OCC(4, 0, 0) THR_OCC(4, 0, 1) THR_OCC(4, 0, 2) THR_OCC(4, 1, 0) THR_OCC(4, 1, 1) THR_OCC(4, 1, 2)
    THR_OCC(8, 0, 0) THR_OCC(8, 0, 1) THR_OCC(8, 0, 2) THR_OCC(8, 1, 0) THR_OCC(8, 1, 1) THR_OCC(8, 1, 2)
    return nb;
}
