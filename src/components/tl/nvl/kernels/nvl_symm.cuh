/* In-place NVLS allreduce (and reduce_scatter(v) out of a symmetric source) on SYMMETRIC USER MEMORY (UCC_TL_NVL_USER_SIZE > 0).
 *
 * When src and dst live in the user region of the team heap (allocated through ucc_tl_nvl_symm_region(), same offsets on every
 * member - the NVSHMEM / ncclMemAlloc+register contract), they are already bound to the team's multicast object.  Nothing is
 * staged and nothing is copied out:
 *     barrier   (every member's kernel runs => its src is final, its dst may be written)
 *     my slice: multimem.ld_reduce of src through the switch -> multimem.st into every member's dst
 *     barrier   (every slice has landed)
 * Each GPU injects count/N (stores) + answers count*(N-1)/N (loads of the others) and receives the same: one vector's worth
 * of bytes per direction, the minimum an allreduce can move, and HBM is touched once for reading and once for writing.
 *
 * d.src[0] / d.dst[0] carry the LOCAL addresses of src / dst inside my heap mapping; the multicast address is the same offset
 * in team.mc_heap.  Requires 16-byte aligned offsets (the allocator hands out 256-byte aligned blocks).
 *
 * Part of nvl_reduce_impl.cuh, which includes it.
 */

template <typename T, int OP>
static __device__ __forceinline__ void symm_body(const nvl_red_args_t &a, BlockSync &bs, const SlicePlan &pl)
{
    constexpr int E = 16 / sizeof(T);
    constexpr int U = NVL_BW_U;
    const nvl_team_dev_t &t = a.team;
    const int N = t.size, me = t.rank;
    const bool rs = a.kind == NVL_RED_REDUCE_SCATTER;   /* reduce_scatter(v): only src is symmetric, my block goes to the local a.dst */
    const size_t so = (size_t)(a.d.src[0] - t.heap[me]), dof = rs ? 0 : (size_t)(a.d.dst[0] - t.heap[me]);
    const float inv_n = 1.0f / (float)N;
    const size_t nt = blockDim.x;

    bs.barrier(t, 1);
    if (rs) {
        const size_t cnt = slice_cnt(a, pl, me), nv = (cnt + E - 1) / E;
        const size_t per = (nv + gridDim.x - 1) / gridDim.x, j0 = dmin((size_t)blockIdx.x * per, nv), j1 = dmin(j0 + per, nv);
        const char *mcs = t.mc_heap + so + slice_off(a, pl, me) * sizeof(T);
        T *db = static_cast<T *>(a.dst);
        const bool dal = ((uintptr_t)db & 15) == 0;
        size_t j = j0 + threadIdx.x;
        for (; j + (size_t)(U - 1) * nt < j1; j += (size_t)U * nt) {
            uint4 r[U];
#pragma unroll
            for (int u = 0; u < U; u++) r[u] = McRed<T, OP>::ld(mcs + (j + (size_t)u * nt) * 16);
#pragma unroll
            for (int u = 0; u < U; u++) {
                uint4 v = r[u];
                if (OP == NVL_OP_AVG) { VecAcc<T, OP> acc; acc.set(v); v = acc.get(inv_n, N); }
                store_dst_vec<T>(db, (j + (size_t)u * nt) * E, cnt, dal, v);   /* bounds-checked: the ragged last vector is cut at cnt */
            }
        }
        for (; j < j1; j += nt) {
            uint4 v = McRed<T, OP>::ld(mcs + j * 16);
            if (OP == NVL_OP_AVG) { VecAcc<T, OP> acc; acc.set(v); v = acc.get(inv_n, N); }
            store_dst_vec<T>(db, j * E, cnt, dal, v);
        }
    } else {
        const size_t cnt = slice_cnt(a, pl, me), nfull = cnt / E, nv = (cnt + E - 1) / E;
        const size_t per = (nv + gridDim.x - 1) / gridDim.x, j0 = dmin((size_t)blockIdx.x * per, nv), j1 = dmin(j0 + per, nv);
        const size_t jfull = dmin(j1, nfull);                               /* whole vectors of my range */
        const char *mcs = t.mc_heap + so + slice_off(a, pl, me) * sizeof(T);
        char *mcd = t.mc_heap + dof + slice_off(a, pl, me) * sizeof(T);
        size_t j = j0 + threadIdx.x;
        for (; j + (size_t)(U - 1) * nt < jfull; j += (size_t)U * nt) {
            uint4 r[U];
#pragma unroll
            for (int u = 0; u < U; u++) r[u] = McRed<T, OP>::ld(mcs + (j + (size_t)u * nt) * 16);
#pragma unroll
            for (int u = 0; u < U; u++) {
                uint4 v = r[u];
                if (OP == NVL_OP_AVG) { VecAcc<T, OP> acc; acc.set(v); v = acc.get(inv_n, N); }
                mc_st_v4(mcd + (j + (size_t)u * nt) * 16, v);
            }
        }
        for (; j < jfull; j += nt) {
            uint4 v = McRed<T, OP>::ld(mcs + j * 16);
            if (OP == NVL_OP_AVG) { VecAcc<T, OP> acc; acc.set(v); v = acc.get(inv_n, N); }
            mc_st_v4(mcd + j * 16, v);
        }
        /* ragged end of the vector (only the last non-empty slice can have one): the 16-byte load stays inside the 256-byte
         * aligned allocation, but the store must not touch bytes behind dst's last element - write the valid elements to every
         * member's unicast mapping instead */
        if (nfull < nv && nfull >= j0 && nfull < j1 && threadIdx.x == 0) {
            uint4 v = McRed<T, OP>::ld(mcs + nfull * 16);
            if (OP == NVL_OP_AVG) { VecAcc<T, OP> acc; acc.set(v); v = acc.get(inv_n, N); }
            for (int p = 0; p < N; p++)
                store_dst_vec<T>(reinterpret_cast<T *>(t.heap[p] + dof) + slice_off(a, pl, me), nfull * E, cnt, false, v);
        }
    }
    bs.barrier(t, 2);
}

template <typename T, int OP> __global__ void __launch_bounds__(NVL_THREADS_MAX, 2) nvl_allreduce_symm_kernel_t(const __grid_constant__ nvl_red_args_t a)
{
    BlockSync bs; bs.init(a.team);
    SlicePlan pl; make_plan<T>(a, pl);
    symm_body<T, OP>(a, bs, pl);
    bs.finish(2);
}
