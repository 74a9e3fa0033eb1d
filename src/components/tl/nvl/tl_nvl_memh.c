/* tl/nvl memory registration: ucc_mem_map() support (reference: tl/ucp/tl_ucp_context.c:506-577 registers with UCX and packs
 * an rkey; here a handle describes a CUDA allocation that peers map over NVLink).
 *
 *   EXPORT  segment {address, len} of device memory -> {cudaIpcMemHandle of the allocation, offset, owner pid / host}; inside
 *           one process (the gtest-style harness) the raw pointer is enough
 *   pack    the record travels inside the core's relocatable handle (core/ucc_mem_map.c)
 *   IMPORT  open the allocation (cached per context by allocation base + handle bytes) -> a pointer valid here
 *
 * A collective whose arguments carry GLOBAL handles (UCC_COLL_ARGS_FLAG_{SRC,DST}_MEMH_GLOBAL: one imported handle per member)
 * gets its zero-copy pointer tables from them at init time (tl_nvl_direct.c: ucc_tl_nvl_zc_init): no per-post handle export, no exchange
 * board round trip, no deferred launch - the registration is paid once.  Convention (same as the reference's one-sided
 * algorithms): a member's buffer sits at the same offset inside its registered segment on every member. */
#include "tl_nvl.h"
#include "utils/ucc_proc_info.h"
#include <unistd.h>

#define NVL_MEMH_MAGIC 0x4e564c4d454d4831ull /* "NVLMEMH1" */

ucc_status_t ucc_tl_nvl_mem_map(const ucc_base_context_t *b_ctx, ucc_mem_map_mode_t mode, void *memh, void *tl_h_p)
{
    ucc_tl_nvl_context_t *ctx = ucc_derived_of(b_ctx, ucc_tl_nvl_context_t);
    nvl_memh_t *h;
    if (mode == UCC_MEM_MAP_MODE_EXPORT) {
        const ucc_mem_map_t *seg = (const ucc_mem_map_t *)memh;
        struct cudaPointerAttributes attr;
        void *base = NULL; size_t alen = 0;
        if (!seg || !seg->address || !seg->len) return UCC_ERR_INVALID_PARAM;
        if (cudaPointerGetAttributes(&attr, seg->address) != cudaSuccess || attr.type != cudaMemoryTypeDevice) { (void)cudaGetLastError(); return UCC_ERR_NOT_SUPPORTED; }
        h = (nvl_memh_t *)calloc(1, sizeof(*h));
        if (!h) return UCC_ERR_NO_MEMORY;
        h->magic = NVL_MEMH_MAGIC; h->host_hash = ucc_local_proc.host_hash; h->pid = (int32_t)getpid(); h->dev = ctx->dev; h->len = seg->len;
        h->addr = (uint64_t)(uintptr_t)seg->address;
        if (ucc_cuda_get_address_range(seg->address, &base, &alen) == UCC_OK && cudaIpcGetMemHandle(&h->ipc, base) == cudaSuccess) {
            h->has_ipc = 1; h->base = (uint64_t)(uintptr_t)base; h->off = (uint64_t)((char *)seg->address - (char *)base);
        } else (void)cudaGetLastError(); /* VMM / pool memory: usable inside the owning process only */
        h->mapped = (char *)seg->address;
        *(void **)tl_h_p = h;
        return UCC_OK;
    }
    if (mode == UCC_MEM_MAP_MODE_IMPORT) {
        nvl_memh_t in;
        memcpy(&in, memh, sizeof(in));
        if (in.magic != NVL_MEMH_MAGIC) return UCC_ERR_INVALID_PARAM;
        h = (nvl_memh_t *)calloc(1, sizeof(*h));
        if (!h) return UCC_ERR_NO_MEMORY;
        *h = in; h->imported = 1; h->opened = NULL; h->mapped = NULL;
        if (in.host_hash == ucc_local_proc.host_hash && in.pid == (int32_t)getpid()) h->mapped = (char *)(uintptr_t)in.addr;
        else if (in.host_hash == ucc_local_proc.host_hash && in.has_ipc) {
            void *m = NULL;
            if (cudaIpcOpenMemHandle(&m, in.ipc, cudaIpcMemLazyEnablePeerAccess) == cudaSuccess) { h->opened = m; h->mapped = (char *)m + in.off; }
            else { tl_debug(b_ctx->lib, "mem_map import: cudaIpcOpenMemHandle failed: %s", cudaGetErrorString(cudaGetLastError())); }
        }
        *(void **)tl_h_p = h; /* mapped == NULL: this member cannot reach the segment; collectives then take the staged kernels */
        return UCC_OK;
    }
    return UCC_ERR_NOT_SUPPORTED;
}

ucc_status_t ucc_tl_nvl_mem_unmap(const ucc_base_context_t *b_ctx, ucc_mem_map_mode_t mode, void *tl_h)
{
    nvl_memh_t *h = (nvl_memh_t *)tl_h;
    (void)b_ctx; (void)mode;
    if (!h || h->magic != NVL_MEMH_MAGIC) return UCC_ERR_INVALID_PARAM;
    if (h->opened && cudaIpcCloseMemHandle(h->opened) != cudaSuccess) (void)cudaGetLastError();
    h->magic = 0;
    free(h);
    return UCC_OK;
}

ucc_status_t ucc_tl_nvl_memh_pack(const ucc_base_context_t *b_ctx, ucc_mem_map_mode_t mode, void *tl_h, void **pack_buffer)
{
    nvl_memh_t *h = (nvl_memh_t *)tl_h, *out;
    char *buf;
    (void)b_ctx; (void)mode;
    if (!h || h->magic != NVL_MEMH_MAGIC) return UCC_ERR_INVALID_PARAM;
    buf = (char *)calloc(1, sizeof(size_t) + sizeof(nvl_memh_t)); /* {size_t len; bytes} as the core expects */
    if (!buf) return UCC_ERR_NO_MEMORY;
    *(size_t *)buf = sizeof(nvl_memh_t);
    out = (nvl_memh_t *)(buf + sizeof(size_t));
    *out = *h; out->mapped = NULL; out->opened = NULL; out->imported = 0;
    *pack_buffer = buf;
    return UCC_OK;
}
