/* tl/nvl zero-copy support: per-collective exchange of the members' USER buffers.
 *
 * The staged kernels copy src into the symmetric heap and the result out of it: two extra passes over HBM for
 * every byte.  For large messages each rank instead publishes (CUDA IPC handle of the allocation, offset) of its
 * src / dst in a small POSIX shm board it owns; every peer maps the allocation once (cached by allocation base,
 * validated by handle bytes) and the kernel then reads / writes the user buffers in place over NVLink.
 * Inside one process (the gtest-style harness) the board simply carries raw pointers.
 *
 * Compared with the reference (tl/cuda alltoallv_ce.c:70-126, tl_cuda_cache.c:62-353): same idea (IPC handle
 * exchange through a shared segment + an open-handle cache) but the segment is single-writer per rank, lock free
 * (sequence numbers), there is no shm barrier, and a rank whose buffer cannot be exported simply says so, which
 * makes all ranks fall back to the staged kernel for that collective - the decision is symmetric by construction. */
#include "tl_nvl.h"
#include "utils/ucc_sys.h"
#include "utils/ucc_atomic.h"
#include <stdio.h>
#include <unistd.h>

#define NVL_LIB(_t) ((_t)->super.super.context->lib)

ucc_status_t ucc_tl_nvl_xb_create(ucc_tl_nvl_team_t *team)
{
    static uint32_t counter = 0;
    void *addr = NULL;
    ucc_status_t st;
    uint32_t my = ucc_atomic_fadd32(&counter, 1);
    if (my == 0) ucc_shm_reap_stale("ucc_b200_nvlxb.");
    snprintf(team->xb_name, sizeof(team->xb_name), "/ucc_b200_nvlxb.%d.%u", (int)getpid(), my);
    st = ucc_shm_create(team->xb_name, sizeof(nvl_xb_seg_t), &addr);
    if (st != UCC_OK) { team->xb_name[0] = 0; return st; }
    memset(addr, 0, sizeof(nvl_xb_seg_t));
    team->xb_mine = (nvl_xb_seg_t *)addr;
    team->xb_named = 1;
    return UCC_OK;
}

ucc_status_t ucc_tl_nvl_xb_attach(ucc_tl_nvl_team_t *team)
{
    ucc_rank_t N = UCC_TL_TEAM_SIZE(team), me = UCC_TL_TEAM_RANK(team);
    for (ucc_rank_t p = 0; p < N; p++) {
        void *addr = NULL;
        if (p == me) { team->xb[p] = team->xb_mine; continue; }
        if (!team->infos[p].xb_name[0] || ucc_shm_attach(team->infos[p].xb_name, sizeof(nvl_xb_seg_t), &addr) != UCC_OK) return UCC_ERR_NO_RESOURCE;
        team->xb[p] = (nvl_xb_seg_t *)addr;
    }
    return UCC_OK;
}

void ucc_tl_nvl_xb_unlink(ucc_tl_nvl_team_t *team)
{ if (team->xb_named) { ucc_shm_unlink(team->xb_name); team->xb_named = 0; } }

static void entry_close(nvl_ipc_entry_t *x)
{
    if (cudaIpcCloseMemHandle(x->mapped) != cudaSuccess) (void)cudaGetLastError();
    if (x->last_use) cudaEventDestroy(x->last_use);
    free(x);
}

/* no table refers to the mapping and the last launch that used it has completed (a query: never a device synchronize, which
 * would also invalidate a global-mode stream capture running on another thread) */
static int entry_idle(const nvl_ipc_entry_t *x)
{
    cudaError_t e;
    if (x->refs) return 0;
    if (!x->last_use) return 1;
    e = cudaEventQuery(x->last_use);
    if (e == cudaSuccess) return 1;
    (void)cudaGetLastError();
    return 0;
}

void ucc_tl_nvl_xb_release(ucc_tl_nvl_team_t *team)
{
    ucc_rank_t N = UCC_TL_TEAM_SIZE(team), me = UCC_TL_TEAM_RANK(team);
    for (ucc_rank_t p = 0; p < N && p < NVL_MAX_PEERS; p++) {
        nvl_ipc_cache_t *c = &team->ipc_cache[p];
        for (unsigned i = 0; i < c->n; i++) entry_close(c->e[i]);
        free(c->e); c->e = NULL; c->n = c->cap = 0;
        if (p != me && team->xb[p]) ucc_shm_detach(team->xb[p], sizeof(nvl_xb_seg_t));
        team->xb[p] = NULL;
    }
    ucc_tl_nvl_xb_unlink(team);
    if (team->xb_mine) { ucc_shm_detach(team->xb_mine, sizeof(nvl_xb_seg_t)); team->xb_mine = NULL; }
}

int ucc_tl_nvl_is_managed(const void *ptr)
{
    struct cudaPointerAttributes attr;
    if (!ptr) return 0;
    if (cudaPointerGetAttributes(&attr, ptr) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
    return attr.type == cudaMemoryTypeManaged;
}

/* A managed buffer (cudaMallocManaged) is never published as mappable, whatever the sharing mode: a peer GPU that loads or stores
 * its pages migrates them or takes a remote fault on every access, so every member stages the collective instead.  Across processes
 * cudaIpcGetMemHandle refuses such memory anyway; inside one process the board would carry the raw pointer. */
static void export_buf(ucc_tl_nvl_team_t *team, const void *ptr, size_t len, nvl_xb_buf_t *b)
{
    memset(b, 0, sizeof(*b));
    if (!ptr || !len) { b->kind = NVL_XB_EMPTY; return; }
    b->len = len;
    if (ucc_tl_nvl_is_managed(ptr)) { b->kind = NVL_XB_NONE; return; }
    if (team->heap_kind == NVL_HEAP_LOCAL) { b->kind = NVL_XB_RAW; b->base = (uint64_t)(uintptr_t)ptr; return; }
    {
        void *base = NULL; size_t alen = 0;
        if (ucc_cuda_get_address_range(ptr, &base, &alen) != UCC_OK) { b->kind = NVL_XB_NONE; return; }
        if (cudaIpcGetMemHandle(&b->handle, base) != cudaSuccess) { (void)cudaGetLastError(); b->kind = NVL_XB_NONE; return; } /* VMM / pool / managed memory */
        b->kind = NVL_XB_IPC; b->base = (uint64_t)(uintptr_t)base; b->alloc_len = alen; b->off = (uint64_t)((const char *)ptr - (const char *)base);
    }
}

void ucc_tl_nvl_xb_export(ucc_tl_nvl_team_t *team, const void *ptr, size_t len, nvl_xb_buf_t *b) { export_buf(team, ptr, len, b); }

/* returns 0 when the slot is still in use by a slow peer (caller retries later) */
static int xb_publish(ucc_tl_nvl_team_t *team, const nvl_zc_t *zc, int usable, const size_t *aux)
{
    ucc_rank_t N = UCC_TL_TEAM_SIZE(team), me = UCC_TL_TEAM_RANK(team);
    nvl_xb_entry_t *e = &team->xb_mine->e[zc->seq % NVL_XB_SLOTS];
    if (zc->seq >= NVL_XB_SLOTS)
        for (ucc_rank_t p = 0; p < N; p++) if (p != me && ucc_load_acquire(&team->xb[p]->consumed) + NVL_XB_SLOTS <= zc->seq) return 0;
    if (usable && !(zc->flags & NVL_ZC_WITHDRAW)) { export_buf(team, zc->src, zc->src_len, &e->src); export_buf(team, zc->dst, zc->dst_len, &e->dst); }
    else { memset(&e->src, 0, sizeof(e->src)); memset(&e->dst, 0, sizeof(e->dst)); e->src.kind = e->dst.kind = NVL_XB_NONE; }
    for (ucc_rank_t p = 0; p < N && p < NVL_MAX_PEERS; p++) e->aux[p] = aux ? (uint64_t)aux[p] : 0;
    ucc_store_release(&e->seq, zc->seq + 1);
    return 1;
}

/* my address of the peer buffer `b`; an IPC mapping comes back referenced in *ent (NULL: nothing to release).  A full cache
 * never closes a referenced or busy mapping: it grows instead.  Mapping happens after the members' symmetric decision to go
 * zero-copy, so running out of room here cannot fall back to staging. */
static char *import_buf(ucc_tl_nvl_team_t *team, ucc_rank_t p, const nvl_xb_buf_t *b, nvl_ipc_entry_t **ent)
{
    nvl_ipc_cache_t *c = &team->ipc_cache[p];
    nvl_ipc_entry_t *x;
    void *mapped = NULL;
    unsigned i;
    *ent = NULL;
    if (b->kind == NVL_XB_RAW) return (char *)(uintptr_t)b->base;
    if (b->kind != NVL_XB_IPC) return NULL;
    for (i = 0; i < c->n; i++) {
        x = c->e[i];
        if (x->stale || x->base != b->base) continue;
        if (!memcmp(&x->handle, &b->handle, sizeof(b->handle))) { x->refs++; *ent = x; return (char *)x->mapped + b->off; }
        /* same address, different allocation: the peer freed and re-allocated; a mapping still in use is closed once idle */
        if (entry_idle(x)) { entry_close(x); c->e[i] = c->e[--c->n]; }
        else x->stale = 1;
        break;
    }
    if (c->n == c->cap) {
        for (i = 0; i < c->n;) {
            if (entry_idle(c->e[i])) { entry_close(c->e[i]); c->e[i] = c->e[--c->n]; }
            else i++;
        }
    }
    if (c->n == c->cap) {
        unsigned cap = c->cap ? 2 * c->cap : NVL_IPC_CACHE_MAX;
        nvl_ipc_entry_t **e = (nvl_ipc_entry_t **)realloc(c->e, cap * sizeof(*e));
        if (!e) return NULL;
        if (c->cap) tl_debug(NVL_LIB(team), "IPC cache of rank %u: %u mappings in use, growing to %u", p, c->n, cap);
        c->e = e; c->cap = cap;
    }
    x = (nvl_ipc_entry_t *)calloc(1, sizeof(*x));
    if (!x) return NULL;
    if (cudaIpcOpenMemHandle(&mapped, b->handle, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
        tl_debug(NVL_LIB(team), "cudaIpcOpenMemHandle of a buffer of rank %u failed: %s", p, cudaGetErrorString(cudaGetLastError()));
        free(x);
        return NULL;
    }
    x->base = b->base; x->len = b->alloc_len; x->handle = b->handle; x->mapped = mapped; x->refs = 1;
    c->e[c->n++] = x;
    *ent = x;
    return (char *)mapped + b->off;
}

/* a mapping for one launch that follows right away: the caller reports that launch with ucc_tl_nvl_ipc_used() before it maps
 * anything else */
char *ucc_tl_nvl_xb_import(ucc_tl_nvl_team_t *team, ucc_rank_t p, const nvl_xb_buf_t *b)
{
    nvl_ipc_entry_t *x;
    char *r = import_buf(team, p, b, &x);
    if (x) x->refs--;
    return r;
}

static void entry_used(nvl_ipc_entry_t *x, cudaStream_t s)
{
    if (!x->last_use && cudaEventCreateWithFlags(&x->last_use, cudaEventDisableTiming) != cudaSuccess) { (void)cudaGetLastError(); x->last_use = NULL; x->refs++; return; } /* untracked: never idle */
    if (cudaEventRecord(x->last_use, s) != cudaSuccess) { (void)cudaGetLastError(); x->refs++; }
}

/* the kernel just launched on s reads or writes `ptr`, which ucc_tl_nvl_xb_import() mapped from rank p */
void ucc_tl_nvl_ipc_used(ucc_tl_nvl_team_t *team, ucc_rank_t p, const void *ptr, cudaStream_t s)
{
    nvl_ipc_cache_t *c = &team->ipc_cache[p];
    for (unsigned i = 0; i < c->n; i++) {
        nvl_ipc_entry_t *x = c->e[i];
        if ((const char *)ptr >= (const char *)x->mapped && (const char *)ptr < (const char *)x->mapped + x->len) { entry_used(x, s); return; }
    }
}

static void zc_unpin(nvl_zc_t *zc)
{
    for (unsigned i = 0; i < zc->npin; i++) zc->pin[i]->refs--;
    zc->npin = 0;
}

/* the direct form of the current post was launched on s (not captured: a captured post only runs tables that a persistent
 * request cached, and they stay referenced until it is finalized).  Tables resolved for this post only are released. */
void ucc_tl_nvl_zc_launched(nvl_zc_t *zc, cudaStream_t s)
{
    for (unsigned i = 0; i < zc->npin; i++) entry_used(zc->pin[i], s);
    if (zc->cache != NVL_ZC_DIRECT) zc_unpin(zc);
}

/* at finalize: the request's tables are no longer used by any future launch */
void ucc_tl_nvl_zc_release(nvl_zc_t *zc) { zc_unpin(zc); }

/* Registered buffers: when the collective carries GLOBAL memory handles (one imported ucc_mem_map handle per member) for every
 * side the zero-copy kernel touches, the pointer tables are built at init from the registrations - the per-post exchange is
 * never used for this request.  Every member evaluates the same handles, flags and sizes, so the outcome is the same everywhere;
 * a member that cannot reach some segment could break that symmetry, so reachability of ALL segments is required on import
 * (unreachable -> h->mapped == NULL -> no table, and since the exporter could not produce an IPC handle either, nobody has one). */
static int memh_tables(ucc_tl_nvl_team_t *team, const ucc_coll_args_t *a, nvl_zc_t *zc)
{
    const ucc_base_context_t *bctx = team->super.super.context;
    ucc_rank_t N = UCC_TL_TEAM_SIZE(team), me = UCC_TL_TEAM_RANK(team);
    int need_src = zc->flags & NVL_ZC_SRC, need_dst = zc->flags & NVL_ZC_DST;
    int use_src = need_src && (a->mask & UCC_COLL_ARGS_FIELD_MEM_MAP_SRC_MEMH) && (a->flags & UCC_COLL_ARGS_FLAG_SRC_MEMH_GLOBAL) && a->src_memh.global_memh;
    int use_dst = need_dst && (a->mask & UCC_COLL_ARGS_FIELD_MEM_MAP_DST_MEMH) && (a->flags & UCC_COLL_ARGS_FLAG_DST_MEMH_GLOBAL) && a->dst_memh.global_memh;
    if ((need_src && !use_src) || (need_dst && !use_dst)) return 0;
    memset(&zc->d, 0, sizeof(zc->d));
    for (int side = 0; side < 2; side++) {
        ucc_mem_map_mem_h *gl = side ? a->dst_memh.global_memh : a->src_memh.global_memh;
        const char *mine = side ? (const char *)zc->dst : (const char *)zc->src;
        nvl_memh_t *hm;
        size_t off;
        if (side ? !use_dst : !use_src) continue;
        hm = (nvl_memh_t *)ucc_mem_map_tl_handle(gl[me], bctx);
        if (!hm || !hm->mapped || mine < hm->mapped || mine >= hm->mapped + hm->len) return 0; /* my buffer is not inside my registered segment */
        off = (size_t)(mine - hm->mapped);
        if ((uintptr_t)mine & 15) return 0;
        for (ucc_rank_t p = 0; p < N; p++) {
            nvl_memh_t *h = (nvl_memh_t *)ucc_mem_map_tl_handle(gl[p], bctx);
            if (!h || !h->mapped || off >= h->len || ((uintptr_t)(h->mapped + off) & 15)) return 0;
            if (side) zc->d.dst[p] = p == me ? (char *)zc->dst : h->mapped + off; else zc->d.src[p] = p == me ? (const char *)zc->src : h->mapped + off;
        }
    }
    return 1;
}

/* at init: the plan of a task whose path has a direct form.  `flags`: NVL_ZC_*; src / dst: my buffers as the peers see them;
 * `reg`: the arguments whose registrations may give the tables (NULL: never) */
void ucc_tl_nvl_zc_init(ucc_tl_nvl_team_t *team, nvl_zc_t *zc, unsigned flags, const void *src, size_t src_len, void *dst, size_t dst_len, const ucc_coll_args_t *reg)
{
    zc->flags = flags; zc->src = src; zc->src_len = src_len; zc->dst = dst; zc->dst_len = dst_len; zc->npin = 0;
    zc->cache = reg && memh_tables(team, reg, zc) ? NVL_ZC_DIRECT : NVL_ZC_RESOLVE;
    if (zc->cache == NVL_ZC_RESOLVE && !team->zcopy) zc->flags = 0; /* no board and nothing cached: always staged */
}

/* at post, in post order (the same on every member): a post without a cached decision takes the next board entry and publishes
 * my buffers (aux: what every member reads back at my index).  A capturing stream cannot wait for the peers, so it tells them
 * "not usable" and everybody stages this one; cached tables need no waiting and are also fine inside a capture. */
void ucc_tl_nvl_zc_post(ucc_tl_nvl_team_t *team, nvl_zc_t *zc, int captured, const size_t *aux)
{
    zc->pending = zc->cache == NVL_ZC_RESOLVE;
    if (!zc->pending) return;
    zc->seq = team->xb_seq++;
    zc->published = xb_publish(team, zc, !captured, aux);
    if (captured) { zc->pending = 0; if (team->xb_mine->consumed < zc->seq + 1) ucc_store_release(&team->xb_mine->consumed, zc->seq + 1); }
}

/* *direct: whether this post runs the direct form, with the tables in zc->d.  UCC_INPROGRESS: not every member has published
 * yet (call again).  aux_for_me: what every member published at my index. */
ucc_status_t ucc_tl_nvl_zc_ready(ucc_tl_nvl_team_t *team, nvl_zc_t *zc, int persistent, const size_t *aux, size_t *aux_for_me, int *direct)
{
    ucc_rank_t N = UCC_TL_TEAM_SIZE(team), me = UCC_TL_TEAM_RANK(team);
    int need_src = zc->flags & NVL_ZC_SRC, need_dst = zc->flags & NVL_ZC_DST, need_align = zc->flags & NVL_ZC_ALIGN, ok = 1;
    nvl_direct_t *d = &zc->d;
    if (!zc->pending) { *direct = zc->cache == NVL_ZC_DIRECT; return UCC_OK; }
    if (!zc->published) zc->published = xb_publish(team, zc, 1, aux);
    if (!zc->published) return UCC_INPROGRESS;
    for (ucc_rank_t p = 0; p < N; p++) if (p != me && ucc_load_acquire(&team->xb[p]->e[zc->seq % NVL_XB_SLOTS].seq) != zc->seq + 1) return UCC_INPROGRESS;
    /* all members published: decide (identically on every rank) whether the buffers can be used in place and map them */
    memset(d, 0, sizeof(*d));
    if (aux_for_me) for (ucc_rank_t p = 0; p < N; p++) aux_for_me[p] = (size_t)team->xb[p]->e[zc->seq % NVL_XB_SLOTS].aux[me];
    for (ucc_rank_t p = 0; p < N && ok; p++) {
        const nvl_xb_entry_t *e = &team->xb[p]->e[zc->seq % NVL_XB_SLOTS];
        if (need_src && e->src.kind != NVL_XB_EMPTY && e->src.kind != NVL_XB_RAW && e->src.kind != NVL_XB_IPC) ok = 0;
        if (need_dst && e->dst.kind != NVL_XB_EMPTY && e->dst.kind != NVL_XB_RAW && e->dst.kind != NVL_XB_IPC) ok = 0;
        /* 16-byte alignment keeps every transaction a full vector; anything else takes the staged kernel */
        if (need_align && need_src && e->src.kind != NVL_XB_EMPTY && ((e->src.base + e->src.off) & 15)) ok = 0;
        if (need_align && need_dst && e->dst.kind != NVL_XB_EMPTY && ((e->dst.base + e->dst.off) & 15)) ok = 0;
    }
    /* up to here every member took the same decision (it only depends on what all of them published).  Mapping a peer's
     * allocation can still fail on THIS rank only; the peers will launch the in-place kernel, so falling back to the staged
     * one here would mix two protocols and corrupt data silently: fail the collective. */
    zc_unpin(zc);
    for (ucc_rank_t p = 0; p < N && ok > 0; p++) {
        const nvl_xb_entry_t *e = &team->xb[p]->e[zc->seq % NVL_XB_SLOTS];
        nvl_ipc_entry_t *x;
        if (p == me) { d->src[p] = (const char *)zc->src; d->dst[p] = (char *)zc->dst; continue; }
        if (need_src && e->src.kind != NVL_XB_EMPTY) { d->src[p] = import_buf(team, p, &e->src, &x); if (x) zc->pin[zc->npin++] = x; if (!d->src[p]) ok = -1; }
        if (need_dst && e->dst.kind != NVL_XB_EMPTY) { d->dst[p] = import_buf(team, p, &e->dst, &x); if (x) zc->pin[zc->npin++] = x; if (!d->dst[p]) ok = -1; }
    }
    if (ok < 0) zc_unpin(zc);
    if (team->xb_mine->consumed < zc->seq + 1) ucc_store_release(&team->xb_mine->consumed, zc->seq + 1);
    tl_debug(NVL_LIB(team), "exchange %lu: %s (src %d dst %d)", (unsigned long)zc->seq, ok > 0 ? "zero-copy" : (ok ? "MAPPING FAILED" : "staged"),
             !!need_src, !!need_dst);
    if (ok < 0) {
        tl_error(NVL_LIB(team), "cannot map a peer's buffer for the zero-copy kernel (the peers will run it): failing the collective; "
                 "UCC_TL_NVL_ZCOPY=n avoids the zero-copy path");
        return UCC_ERR_NO_RESOURCE;
    }
    zc->pending = 0;
    /* persistent request: the buffers are fixed for the lifetime of the request, so every later post of it (same decision on
     * every member - they all re-post the same request) launches straight away with these tables: no handle export, no board
     * round trip, no deferred launch.  Its mappings stay referenced until the request is finalized (ucc_tl_nvl_zc_release). */
    if (persistent) zc->cache = ok ? NVL_ZC_DIRECT : NVL_ZC_STAGED;
    *direct = ok;
    return UCC_OK;
}
