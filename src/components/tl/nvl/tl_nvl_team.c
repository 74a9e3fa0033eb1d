/* tl/nvl team creation: symmetric heap allocation, handle exchange over the team OOB,
 * peer mapping, optional NVLS multicast binding.  Every decision that could differ between
 * ranks is agreed through an OOB allgather so all members end up in the same mode. */
#include "tl_nvl.h"
#include "coll_patterns/ring.h"
#include "core/ucc_lib.h"
static inline int same_pid_pair_unknown(int topo_known) { return !topo_known; }
#include "core/ucc_service_coll.h"
#include "utils/ucc_sys.h"
#include "utils/ucc_math.h"
#include <pthread.h>
#include <unistd.h>

#define NVL_LIB(_t) ((_t)->super.super.context->lib)

/* ------------------------------------------------------------------ */
/* fd server: a helper thread hands my memory handles to peers         */
/* ------------------------------------------------------------------ */
typedef struct nvl_fd_server { int lsock[2]; int fd[2]; volatile int *stop; } nvl_fd_server_t;
static void *fd_server_main(void *arg)
{
    nvl_fd_server_t *s = (nvl_fd_server_t *)arg;
    while (!*s->stop) {
        int served = 0;
        for (int i = 0; i < 2; i++) if (s->lsock[i] >= 0 && s->fd[i] >= 0 && ucc_sys_fd_server_serve_once(s->lsock[i], s->fd[i]) > 0) served = 1;
        if (!served) usleep(200);
    }
    return NULL;
}
static nvl_fd_server_t *g_srv_of(ucc_tl_nvl_team_t *t) { return (nvl_fd_server_t *)t->srv_thread; }

typedef struct nvl_srv_state { nvl_fd_server_t srv; pthread_t th; int started; } nvl_srv_state_t;

static ucc_status_t fd_server_start(ucc_tl_nvl_team_t *team, const char *name0)
{
    nvl_srv_state_t *st = (nvl_srv_state_t *)calloc(1, sizeof(*st));
    if (!st) return UCC_ERR_NO_MEMORY;
    st->srv.lsock[0] = ucc_sys_fd_server_open(name0); st->srv.lsock[1] = -1;
    st->srv.fd[0] = team->heap_fd; st->srv.fd[1] = -1; st->srv.stop = &team->srv_stop;
    if (st->srv.lsock[0] < 0) { free(st); return UCC_ERR_NO_RESOURCE; }
    team->srv_stop = 0;
    if (pthread_create(&st->th, NULL, fd_server_main, &st->srv)) { close(st->srv.lsock[0]); free(st); return UCC_ERR_NO_RESOURCE; }
    st->started = 1;
    team->srv_thread = st;
    return UCC_OK;
}
static ucc_status_t fd_server_add(ucc_tl_nvl_team_t *team, const char *name1, int fd)
{
    nvl_srv_state_t *st = (nvl_srv_state_t *)team->srv_thread;
    int s;
    if (!st) return UCC_ERR_NO_RESOURCE;
    s = ucc_sys_fd_server_open(name1);
    if (s < 0) return UCC_ERR_NO_RESOURCE;
    st->srv.fd[1] = fd; ucc_memory_cpu_store_fence(); st->srv.lsock[1] = s;
    return UCC_OK;
}
static void fd_server_stop(ucc_tl_nvl_team_t *team)
{
    nvl_srv_state_t *st = (nvl_srv_state_t *)team->srv_thread;
    if (!st) return;
    team->srv_stop = 1;
    if (st->started) pthread_join(st->th, NULL);
    for (int i = 0; i < 2; i++) if (st->srv.lsock[i] >= 0) close(st->srv.lsock[i]);
    free(st); team->srv_thread = NULL;
    (void)g_srv_of;
}
static int fetch_fd(ucc_tl_nvl_team_t *team, int pid, int remote_fd, const char *sock)
{
    ucc_tl_nvl_context_t *ctx = NVL_CTX(team);
    int fd = -1;
    if (ctx->cfg.fd_via_pidfd != UCC_NO) fd = ucc_sys_pidfd_getfd(pid, remote_fd);
    if (fd < 0) fd = ucc_sys_fd_recv(sock, 20000);
    return fd;
}

/* ------------------------------------------------------------------ */
/* heap                                                                */
/* ------------------------------------------------------------------ */
static ucc_status_t vmm_prop(int dev, CUmemAllocationProp *prop)
{
    memset(prop, 0, sizeof(*prop));
    prop->type = CU_MEM_ALLOCATION_TYPE_PINNED; prop->location.type = CU_MEM_LOCATION_TYPE_DEVICE; prop->location.id = dev;
    prop->requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    return UCC_OK;
}
static ucc_status_t map_handle(CUmemGenericAllocationHandle h, size_t size, size_t gran, int dev, char **va_p)
{
    CUdeviceptr va = 0; CUmemAccessDesc ad;
    CU_CHECK(ucc_cu.cuMemAddressReserve(&va, size, gran, 0, 0));
    if (ucc_cu.cuMemMap(va, size, 0, h, 0) != CUDA_SUCCESS) { ucc_cu.cuMemAddressFree(va, size); return UCC_ERR_NO_RESOURCE; }
    memset(&ad, 0, sizeof(ad)); ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE; ad.location.id = dev; ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    if (ucc_cu.cuMemSetAccess(va, size, &ad, 1) != CUDA_SUCCESS) { ucc_cu.cuMemUnmap(va, size); ucc_cu.cuMemAddressFree(va, size); return UCC_ERR_NO_RESOURCE; }
    *va_p = (char *)(uintptr_t)va;
    return UCC_OK;
}
static void unmap_va(char *va, size_t size) { if (!va) return; ucc_cu.cuMemUnmap((CUdeviceptr)(uintptr_t)va, size); ucc_cu.cuMemAddressFree((CUdeviceptr)(uintptr_t)va, size); }

static ucc_status_t heap_alloc(ucc_tl_nvl_team_t *team, int want_mc)
{
    ucc_tl_nvl_context_t *ctx = NVL_CTX(team);
    size_t size, gran = 2u << 20;
    team->nlanes = ctx->cfg.slots;
    team->lane_stride = ucc_align_up(NVL_DATA_OFFSET + ctx->cfg.symmetric_size, (size_t)2 << 20);
    size = team->lane_stride * team->nlanes + ctx->cfg.user_size;   /* [lane 0][lane 1]...[user region] */
    if (team->heap_kind == NVL_HEAP_VMM) {
        CUmemAllocationProp prop; size_t g = 0;
        vmm_prop(ctx->dev, &prop);
        if (ucc_cu.cuMemGetAllocationGranularity(&g, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS && g > gran) gran = g;
        if (want_mc && ucc_cu.cuMulticastGetGranularity) {
            CUmulticastObjectProp mp; memset(&mp, 0, sizeof(mp));
            mp.numDevices = UCC_TL_TEAM_SIZE(team); mp.size = size; mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
            g = 0;
            if (ucc_cu.cuMulticastGetGranularity(&g, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS && g > gran) gran = g;
        }
        size = ucc_align_up(size, gran);
        if (ucc_cu.cuMemCreate(&team->mem_handle, size, &prop, 0) != CUDA_SUCCESS) return UCC_ERR_NO_MEMORY;
        if (map_handle(team->mem_handle, size, gran, ctx->dev, &team->heap) != UCC_OK) { ucc_cu.cuMemRelease(team->mem_handle); return UCC_ERR_NO_MEMORY; }
        if (ucc_cu.cuMemExportToShareableHandle(&team->heap_fd, team->mem_handle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0) != CUDA_SUCCESS) {
            unmap_va(team->heap, size); ucc_cu.cuMemRelease(team->mem_handle); return UCC_ERR_NO_RESOURCE;
        }
    } else {
        size = ucc_align_up(size, gran);
        CUDA_CHECK(cudaMalloc((void **)&team->heap, size));
    }
    team->heap_size = size; team->mc_size = size;
    for (unsigned l = 0; l < team->nlanes; l++) CUDA_CHECK(cudaMemset(team->heap + l * team->lane_stride, 0, NVL_DATA_OFFSET));
    CUDA_CHECK(cudaDeviceSynchronize());
    return UCC_OK;
}

static void team_release(ucc_tl_nvl_team_t *team)
{
    int N = (int)UCC_TL_TEAM_SIZE(team), me = (int)UCC_TL_TEAM_RANK(team);
    fd_server_stop(team);
    if (team->stream) { cudaStreamSynchronize(team->stream); cudaStreamDestroy(team->stream); team->stream = NULL; }
    for (int p = 0; p < NVL_MAX_PEERS; p++) {
        if (team->p2p_stream[p]) { cudaStreamSynchronize(team->p2p_stream[p]); cudaStreamDestroy(team->p2p_stream[p]); team->p2p_stream[p] = NULL; }
        if (team->p2p_side_event[p]) { cudaEventDestroy(team->p2p_side_event[p]); team->p2p_side_event[p] = NULL; }
    }
    if (team->mc_va) { unmap_va(team->mc_va, team->mc_size); team->mc_va = NULL; }
    if (team->nvls || team->mc_handle) {
        if (team->mc_handle) { CUdevice d; if (ucc_cu.cuDeviceGet(&d, NVL_CTX(team)->dev) == CUDA_SUCCESS && ucc_cu.cuMulticastUnbind) ucc_cu.cuMulticastUnbind(team->mc_handle, d, 0, team->mc_size);
            ucc_cu.cuMemRelease(team->mc_handle); team->mc_handle = 0; }
    }
    for (int p = 0; p < N; p++) {
        if (p == me || !team->peer_va[p]) continue;
        if (team->heap_kind == NVL_HEAP_VMM) { unmap_va(team->peer_va[p], team->infos ? team->infos[p].size : team->heap_size); if (team->peer_handle[p]) ucc_cu.cuMemRelease(team->peer_handle[p]); }
        else if (team->heap_kind == NVL_HEAP_IPC) cudaIpcCloseMemHandle(team->peer_va[p]);
        team->peer_va[p] = NULL;
    }
    if (team->heap) {
        if (team->heap_kind == NVL_HEAP_VMM) { unmap_va(team->heap, team->heap_size); ucc_cu.cuMemRelease(team->mem_handle); if (team->heap_fd >= 0) close(team->heap_fd); }
        else cudaFree(team->heap);
        team->heap = NULL;
    }
    if (team->mc_fd >= 0) { close(team->mc_fd); team->mc_fd = -1; }
    if (team->host_err) { cudaFreeHost(team->host_err); team->host_err = NULL; }
    for (unsigned l = 0; l < NVL_MAX_LANES; l++) if (team->order_event[l]) { cudaEventDestroy(team->order_event[l]); team->order_event[l] = NULL; }
    ucc_tl_nvl_xb_release(team);
    if (team->oob_internal) { ucc_internal_oob_finalize(&team->oob); team->oob_internal = 0; }
    free(team->infos); team->infos = NULL; free(team->sync_vals); team->sync_vals = NULL;
    (void)cudaGetLastError();
}

/* ------------------------------------------------------------------ */
/* create                                                              */
/* ------------------------------------------------------------------ */
static ucc_status_t team_finish(ucc_tl_nvl_team_t *team);
static void registry_add(ucc_tl_nvl_team_t *team);
ucc_status_t ucc_tl_nvl_team_create_post(ucc_base_context_t *b_ctx, const ucc_base_team_params_t *params, ucc_base_team_t **team_p)
{
    ucc_tl_nvl_context_t *ctx = ucc_derived_of(b_ctx, ucc_tl_nvl_context_t);
    ucc_tl_nvl_team_t *team;
    ucc_rank_t N = params->size;
    int same_pid = 1, all_vmm = 1, all_mc = 1, distinct_dev = 1, want_mc, dev;
    int devs[NVL_MAX_PEERS], gpu_idx[NVL_MAX_PEERS];
    ucc_status_t st;
    if (N < 1 || N > NVL_MAX_PEERS) return UCC_ERR_NOT_SUPPORTED;
    if (cudaGetDevice(&dev) != cudaSuccess || dev != ctx->dev) { (void)cudaGetLastError(); tl_debug(b_ctx->lib, "current device differs from the context's device"); return UCC_ERR_NOT_SUPPORTED; }
    team = (ucc_tl_nvl_team_t *)calloc(1, sizeof(*team));
    if (!team) return UCC_ERR_NO_MEMORY;
    team->super.super.context = b_ctx; team->super.super.params = *params;
    team->heap_fd = -1; team->mc_fd = -1; team->srv_sock = -1;
    if (N == 1) { /* nothing to share: collectives on CUDA buffers become one copy kernel on the caller's stream */
        team->self = 1; team->nlanes = 1; team->heap_kind = NVL_HEAP_LOCAL;
        st = team_finish(team);
        if (st != UCC_OK) { team_release(team); free(team); return st; }
        *team_p = &team->super.super;
        return UCC_OK;
    }
    for (ucc_rank_t r = 0; r < N; r++) {
        uint32_t len = 0;
        ucc_tl_nvl_addr_t *a = (ucc_tl_nvl_addr_t *)ucc_get_team_ep_addr(b_ctx->ucc_context, params->team, ucc_ep_map_eval(params->map, r), ucc_tl_nvl.super.id, &len);
        if (!a || len < sizeof(*a) || a->host_hash != ctx->addr.host_hash) { tl_debug(b_ctx->lib, "rank %u is not reachable over NVLink from here", r); free(team); return UCC_ERR_NOT_SUPPORTED; }
        if (a->pid != ctx->addr.pid) same_pid = 0;
        if (!a->vmm_ok) all_vmm = 0;
        if (!a->mc_ok) all_mc = 0;
        devs[r] = a->dev;
        for (ucc_rank_t q = 0; q < r; q++) if (devs[q] == a->dev) distinct_dev = 0;
        /* the member's GPU in this host's sysinfo table (all members are on this host, see above) */
        gpu_idx[r] = -1;
        for (int g = 0; g < ucc_local_host.n_gpus; g++)
            if (a->pci_bus >= 0 && ucc_local_host.gpus[g].pci.domain == (uint16_t)a->pci_domain && ucc_local_host.gpus[g].pci.bus == (uint8_t)a->pci_bus && ucc_local_host.gpus[g].pci.device == (uint8_t)a->pci_device) gpu_idx[r] = g;
    }
    /* NVLink graph of the team (reference tl_cuda_team_topo.c:119-429 builds the same from its own NVML scan): a pair of
     * different GPUs without an NVLink path would make every kernel crawl over PCIe - such a team is left to the next TL */
    team->topo_known = 0; team->nvswitch = 0;
    /* "known" only when the NVML scan saw NVLinks at all: a container that hides the link state must not make every pair look unconnected */
    for (int g = 0; g < ucc_local_host.n_gpus; g++) if (ucc_local_host.gpus[g].caps & (UCC_GPU_CAP_NVLINK | UCC_GPU_CAP_NVSWITCH)) team->topo_known = 1;
    for (ucc_rank_t r = 0; r < N; r++) {
        if (gpu_idx[r] < 0) team->topo_known = 0;
        else if (ucc_local_host.gpus[gpu_idx[r]].caps & UCC_GPU_CAP_NVSWITCH) team->nvswitch = 1;
    }
    for (ucc_rank_t r = 0; r < N; r++) for (ucc_rank_t q = 0; q < N; q++) {
        team->links[r][q] = (team->topo_known && r != q && gpu_idx[r] != gpu_idx[q]) ? ucc_local_host.nvlink_matrix[gpu_idx[r]][gpu_idx[q]] : 0;
        if (r != q && devs[r] != devs[q] && !same_pid_pair_unknown(team->topo_known) && team->links[r][q] == 0 && ctx->cfg.require_nvlink != UCC_NO) {
            tl_debug(b_ctx->lib, "members %u and %u have no NVLink path: tl/nvl does not serve this team", r, q); free(team); return UCC_ERR_NOT_SUPPORTED;
        }
    }
    if (!team->topo_known && ctx->cfg.require_nvlink == UCC_YES && N > 1 && distinct_dev) { tl_debug(b_ctx->lib, "NVLink topology unknown and REQUIRE_NVLINK=y"); free(team); return UCC_ERR_NOT_SUPPORTED; }
    /* ring order: consecutive members share the most links (identity behind an NVSwitch, where every pair is equivalent) */
    if (team->topo_known && !team->nvswitch && N > 2) {
        uint8_t flat[NVL_MAX_PEERS * NVL_MAX_PEERS];
        for (ucc_rank_t r = 0; r < N; r++) for (ucc_rank_t q = 0; q < N; q++) flat[r * N + q] = team->links[r][q];
        ucc_ring_build_from_links(flat, N, team->ring_order);
    } else for (ucc_rank_t r = 0; r < N; r++) team->ring_order[r] = r;
    if (ctx->cfg.ring_reverse) for (ucc_rank_t r = 0; r < N / 2; r++) { ucc_rank_t x = team->ring_order[r]; team->ring_order[r] = team->ring_order[N - 1 - r]; team->ring_order[N - 1 - r] = x; }
    team->heap_kind = same_pid ? NVL_HEAP_LOCAL : (all_vmm ? NVL_HEAP_VMM : NVL_HEAP_IPC);
    want_mc = (team->heap_kind == NVL_HEAP_VMM) && all_mc && distinct_dev && ctx->cfg.use_nvls != UCC_NO;
    team->nvls = 0;
    /* OOB for the handshake: the team's own, or one built on the service team */
    if (params->params.mask & UCC_TEAM_PARAM_FIELD_OOB) team->oob = params->params.oob;
    else {
        ucc_subset_t s; s.map = params->map; s.myrank = params->rank;
        st = ucc_internal_oob_init(params->team, s, &team->oob);
        if (st != UCC_OK) { free(team); return UCC_ERR_NOT_SUPPORTED; }
        team->oob_internal = 1;
    }
    if (team->oob.n_oob_eps != N) { tl_debug(b_ctx->lib, "team OOB size mismatch"); if (team->oob_internal) ucc_internal_oob_finalize(&team->oob); free(team); return UCC_ERR_NOT_SUPPORTED; }
    team->infos = (nvl_rank_info_t *)calloc(N, sizeof(nvl_rank_info_t));
    team->sync_vals = (int32_t *)calloc((size_t)N * 4, sizeof(int32_t));
    memset(&team->my_info, 0, sizeof(team->my_info));
    team->my_info.pid = ctx->addr.pid; team->my_info.dev = ctx->dev; team->my_info.kind = (int32_t)team->heap_kind; team->my_info.fd = -1; team->my_info.mc_fd = -1;
    st = heap_alloc(team, want_mc);
    if (st == UCC_OK && team->heap_kind == NVL_HEAP_VMM) {
        snprintf(team->my_info.sock, sizeof(team->my_info.sock), "ucc_nvl.%d.%p", (int)getpid(), (void *)team);
        st = fd_server_start(team, team->my_info.sock);
        team->my_info.fd = team->heap_fd;
    }
    if (st == UCC_OK && team->heap_kind == NVL_HEAP_IPC && cudaIpcGetMemHandle(&team->my_info.ipc, team->heap) != cudaSuccess) { (void)cudaGetLastError(); st = UCC_ERR_NO_RESOURCE; }
    team->my_info.status = (int32_t)st; team->my_info.ptr = (uint64_t)(uintptr_t)team->heap; team->my_info.size = team->heap_size;
    team->sync_send[3] = want_mc;
    if (ctx->cfg.zcopy != UCC_NO && ucc_tl_nvl_xb_create(team) == UCC_OK) snprintf(team->my_info.xb_name, sizeof(team->my_info.xb_name), "%s", team->xb_name);
    st = team->oob.allgather(&team->my_info, team->infos, sizeof(nvl_rank_info_t), team->oob.coll_info, &team->oob_req);
    if (st != UCC_OK) { team_release(team); free(team); return st; }
    team->state = NVL_TEAM_XCHG_INFO;
    *team_p = &team->super.super;
    return UCC_OK;
}

static ucc_status_t post_sync(ucc_tl_nvl_team_t *team, int32_t v0, int32_t v1)
{
    team->sync_send[0] = v0; team->sync_send[1] = v1;
    return team->oob.allgather(team->sync_send, team->sync_vals, 4 * sizeof(int32_t), team->oob.coll_info, &team->oob_req);
}
/* returns INPROGRESS, or OK with *all_ok telling whether every rank reported UCC_OK in slot 0 */
static ucc_status_t test_sync(ucc_tl_nvl_team_t *team, int *all_ok)
{
    ucc_status_t st = team->oob.req_test(team->oob_req);
    if (st == UCC_INPROGRESS) return st;
    team->oob.req_free(team->oob_req); team->oob_req = NULL;
    if (st < 0) return st;
    *all_ok = 1;
    for (ucc_rank_t r = 0; r < UCC_TL_TEAM_SIZE(team); r++) if (team->sync_vals[4 * r] != UCC_OK) *all_ok = 0;
    return UCC_OK;
}

static ucc_status_t map_peers(ucc_tl_nvl_team_t *team)
{
    ucc_tl_nvl_context_t *ctx = NVL_CTX(team);
    ucc_rank_t N = UCC_TL_TEAM_SIZE(team), me = UCC_TL_TEAM_RANK(team);
    for (ucc_rank_t p = 0; p < N; p++) {
        nvl_rank_info_t *pi = &team->infos[p];
        if (p == me) { team->peer_va[p] = team->heap; continue; }
        if (team->heap_kind == NVL_HEAP_LOCAL) {
            if (pi->dev != ctx->dev) { cudaError_t e = cudaDeviceEnablePeerAccess(pi->dev, 0); if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { (void)cudaGetLastError(); return UCC_ERR_NOT_SUPPORTED; } (void)cudaGetLastError(); }
            team->peer_va[p] = (char *)(uintptr_t)pi->ptr;
        } else if (team->heap_kind == NVL_HEAP_VMM) {
            int fd = fetch_fd(team, pi->pid, pi->fd, pi->sock);
            CUresult r;
            if (fd < 0) { tl_debug(NVL_LIB(team), "could not obtain the heap handle of rank %u", p); return UCC_ERR_NO_RESOURCE; }
            r = ucc_cu.cuMemImportFromShareableHandle(&team->peer_handle[p], (void *)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
            close(fd);
            if (r != CUDA_SUCCESS) { tl_debug(NVL_LIB(team), "cuMemImportFromShareableHandle failed: %s", ucc_cu_err_str(r)); return UCC_ERR_NO_RESOURCE; }
            if (map_handle(team->peer_handle[p], pi->size, 2u << 20, ctx->dev, &team->peer_va[p]) != UCC_OK) return UCC_ERR_NO_RESOURCE;
        } else {
            void *ptr = NULL;
            if (cudaIpcOpenMemHandle(&ptr, pi->ipc, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { (void)cudaGetLastError(); return UCC_ERR_NO_RESOURCE; }
            team->peer_va[p] = (char *)ptr;
        }
    }
    return UCC_OK;
}

static ucc_status_t team_finish(ucc_tl_nvl_team_t *team)
{
    ucc_tl_nvl_context_t *ctx = NVL_CTX(team);
    ucc_rank_t N = UCC_TL_TEAM_SIZE(team);
    fd_server_stop(team);
    if (team->heap_fd >= 0) { close(team->heap_fd); team->heap_fd = -1; }
    if (team->mc_fd >= 0) { close(team->mc_fd); team->mc_fd = -1; }
    CUDA_CHECK(cudaStreamCreateWithFlags(&team->stream, cudaStreamNonBlocking));
    CUDA_CHECK(cudaHostAlloc((void **)&team->host_err, sizeof(uint32_t), cudaHostAllocMapped));
    *team->host_err = 0;
    for (unsigned l = 0; l < team->nlanes; l++) CUDA_CHECK(cudaEventCreateWithFlags(&team->order_event[l], cudaEventDisableTiming));
    ucc_list_head_init(&team->launch_q); ucc_spinlock_init(&team->launch_lock);
    memset(team->last_stream, 0, sizeof(team->last_stream)); memset(team->last_event, 0, sizeof(team->last_event)); team->lane_seq = 0; team->xb_seq = 0;
    memset(&team->dev, 0, sizeof(team->dev));
    team->dev.rank = (int)UCC_TL_TEAM_RANK(team); team->dev.size = (int)N;
    for (ucc_rank_t p = 0; p < N; p++) team->dev.heap[p] = team->peer_va[p];
    team->dev.mc_heap = team->nvls ? team->mc_va : NULL;
    team->dev.data_size = ctx->cfg.symmetric_size;
    team->dev.timeout_ns = (uint64_t)(ctx->cfg.timeout * 1e9);
    { void *dptr = NULL; CUDA_CHECK(cudaHostGetDevicePointer(&dptr, team->host_err, 0)); team->dev.host_err = (uint32_t *)dptr; }
    team->state = NVL_TEAM_READY;
    registry_add(team);
    tl_debug(NVL_LIB(team), "team %p ready: size %u, heap %s %zu MB, nvls %d", (void *)team, N,
             team->heap_kind == NVL_HEAP_LOCAL ? "local" : team->heap_kind == NVL_HEAP_VMM ? "vmm" : "ipc", team->heap_size >> 20, team->nvls);
    return UCC_OK;
}

ucc_status_t ucc_tl_nvl_team_create_test(ucc_base_team_t *b)
{
    ucc_tl_nvl_team_t *team = ucc_derived_of(b, ucc_tl_nvl_team_t);
    ucc_tl_nvl_context_t *ctx = NVL_CTX(team);
    ucc_rank_t N = UCC_TL_TEAM_SIZE(team), me = UCC_TL_TEAM_RANK(team);
    ucc_status_t st;
    int ok = 0, want_mc = team->sync_send[3];
    switch (team->state) {
    case NVL_TEAM_XCHG_INFO:
        st = team->oob.req_test(team->oob_req);
        if (st == UCC_INPROGRESS) return st;
        team->oob.req_free(team->oob_req); team->oob_req = NULL;
        if (st < 0) goto fail;
        st = UCC_OK;
        for (ucc_rank_t r = 0; r < N; r++) if (team->infos[r].status != UCC_OK) st = UCC_ERR_NOT_SUPPORTED;
        if (st == UCC_OK) st = map_peers(team);
        team->sync_send[2] = (st == UCC_OK && team->xb_mine && ucc_tl_nvl_xb_attach(team) == UCC_OK); /* zero-copy needs every board */
        if ((st = post_sync(team, (int32_t)st, 0)) != UCC_OK) goto fail;
        team->state = NVL_TEAM_SYNC1;
        /* fall through */
    case NVL_TEAM_SYNC1:
        st = test_sync(team, &ok);
        if (st == UCC_INPROGRESS) return st;
        if (st < 0 || !ok) { st = UCC_ERR_NOT_SUPPORTED; goto fail; }
        team->zcopy = ucc_cu.cuStreamWaitValue32 && ucc_cu.cuStreamWriteValue32; /* deferred launches park user streams on a gate word */
        for (ucc_rank_t r = 0; r < N; r++) if (!team->sync_vals[4 * r + 2]) team->zcopy = 0;
        ucc_tl_nvl_xb_unlink(team); /* everybody who could attach has done so */
        if (!want_mc) return team_finish(team);
        /* rank 0 creates the multicast object and offers it to the others */
        st = UCC_OK;
        if (me == 0) {
            CUmulticastObjectProp mp; memset(&mp, 0, sizeof(mp));
            mp.numDevices = N; mp.size = team->mc_size; mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
            if (ucc_cu.cuMulticastCreate(&team->mc_handle, &mp) != CUDA_SUCCESS) { team->mc_handle = 0; st = UCC_ERR_NOT_SUPPORTED; }
            else if (ucc_cu.cuMemExportToShareableHandle(&team->mc_fd, team->mc_handle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0) != CUDA_SUCCESS) st = UCC_ERR_NOT_SUPPORTED;
            else { char nm[64]; snprintf(nm, sizeof(nm), "%s.mc", team->my_info.sock); st = fd_server_add(team, nm, team->mc_fd); }
        }
        if ((st = post_sync(team, (int32_t)st, team->mc_fd)) != UCC_OK) goto fail;
        team->state = NVL_TEAM_MC_CREATE;
        /* fall through */
    case NVL_TEAM_MC_CREATE: {
        CUdevice cudev;
        st = test_sync(team, &ok);
        if (st == UCC_INPROGRESS) return st;
        if (st < 0) goto fail;
        if (team->sync_vals[0] != UCC_OK) { tl_debug(NVL_LIB(team), "multicast object creation failed, continuing without NVLS"); return team_finish(team); }
        st = UCC_OK;
        if (me != 0) {
            char nm[64]; int fd;
            snprintf(nm, sizeof(nm), "%s.mc", team->infos[0].sock);
            fd = fetch_fd(team, team->infos[0].pid, team->sync_vals[1], nm);
            if (fd < 0 || ucc_cu.cuMemImportFromShareableHandle(&team->mc_handle, (void *)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR) != CUDA_SUCCESS) { team->mc_handle = 0; st = UCC_ERR_NOT_SUPPORTED; }
            if (fd >= 0) close(fd);
        }
        if (st == UCC_OK && (ucc_cu.cuDeviceGet(&cudev, ctx->dev) != CUDA_SUCCESS || ucc_cu.cuMulticastAddDevice(team->mc_handle, cudev) != CUDA_SUCCESS)) st = UCC_ERR_NOT_SUPPORTED;
        if ((st = post_sync(team, (int32_t)st, 0)) != UCC_OK) goto fail;
        team->state = NVL_TEAM_MC_ADDED;
    }   /* fall through */
    case NVL_TEAM_MC_ADDED:
        st = test_sync(team, &ok);
        if (st == UCC_INPROGRESS) return st;
        if (st < 0) goto fail;
        if (!ok) { tl_debug(NVL_LIB(team), "not every device joined the multicast group, continuing without NVLS"); if (team->mc_handle) { ucc_cu.cuMemRelease(team->mc_handle); team->mc_handle = 0; } return team_finish(team); }
        st = UCC_OK;
        if (ucc_cu.cuMulticastBindMem(team->mc_handle, 0, team->mem_handle, 0, team->mc_size, 0) != CUDA_SUCCESS) st = UCC_ERR_NOT_SUPPORTED;
        else if (map_handle(team->mc_handle, team->mc_size, 2u << 20, ctx->dev, &team->mc_va) != UCC_OK) st = UCC_ERR_NOT_SUPPORTED;
        if ((st = post_sync(team, (int32_t)st, 0)) != UCC_OK) goto fail;
        team->state = NVL_TEAM_MC_BOUND;
        /* fall through */
    case NVL_TEAM_MC_BOUND:
        st = test_sync(team, &ok);
        if (st == UCC_INPROGRESS) return st;
        if (st < 0) goto fail;
        team->nvls = ok;
        if (!ok) { tl_debug(NVL_LIB(team), "multicast bind failed on some rank, continuing without NVLS"); if (team->mc_va) { unmap_va(team->mc_va, team->mc_size); team->mc_va = NULL; } }
        return team_finish(team);
    case NVL_TEAM_READY: return UCC_OK;
    default: st = UCC_ERR_NOT_SUPPORTED; break;
    }
fail:
    team->state = NVL_TEAM_FAILED;
    team_release(team);
    free(team);
    return st < 0 ? st : UCC_ERR_NOT_SUPPORTED;
}

/* ------------------------------------------------------------------ */
/* symmetric user region                                               */
/* ------------------------------------------------------------------ */
/* ready teams, so that an application holding only the ucc_team_h can ask for the user region of the tl/nvl team that spans it,
 * or for its device-error latch */
#define NVL_REG_MAX 1024
static ucc_tl_nvl_team_t *g_teams[NVL_REG_MAX];
static ucc_spinlock_t     g_teams_lock;
static void registry_add(ucc_tl_nvl_team_t *team)
{ ucc_spin_lock(&g_teams_lock); for (int i = 0; i < NVL_REG_MAX; i++) if (!g_teams[i]) { g_teams[i] = team; break; } ucc_spin_unlock(&g_teams_lock); }
static void registry_del(ucc_tl_nvl_team_t *team)
{ ucc_spin_lock(&g_teams_lock); for (int i = 0; i < NVL_REG_MAX; i++) if (g_teams[i] == team) g_teams[i] = NULL; ucc_spin_unlock(&g_teams_lock); }

/* Base address (in this process) and size of the symmetric user region of the tl/nvl team covering ALL members of `core_team`
 * (UCC_TL_NVL_USER_SIZE > 0).  *nvls tells whether the region is bound to an NVSwitch multicast object, i.e. whether
 * allreduce on buffers inside it takes the in-place in-switch path.  The caller sub-allocates; a buffer must sit at the
 * same offset on every member. */
UCC_EXPORT ucc_status_t ucc_tl_nvl_symm_region(ucc_team_h core_team, void **base, size_t *size, int *nvls)
{
    ucc_status_t st = UCC_ERR_NOT_FOUND;
    ucc_spin_lock(&g_teams_lock);
    for (int i = 0; i < NVL_REG_MAX; i++) {
        ucc_tl_nvl_team_t *t = g_teams[i];
        if (!t || t->self || (ucc_team_h)t->super.super.params.team != core_team || UCC_TL_TEAM_SIZE(t) != ucc_team_size_(core_team)) continue;
        if (!NVL_CTX(t)->cfg.user_size) continue;
        *base = t->heap + t->lane_stride * t->nlanes; *size = NVL_CTX(t)->cfg.user_size;
        if (nvls) *nvls = t->nvls;
        st = UCC_OK; break;
    }
    ucc_spin_unlock(&g_teams_lock);
    return st;
}

/* Reads and clears the device-error latch of every tl/nvl team of `core_team`: 1 when a kernel of one of them gave up a
 * device-side wait (TL_NVL_TIMEOUT) since the last call, 0 otherwise, -1 when the core team has no tl/nvl team.  An eager
 * collective reports such a timeout through its request; a collective replayed from a CUDA graph has no request, so an
 * application that replays graphs asks here after synchronizing the replay stream. */
UCC_EXPORT int ucc_tl_nvl_take_device_error(ucc_team_h core_team)
{
    int r = -1;
    ucc_spin_lock(&g_teams_lock);
    for (int i = 0; i < NVL_REG_MAX; i++) {
        ucc_tl_nvl_team_t *t = g_teams[i];
        if (!t || (ucc_team_h)t->super.super.params.team != core_team) continue;
        if (r < 0) r = 0;
        if (t->host_err && __atomic_exchange_n(t->host_err, 0, __ATOMIC_ACQ_REL)) r = 1;
    }
    ucc_spin_unlock(&g_teams_lock);
    return r;
}

ucc_status_t ucc_tl_nvl_team_destroy(ucc_base_team_t *b)
{
    ucc_tl_nvl_team_t *team = ucc_derived_of(b, ucc_tl_nvl_team_t);
    registry_del(team);
    team_release(team);
    free(team);
    return UCC_OK;
}
