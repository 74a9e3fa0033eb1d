/* tl/nvl: the NVLink / NVSwitch transport (role of reference tl/cuda, 10.3 K LoC).
 *
 * Design (NVLink-first, not a port):
 *   - one symmetric heap per team, mapped into every member's address space at team
 *     creation (CUDA VMM handles passed as POSIX fds between processes, plain pointers
 *     between contexts of one process) and, when the fabric offers it, additionally bound
 *     to an NVLS multicast object;
 *   - data plane AND synchronisation plane live on the GPU: every collective is one kernel
 *     (kernels/nvl_kernels.cu) that signals peers with flag words in their heaps; the host only
 *     enqueues the kernel and polls one CUDA event;
 *   - no shared-memory control segment, no CPU step counters, no per-collective IPC handle
 *     exchange, no executor round trips (compare reference tl_cuda_team.c:62-217,
 *     reduce_scatterv_linear.c:229-328, alltoallv_ce.c:70-126).
 */
#ifndef UCC_TL_NVL_H_
#define UCC_TL_NVL_H_
#include "components/tl/ucc_tl.h"
#include "components/mc/ucc_mc.h"
#include "core/ucc_context.h"
#include "core/ucc_team.h"
#include "core/ucc_ee.h"
#include "utils/ucc_mpool.h"
#include "utils/ucc_list.h"
#include "utils/ucc_atomic.h"
#include "utils/cuda/ucc_cuda_util.h"
#include "kernels/nvl_kernels.h"

#define UCC_TL_NVL_DEFAULT_SCORE 40
#define UCC_TL_NVL_SUPPORTED_COLLS UCC_COLL_TYPE_ALL

typedef struct ucc_tl_nvl_lib_config { ucc_tl_lib_config_t super; } ucc_tl_nvl_lib_config_t;
typedef struct ucc_tl_nvl_context_config {
    ucc_tl_context_config_t super;
    size_t   symmetric_size;   /* data region of the per-team heap */
    unsigned nblocks;          /* CTAs per collective kernel (auto: by message size) */
    unsigned max_blocks;
    unsigned nthreads;
    double   timeout;          /* device spin budget, seconds */
    int      use_nvls;         /* ternary */
    int      use_vmm;          /* ternary: VMM+fd export (needed for NVLS) or cudaMalloc+cudaIpc */
    size_t   oneshot_thresh;   /* allreduce: one-shot push below, two-shot above */
    size_t   nvls_thresh;      /* allreduce: use NVLS at or above this size */
    int      fd_via_pidfd;     /* ternary: try pidfd_getfd before the unix socket */
    int      zcopy;            /* ternary: read / write the members' user buffers in place (CUDA IPC) */
    size_t   zcopy_thresh;     /* ... for messages of at least this size */
    size_t   user_size;        /* symmetric USER region appended to every team heap (0: none), see ucc_tl_nvl_symm_region() */
    int      ring_reverse;     /* debug / test knob: walk the ring in the opposite direction (exercises non-identity ring orders) */
    int      require_nvlink;   /* ternary: refuse teams with a GPU pair that has no NVLink path (try: only when the topology is known) */
    int      bulk;             /* ternary: TMA bulk copies (cp.async.bulk) as the data mover of the zero-copy push exchange */
    size_t   bulk_thresh;
    unsigned bulk_ctas;        /* one-warp CTAs of a bulk-copy kernel */
    double   p2p_timeout;      /* seconds a send / recv kernel waits for the peer (0: forever) */
    size_t   p2p_rndv_thresh;  /* send / recv of at least this size: rendezvous (sender stores into the receiver's buffer) */
    unsigned slots;            /* independent collective lanes per team (reference tl/cuda MAX_CONCURRENT): collectives on different lanes may overlap */
} ucc_tl_nvl_context_config_t;

/* ---- zero-copy buffer exchange board (tl_nvl_direct.c): one single-writer POSIX shm segment per rank ---- */
#define NVL_MAX_LANES 8
#define NVL_EVENT_CACHE 256
#define NVL_XB_SLOTS 64
#define NVL_IPC_CACHE_MAX 64
typedef enum { NVL_XB_NONE = 0, NVL_XB_EMPTY, NVL_XB_RAW, NVL_XB_IPC } nvl_xb_kind_t;
typedef struct nvl_xb_buf { int32_t kind; int32_t pad; uint64_t base, off, len, alloc_len; cudaIpcMemHandle_t handle; } nvl_xb_buf_t;
typedef struct nvl_xb_entry { uint64_t seq; nvl_xb_buf_t src, dst; uint64_t aux[NVL_MAX_PEERS]; /* alltoallv: byte offset of source p's block inside my dst */ } nvl_xb_entry_t;
/* rendezvous send / recv: rz[p][k % NVL_XB_RZ_SLOTS] is written by the board's owner (the RECEIVER) for its k-th large receive from
 * member p (seq = k + 1); rz_consumed[p] is written by the owner as SENDER: how many receive posts of member p it has used;
 * rz_launched[p], also written as sender: how many zero-copy push kernels towards member p have been launched */
#define NVL_XB_RZ_SLOTS 4
typedef struct nvl_xb_rz { uint64_t seq; nvl_xb_buf_t buf; } nvl_xb_rz_t;
typedef struct nvl_xb_seg { uint64_t consumed; uint64_t pad[7]; nvl_xb_entry_t e[NVL_XB_SLOTS];
                            uint64_t rz_consumed[NVL_MAX_PEERS]; uint32_t rz_launched[NVL_MAX_PEERS]; nvl_xb_rz_t rz[NVL_MAX_PEERS][NVL_XB_RZ_SLOTS]; } nvl_xb_seg_t;
/* one peer allocation mapped through CUDA IPC.  refs: zero-copy plans whose tables point into it (a persistent request's cached
 * tables until the request is finalized; any other post from its mapping to its launch).  last_use: recorded behind the latest
 * eager launch that used it.  An entry is idle, and may be closed, once it has no refs and last_use has completed. */
typedef struct nvl_ipc_entry { uint64_t base; size_t len; cudaIpcMemHandle_t handle; void *mapped; unsigned refs; int stale; cudaEvent_t last_use; } nvl_ipc_entry_t;
/* per peer; holds NVL_IPC_CACHE_MAX entries, a full cache closes its idle entries and grows when none is idle */
typedef struct nvl_ipc_cache { unsigned n, cap; nvl_ipc_entry_t **e; } nvl_ipc_cache_t;

typedef struct ucc_tl_nvl_lib { ucc_tl_lib_t super; } ucc_tl_nvl_lib_t;

typedef struct ucc_tl_nvl_addr { /* published through the core address exchange */
    uint64_t host_hash; int32_t pid; int32_t dev; uint64_t ep_id; int32_t vmm_ok, mc_ok;
    int32_t  pci_domain, pci_bus, pci_device; /* identifies the GPU on its host whatever CUDA_VISIBLE_DEVICES says (-1: unknown) */
} ucc_tl_nvl_addr_t;

typedef struct ucc_tl_nvl_context {
    ucc_tl_context_t            super;
    ucc_tl_nvl_context_config_t cfg;
    ucc_tl_nvl_addr_t           addr;
    int                         dev;
    int                         sm_count;
    unsigned                    lane_blocks;   /* CTAs one collective kernel may use: all lanes of a team together stay co-resident */
    ucc_mpool_t                 task_mp;
    ucc_thread_mode_t           tm;
    /* completion events are recycled: creating / destroying one per request costs more host time than launching a small collective */
    cudaEvent_t                 ev_cache[NVL_EVENT_CACHE];
    unsigned                    n_ev_cache;
    ucc_spinlock_t              ev_lock;
} ucc_tl_nvl_context_t;

typedef enum { NVL_HEAP_LOCAL, NVL_HEAP_VMM, NVL_HEAP_IPC } nvl_heap_kind_t;
/* what every rank tells the others about its heap */
typedef struct nvl_rank_info {
    int32_t  pid, dev, kind, fd, mc_fd;
    int32_t  status;     /* UCC_OK or the error that makes this rank unusable */
    uint64_t ptr;        /* LOCAL: device pointer valid inside that process */
    uint64_t size;
    cudaIpcMemHandle_t ipc;
    char     sock[48];   /* abstract unix socket serving the fds */
    char     xb_name[48];/* POSIX shm name of this rank's buffer exchange board ("" = none) */
} nvl_rank_info_t;

typedef enum { NVL_TEAM_INIT, NVL_TEAM_XCHG_INFO, NVL_TEAM_MAP, NVL_TEAM_SYNC1, NVL_TEAM_MC_CREATE, NVL_TEAM_MC_IMPORT,
               NVL_TEAM_MC_ADDED, NVL_TEAM_MC_BOUND, NVL_TEAM_READY, NVL_TEAM_FAILED } nvl_team_state_t;

typedef struct ucc_tl_nvl_team {
    ucc_tl_team_t     super;
    nvl_team_state_t  state;
    int               self;                 /* single-member team: no heap, collectives are local copies */
    ucc_team_oob_coll_t oob;
    int               oob_internal;
    void             *oob_req;
    nvl_rank_info_t   my_info, *infos;
    int32_t          *sync_vals, sync_send[4];
    /* heap */
    nvl_heap_kind_t   heap_kind;
    size_t            heap_size;
    char             *heap;                 /* my heap (device VA) */
    CUmemGenericAllocationHandle mem_handle;/* VMM */
    int               heap_fd;
    char             *peer_va[NVL_MAX_PEERS];
    CUmemGenericAllocationHandle peer_handle[NVL_MAX_PEERS];
    /* NVLS */
    int               nvls;                 /* multicast mapping is live */
    CUmemGenericAllocationHandle mc_handle;
    int               mc_fd;
    char             *mc_va;
    size_t            mc_size;
    /* fd server */
    int               srv_sock; void *srv_thread; volatile int srv_stop;
    /* runtime */
    nvl_team_dev_t    dev;
    cudaStream_t      stream;
    uint32_t         *host_err;             /* pinned, device mapped */
    /* zero-copy exchange */
    int               zcopy;                /* boards of all members are mapped */
    char              xb_name[48]; int xb_named;
    nvl_xb_seg_t     *xb_mine, *xb[NVL_MAX_PEERS];
    nvl_ipc_cache_t   ipc_cache[NVL_MAX_PEERS];
    uint64_t          xb_seq;               /* next exchange sequence (advances at post, same order on every rank) */
    /* launch ordering: kernels of one team must start in post order on every rank (the device-side epochs assume it) */
    ucc_list_link_t   launch_q;             /* posted tasks whose kernel is not launched yet */
    ucc_spinlock_t    launch_lock;
    /* NVLink topology of the team (sysinfo graph: topo/cuda/sysinfo_cuda.c -> ucc_local_host): links[r][q] = NVLinks between the GPUs
     * of members r and q (0: unknown / none), ring_order = visit order in which consecutive members share the most links */
    uint8_t           links[NVL_MAX_PEERS][NVL_MAX_PEERS];
    int               topo_known, nvswitch;
    ucc_rank_t        ring_order[NVL_MAX_PEERS];
    /* lanes ("slots"): the heap holds `nlanes` complete copies of [control | one-shot | p2p | data]; consecutive collectives take
     * consecutive lanes (post order, identical on every member), so up to nlanes collectives of a team - posted on different
     * streams - run concurrently with their own flags, epochs and staging space.  Kernels of ONE lane still start in post order. */
    unsigned          nlanes;
    size_t            lane_stride;
    uint32_t          lane_seq;             /* next lane (advances at post) */
    cudaStream_t      last_stream[NVL_MAX_LANES];  /* stream of the lane's most recent launch */
    cudaEvent_t       order_event[NVL_MAX_LANES];  /* spare event: swapped with a finalized task's event that last_event points to */
    cudaEvent_t       last_event[NVL_MAX_LANES];   /* completion event of the lane's most recent launch */
    /* send / recv (two-member active sets).  Sends to one peer are launched in post order (p2p_post_seq / p2p_launch_seq); sends
     * that had to wait for the receiver (rendezvous) run on a per-peer side stream, the user's stream then waits for their event */
    uint32_t          p2p_post_seq[NVL_MAX_PEERS], p2p_launch_seq[NVL_MAX_PEERS];
    uint64_t          rz_tx[NVL_MAX_PEERS];     /* large sends posted to peer (index into the receiver's board entries) */
    uint64_t          rz_rx[NVL_MAX_PEERS];     /* large receives posted from peer */
    uint64_t          rz_pub[NVL_MAX_PEERS];    /* large receives from peer already published */
    uint32_t          rz_zc_tx[NVL_MAX_PEERS], rz_zc_rx[NVL_MAX_PEERS]; /* ... of those, the ones that really go zero-copy (device counter p2p_rz_done) */
    cudaStream_t      p2p_stream[NVL_MAX_PEERS];
    cudaEvent_t       p2p_side_event[NVL_MAX_PEERS]; int p2p_side_used[NVL_MAX_PEERS];
} ucc_tl_nvl_team_t;

/* How a task launches, chosen at init and never changed afterwards.  A post only resolves whether the members' buffers could be
 * mapped (u.red.direct / u.xchg.direct): that bit picks the path's direct (zero-copy) form over its staged form, where it has one.
 * Reduction paths use u.red, the ones from NVL_PATH_AG_SYMM to NVL_PATH_SELF_COPY_CE use u.xchg, send / recv uses u.p2p. */
typedef enum {
    NVL_PATH_ONESHOT,      /* one-shot allreduce */
    NVL_PATH_ONESHOT_RS,   /* one-shot reduce_scatter(v) (kernels/nvl_oneshot_rs.cuh) */
    NVL_PATH_TWOSHOT,      /* staged two-shot reduction; direct: in place in the members' buffers */
    NVL_PATH_NVLS,         /* staged two-shot reduction through the switch */
    NVL_PATH_RING,         /* step-structured reduction, ring schedule */
    NVL_PATH_RHD,          /* step-structured reduction, recursive halving / doubling */
    NVL_PATH_NVLS_PIPE,    /* pipelined staged NVLS allreduce (kernels/nvl_pipe.cuh) */
    NVL_PATH_SYMM,         /* NVLS reduction on symmetric user memory, nothing staged (kernels/nvl_symm.cuh) */
    NVL_PATH_RED_CE,       /* allreduce / reduce_scatter(v) under UCC_COLL_ARGS_HINT_OPTIMIZE_OVERLAP_GPU; direct: the copy engines pull
                              the peers' blocks into my heap, a small local kernel reduces them; staged: the two-shot staged kernel */
    NVL_PATH_AG_SYMM,      /* allgather into a symmetric destination by multimem.st (u.xchg: src, src_bytes, dst, push_off) */
    NVL_PATH_PULL,         /* stage + pull exchange; direct: pull from the members' source buffers */
    NVL_PATH_PULL_NVLS,    /* exchange whose staging multicasts into every heap (u.xchg.use_mc) */
    NVL_PATH_PULL_RING,    /* allgather(v) in N-1 neighbour steps (u.xchg.ring) */
    NVL_PATH_PUSH,         /* direct: store my blocks into the members' destinations (kernels/nvl_push.cu); staged: pull */
    NVL_PATH_PUSH_BULK,    /* the same, moved by TMA bulk copies */
    NVL_PATH_PUSH_CE,      /* the same, one cudaMemcpyAsync per peer between two barrier kernels */
    NVL_PATH_XCHG_CE,      /* bcast / gather(v) / scatter(v) under the overlap hint; direct: cudaMemcpyAsync to / from the root's mapped
                              buffer between two barrier kernels; staged: pull */
    NVL_PATH_SWAP,         /* in-place alltoall(v); direct: pairwise swap kernel (kernels/nvl_swap.cu); staged: self-copy + pull */
    NVL_PATH_SELF_COPY,    /* team of one: u.xchg.{dst,src,src_bytes} describe the only data movement, copied by a kernel */
    NVL_PATH_SELF_COPY_CE, /* ... copied by cudaMemcpyAsync */
    NVL_PATH_BARRIER,
    NVL_PATH_P2P,          /* two-member active-set bcast = send / recv over a heap channel (kernels/nvl_p2p.cu, u.p2p) */
    NVL_PATH_NUM
} nvl_path_t;
typedef enum { NVL_TASK_LAUNCHED, NVL_TASK_QUEUED, NVL_TASK_P2P_WAIT /* send waiting for its turn / for the receiver's buffer */ } nvl_task_state_t;
/* Zero-copy plan of a task (tl_nvl_direct.c): where a post finds the members' buffers for its path's direct form - tables built
 * from registrations at init, the tables the first post of a persistent request resolved, or the exchange board at every post.
 * It holds no pointer into the task: nvl_rebuild swaps task bodies. */
enum { NVL_ZC_SRC = 1, NVL_ZC_DST = 2, /* sides every member's direct form touches */
       NVL_ZC_ALIGN = 4, /* a board entry that is not 16-byte aligned makes every member stage */
       NVL_ZC_WITHDRAW = 8 /* I publish my buffers as not mappable, which makes every member stage */ };
typedef enum { NVL_ZC_RESOLVE, NVL_ZC_STAGED, NVL_ZC_DIRECT } nvl_zc_cache_t;
typedef struct nvl_zc {
    unsigned       flags;              /* NVL_ZC_*; 0: the direct form is not wanted */
    const void    *src; void *dst; size_t src_len, dst_len; /* mine, as published */
    nvl_zc_cache_t cache;              /* RESOLVE: at every post; STAGED / DIRECT: for every post, with the tables in d */
    nvl_direct_t   d;
    uint64_t       seq;                /* board entry of the current post */
    int            published, pending; /* pending: the current post resolves through the board */
    nvl_ipc_entry_t *pin[2 * NVL_MAX_PEERS]; unsigned npin; /* the IPC mappings the tables in d point into, referenced */
} nvl_zc_t;
typedef struct ucc_tl_nvl_task {
    ucc_coll_task_t     super;
    ucc_tl_nvl_team_t  *team;
    nvl_path_t          path;
    union { nvl_red_args_t red; nvl_xchg_args_t xchg; nvl_p2p_args_t p2p; } u;
    int                 nblocks, nthreads;
    cudaEvent_t         event;
    cudaStream_t        stream;     /* stream of the current post */
    int                 captured;   /* posted into a capturing stream: completes immediately */
    unsigned            lane;       /* lane of the current post */
    /* zero-copy / deferred launch */
    nvl_task_state_t    state;
    ucc_list_link_t     q_elem;
    nvl_zc_t            zc;
    cudaEvent_t         in_event;
    /* send / recv */
    int                 p2p_rndv;      /* large message: rendezvous protocol */
    uint32_t            p2p_order;     /* send: position among the sends to this peer */
    uint64_t            rz_seq;        /* rendezvous: index among the large messages of the pair */
    int                 p2p_ee_done;   /* the UCC_EVENT_COLLECTIVE_POST of this post was delivered */
    int                 rz_wait_pending;/* recv: the wait kernel is not in the stream yet (it follows the launch of the sender's push) */
    int                 rz_stream_idle;/* recv: the stream had nothing queued at post time */
    int                 rz_pub_pending;/* recv: the buffer is not on the board yet (stream not there yet / slot busy / not my turn) */
    nvl_xb_buf_t        rz_buf;        /* recv: what will be published */
    /* push paths: what the direct form stores where (XCHG_CE: recv_off = what the root publishes for member p - where p's block
     * lands in the root's destination (gather(v)) or starts in its source (scatter(v)); peer_land[root] = that entry for me) */
    struct { size_t send_off[NVL_MAX_PEERS], send_bytes[NVL_MAX_PEERS], land_off[NVL_MAX_PEERS], recv_off[NVL_MAX_PEERS], peer_land[NVL_MAX_PEERS]; int lookup; } push;
} ucc_tl_nvl_task_t;

/* tl/nvl part of a ucc_mem_map() handle (tl_nvl_memh.c) */
typedef struct nvl_memh {
    uint64_t magic, host_hash, addr, base, off, len;
    int32_t  pid, dev, has_ipc, imported;
    cudaIpcMemHandle_t ipc;
    char    *mapped;   /* address of the segment in THIS process (NULL: unreachable) */
    void    *opened;   /* cudaIpcOpenMemHandle result to close at unmap */
} nvl_memh_t;
ucc_status_t ucc_tl_nvl_mem_map(const ucc_base_context_t *ctx, ucc_mem_map_mode_t mode, void *memh, void *tl_h);
ucc_status_t ucc_tl_nvl_mem_unmap(const ucc_base_context_t *ctx, ucc_mem_map_mode_t mode, void *tl_h);
ucc_status_t ucc_tl_nvl_memh_pack(const ucc_base_context_t *ctx, ucc_mem_map_mode_t mode, void *tl_h, void **pack_buffer);

ucc_status_t ucc_tl_nvl_xb_create(ucc_tl_nvl_team_t *team);
ucc_status_t ucc_tl_nvl_xb_attach(ucc_tl_nvl_team_t *team);
void         ucc_tl_nvl_xb_unlink(ucc_tl_nvl_team_t *team);
void         ucc_tl_nvl_xb_release(ucc_tl_nvl_team_t *team);
int          ucc_tl_nvl_is_managed(const void *ptr);
void         ucc_tl_nvl_xb_export(ucc_tl_nvl_team_t *team, const void *ptr, size_t len, nvl_xb_buf_t *b);
char        *ucc_tl_nvl_xb_import(ucc_tl_nvl_team_t *team, ucc_rank_t p, const nvl_xb_buf_t *b);
void         ucc_tl_nvl_zc_init(ucc_tl_nvl_team_t *team, nvl_zc_t *zc, unsigned flags, const void *src, size_t src_len, void *dst, size_t dst_len, const ucc_coll_args_t *reg);
void         ucc_tl_nvl_zc_post(ucc_tl_nvl_team_t *team, nvl_zc_t *zc, int captured, const size_t *aux);
ucc_status_t ucc_tl_nvl_zc_ready(ucc_tl_nvl_team_t *team, nvl_zc_t *zc, int persistent, const size_t *aux, size_t *aux_for_me, int *direct);
void         ucc_tl_nvl_zc_launched(nvl_zc_t *zc, cudaStream_t s);
void         ucc_tl_nvl_zc_release(nvl_zc_t *zc);
void         ucc_tl_nvl_ipc_used(ucc_tl_nvl_team_t *team, ucc_rank_t p, const void *ptr, cudaStream_t s);

#define NVL_CTX(_team) ucc_derived_of((_team)->super.super.context, ucc_tl_nvl_context_t)
extern ucc_tl_iface_t ucc_tl_nvl;
extern ucc_config_field_t ucc_tl_nvl_context_config_table[];

ucc_status_t ucc_tl_nvl_team_create_post(ucc_base_context_t *ctx, const ucc_base_team_params_t *params, ucc_base_team_t **team);
ucc_status_t ucc_tl_nvl_team_create_test(ucc_base_team_t *team);
ucc_status_t ucc_tl_nvl_team_destroy(ucc_base_team_t *team);
ucc_status_t ucc_tl_nvl_team_get_scores(ucc_base_team_t *team, ucc_coll_score_t **score);
ucc_status_t ucc_tl_nvl_coll_init(ucc_base_coll_args_t *args, ucc_base_team_t *team, ucc_coll_task_t **task);
ucc_status_t ucc_tl_nvl_alg_id_to_init(int alg_id, const char *alg_id_str, ucc_coll_type_t coll_type, ucc_memory_type_t mem_type, ucc_base_coll_init_fn_t *init);
void         ucc_tl_nvl_register_alg_info(void);
#endif
