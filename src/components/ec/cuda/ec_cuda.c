/* ec/cuda: CUDA execution component.
 *   events    - cudaEvent wrappers pooled per process
 *   executor  - three flavours selected at start():
 *       interruptible   (no stream given)  every task is a kernel / async memcpy on one of N internal
 *                                          streams + a completion event
 *       persistent      (user stream given) a resident worker kernel on the user's stream pops tasks
 *                                          from a host-pinned ring, so tasks are ordered with the
 *                                          user's work without further launches
 *       persistent_wait (user stream given, no task types requested) a 1-thread kernel only holds the
 *                                          stream until the executor is stopped
 * Capabilities and knobs follow reference ec/cuda (ec_cuda.c:21-76, ec_cuda_executor_*.c). */
#include "components/ec/base/ucc_ec_base.h"
#include "utils/ucc_mpool.h"
#include "utils/ucc_math.h"
#include "utils/ucc_string.h"
#include "utils/cuda/ucc_cuda_util.h"
#include "core/ucc_dt.h"
#include "kernels/ec_cuda_kernels.h"

typedef enum { EC_CUDA_TASK_KERNEL, EC_CUDA_TASK_MEMOPS, EC_CUDA_TASK_AUTO } ec_cuda_stream_task_mode_t;
typedef struct ucc_ec_cuda_config {
    ucc_ec_config_t super;
    unsigned stream_task_mode;
    unsigned exec_num_workers, exec_num_threads, exec_max_tasks, exec_num_streams;
    size_t   exec_copy_thresh;
    unsigned reduce_num_blocks, reduce_num_threads;
    int      use_cooperative_launch;
} ucc_ec_cuda_config_t;

typedef enum { EXEC_INITIALIZED, EXEC_POSTED, EXEC_STARTED, EXEC_SHUTDOWN } exec_state_t;
typedef enum { EXEC_MODE_INTERRUPTIBLE, EXEC_MODE_PERSISTENT, EXEC_MODE_PERSISTENT_WAIT } exec_mode_t;
typedef struct ucc_ec_cuda_executor {
    ucc_ee_executor_t super;
    exec_mode_t       mode;
    exec_state_t      state;
    uint64_t          task_types;
    ec_ring_t        *ring, *ring_dev;  /* persistent: host-pinned ring + its device alias */
    uint32_t          pidx;
    volatile uint32_t *wait_state, *wait_state_dev;
} ucc_ec_cuda_executor_t;
typedef struct ucc_ec_cuda_task { ucc_ee_executor_task_t super; cudaEvent_t event; ec_ring_slot_t *slot; } ucc_ec_cuda_task_t;

typedef struct ucc_ec_cuda {
    ucc_ec_base_t     super;
    ucc_thread_mode_t tm;
    ucc_mpool_t       events, executors, tasks;
    cudaStream_t     *streams; unsigned n_streams, rr; int streams_dev;
    ucc_spinlock_t    lock;
} ucc_ec_cuda_t;
extern ucc_ec_cuda_t ucc_ec_cuda;
#define EC_CFG ((ucc_ec_cuda_config_t *)ucc_ec_cuda.super.config)
#define ec_error(_f, ...) ucc_log_component(UCC_LOG_LEVEL_ERROR, &ucc_ec_cuda.super.config->log_component, _f, ##__VA_ARGS__)
#define ec_debug(_f, ...) ucc_log_component(UCC_LOG_LEVEL_DEBUG, &ucc_ec_cuda.super.config->log_component, _f, ##__VA_ARGS__)

static const char *stream_task_modes[] = {"kernel", "memops", "auto", NULL};
static ucc_config_field_t ucc_ec_cuda_config_table[] = {
    {"", "", NULL, ucc_offsetof(ucc_ec_cuda_config_t, super), UCC_CONFIG_TYPE_TABLE(ucc_ec_config_table)},
    {"STREAM_TASK_MODE", "auto", "Mechanism used to hold a user stream for a triggered collective (kernel: wait kernel, memops: stream memory operations)",
     ucc_offsetof(ucc_ec_cuda_config_t, stream_task_mode), UCC_CONFIG_TYPE_ENUM(stream_task_modes)},
    {"EXEC_NUM_WORKERS", "1", "Number of worker thread blocks of the persistent executor", ucc_offsetof(ucc_ec_cuda_config_t, exec_num_workers), UCC_CONFIG_TYPE_UINT},
    {"EXEC_NUM_THREADS", "512", "Threads per block of the persistent executor", ucc_offsetof(ucc_ec_cuda_config_t, exec_num_threads), UCC_CONFIG_TYPE_UINT},
    {"EXEC_MAX_TASKS", "128", "Depth of the persistent executor task ring", ucc_offsetof(ucc_ec_cuda_config_t, exec_max_tasks), UCC_CONFIG_TYPE_UINT},
    {"EXEC_NUM_STREAMS", "16", "Number of internal streams used by the interruptible executor", ucc_offsetof(ucc_ec_cuda_config_t, exec_num_streams), UCC_CONFIG_TYPE_UINT},
    {"EXEC_COPY_LARGE_THRESH", "1M", "Multi-buffer copies with a member at least this big use the copy engines (cudaMemcpyAsync) instead of the copy kernel",
     ucc_offsetof(ucc_ec_cuda_config_t, exec_copy_thresh), UCC_CONFIG_TYPE_MEMUNITS},
    {"REDUCE_NUM_BLOCKS", "auto", "Thread blocks of a reduction kernel (auto: from the element count)", ucc_offsetof(ucc_ec_cuda_config_t, reduce_num_blocks), UCC_CONFIG_TYPE_UINT},
    {"REDUCE_NUM_THREADS", "512", "Threads per block of a reduction kernel", ucc_offsetof(ucc_ec_cuda_config_t, reduce_num_threads), UCC_CONFIG_TYPE_UINT},
    {"USE_COOPERATIVE_LAUNCH", "0", "Launch the persistent executor kernel cooperatively", ucc_offsetof(ucc_ec_cuda_config_t, use_cooperative_launch), UCC_CONFIG_TYPE_BOOL},
    {NULL}};

static void event_obj_init(ucc_mpool_t *mp, void *obj, void *chunk) { (void)mp; (void)chunk; if (cudaEventCreateWithFlags((cudaEvent_t *)obj, cudaEventDisableTiming) != cudaSuccess) { (void)cudaGetLastError(); *(cudaEvent_t *)obj = NULL; } }
/* Pinned, device-mapped control blocks of the persistent executors (task ring / wait word) are RECYCLED: cudaHostAlloc and above all
 * cudaFreeHost synchronise the whole device, so an executor started or stopped by one collective stalled on every kernel running
 * on the GPU - e.g. on the spinning kernels of collectives that wait for this very rank (a hierarchical allreduce whose leaders
 * reduce through the host TL while the other ranks already sit in the node broadcast). */
typedef struct ec_pin_blk { struct ec_pin_blk *next; } ec_pin_blk_t;
static ec_pin_blk_t  *ec_pin_free;
static size_t         ec_pin_size;
static ucc_spinlock_t ec_pin_lock;
static int            ec_pin_lock_init;
static void *ec_pin_get(size_t sz)
{
    ec_pin_blk_t *b = NULL;
    void *p = NULL;
    if (!ec_pin_lock_init) { ucc_spinlock_init(&ec_pin_lock); ec_pin_lock_init = 1; }
    ucc_spin_lock(&ec_pin_lock);
    if (ec_pin_free && ec_pin_size >= sz) { b = ec_pin_free; ec_pin_free = b->next; }
    ucc_spin_unlock(&ec_pin_lock);
    if (b) return b;
    if (sz < ec_pin_size) sz = ec_pin_size;
    if (cudaHostAlloc(&p, sz, cudaHostAllocMapped) != cudaSuccess) { (void)cudaGetLastError(); return NULL; }
    ucc_spin_lock(&ec_pin_lock);
    if (sz > ec_pin_size) ec_pin_size = sz; /* blocks already on the list keep their (smaller) size: only handed out while sizes agree */
    ucc_spin_unlock(&ec_pin_lock);
    return p;
}
static void ec_pin_put(void *p)
{
    ec_pin_blk_t *b = (ec_pin_blk_t *)p;
    ucc_spin_lock(&ec_pin_lock);
    b->next = ec_pin_free; ec_pin_free = b;
    ucc_spin_unlock(&ec_pin_lock);
}
static void ec_pin_drain(void)
{
    while (ec_pin_free) { ec_pin_blk_t *b = ec_pin_free; ec_pin_free = b->next; cudaFreeHost(b); }
    ec_pin_size = 0;
}

static void event_obj_cleanup(ucc_mpool_t *mp, void *obj) { (void)mp; if (*(cudaEvent_t *)obj) cudaEventDestroy(*(cudaEvent_t *)obj); }

static ucc_status_t ec_cuda_init(const ucc_ec_params_t *p)
{
    static ucc_mpool_ops_t ev_ops = {NULL, NULL, event_obj_init, event_obj_cleanup};
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { (void)cudaGetLastError(); ec_debug("cuda devices are not found"); return UCC_ERR_NO_RESOURCE; }
    ucc_ec_cuda.tm = p->thread_mode; ucc_ec_cuda.streams = NULL; ucc_ec_cuda.n_streams = 0; ucc_ec_cuda.rr = 0;
    ucc_spinlock_init(&ucc_ec_cuda.lock);
    ucc_mpool_init(&ucc_ec_cuda.events, 0, sizeof(cudaEvent_t), 0, 8, 16, (unsigned)-1, &ev_ops, UCC_THREAD_MULTIPLE, "ec cuda events");
    ucc_mpool_init(&ucc_ec_cuda.executors, 0, sizeof(ucc_ec_cuda_executor_t), 0, 64, 8, (unsigned)-1, NULL, UCC_THREAD_MULTIPLE, "ec cuda executors");
    ucc_mpool_init(&ucc_ec_cuda.tasks, 0, sizeof(ucc_ec_cuda_task_t), 0, 64, 32, (unsigned)-1, NULL, UCC_THREAD_MULTIPLE, "ec cuda tasks");
    return UCC_OK;
}
static ucc_status_t ec_cuda_get_attr(ucc_ec_attr_t *a) { a->max_executors_bufs = EC_MAX_SRCS; return UCC_OK; }
static ucc_status_t ec_cuda_finalize(void)
{
    for (unsigned i = 0; i < ucc_ec_cuda.n_streams; i++) cudaStreamDestroy(ucc_ec_cuda.streams[i]);
    free(ucc_ec_cuda.streams); ucc_ec_cuda.streams = NULL; ucc_ec_cuda.n_streams = 0;
    ucc_mpool_cleanup(&ucc_ec_cuda.events, 0); ucc_mpool_cleanup(&ucc_ec_cuda.executors, 1); ucc_mpool_cleanup(&ucc_ec_cuda.tasks, 1);
    ec_pin_drain();
    (void)cudaGetLastError();
    return UCC_OK;
}
static ucc_status_t next_stream(cudaStream_t *s)
{
    ucc_spin_lock(&ucc_ec_cuda.lock);
    if (!ucc_ec_cuda.streams) {
        unsigned n = EC_CFG->exec_num_streams ? EC_CFG->exec_num_streams : 1;
        ucc_ec_cuda.streams = (cudaStream_t *)calloc(n, sizeof(cudaStream_t));
        for (unsigned i = 0; i < n; i++) if (cudaStreamCreateWithFlags(&ucc_ec_cuda.streams[i], cudaStreamNonBlocking) != cudaSuccess) { (void)cudaGetLastError(); ucc_spin_unlock(&ucc_ec_cuda.lock); return UCC_ERR_NO_RESOURCE; }
        ucc_ec_cuda.n_streams = n;
    }
    *s = ucc_ec_cuda.streams[ucc_ec_cuda.rr++ % ucc_ec_cuda.n_streams];
    ucc_spin_unlock(&ucc_ec_cuda.lock);
    return UCC_OK;
}

/* ---- events ---- */
static ucc_status_t ev_create(void **event) { cudaEvent_t *e = (cudaEvent_t *)ucc_mpool_get(&ucc_ec_cuda.events); if (!e || !*e) return UCC_ERR_NO_MEMORY; *event = e; return UCC_OK; }
static ucc_status_t ev_destroy(void *event) { ucc_mpool_put(event); return UCC_OK; }
static ucc_status_t ev_post(void *ee_context, void *event) { CUDA_CHECK(cudaEventRecord(*(cudaEvent_t *)event, (cudaStream_t)ee_context)); return UCC_OK; }
static ucc_status_t ev_test(void *event)
{ cudaError_t e = cudaEventQuery(*(cudaEvent_t *)event); if (e == cudaErrorNotReady) { (void)cudaGetLastError(); return UCC_INPROGRESS; } return ucc_cuda_error_to_status(e); }

/* ---- translation ---- */
static int to_ec_dt(ucc_datatype_t dt)
{
    switch (dt) {
    case UCC_DT_INT8: return EC_DT_I8; case UCC_DT_INT16: return EC_DT_I16; case UCC_DT_INT32: return EC_DT_I32; case UCC_DT_INT64: return EC_DT_I64;
    case UCC_DT_UINT8: return EC_DT_U8; case UCC_DT_UINT16: return EC_DT_U16; case UCC_DT_UINT32: return EC_DT_U32; case UCC_DT_UINT64: return EC_DT_U64;
    case UCC_DT_FLOAT16: return EC_DT_F16; case UCC_DT_FLOAT32: return EC_DT_F32; case UCC_DT_FLOAT64: return EC_DT_F64; case UCC_DT_BFLOAT16: return EC_DT_BF16;
    case UCC_DT_FLOAT32_COMPLEX: return EC_DT_C64; case UCC_DT_FLOAT64_COMPLEX: return EC_DT_C128;
    case UCC_DT_INT128: return EC_DT_I128; case UCC_DT_UINT128: return EC_DT_U128;
    default: return -1;
    }
}
static int to_ec_op(ucc_reduction_op_t op) { return op == UCC_OP_AVG ? EC_OP_SUM : (op <= UCC_OP_BXOR ? (int)op : -1); }
static int ec_op_index(ucc_reduction_op_t op)
{
    switch (op) { case UCC_OP_SUM: case UCC_OP_AVG: return EC_OP_SUM; case UCC_OP_PROD: return EC_OP_PROD; case UCC_OP_MAX: return EC_OP_MAX; case UCC_OP_MIN: return EC_OP_MIN;
    case UCC_OP_LAND: return EC_OP_LAND; case UCC_OP_LOR: return EC_OP_LOR; case UCC_OP_LXOR: return EC_OP_LXOR; case UCC_OP_BAND: return EC_OP_BAND;
    case UCC_OP_BOR: return EC_OP_BOR; case UCC_OP_BXOR: return EC_OP_BXOR; default: return -1; }
}

/* fill a ring-slot style description from executor task args; returns kind or <0 */
static int describe(const ucc_ee_executor_task_args_t *a, ec_ring_slot_t *d)
{
    int with_alpha = !!(a->flags & UCC_EEE_TASK_FLAG_REDUCE_WITH_ALPHA);
    (void)to_ec_op;
    switch (a->task_type) {
    case UCC_EE_EXECUTOR_TASK_REDUCE: {
        ec_reduce_args_t *r = &d->u.reduce; void *const *srcs = (a->flags & UCC_EEE_TASK_FLAG_REDUCE_SRCS_EXT) ? (void *const *)a->reduce.srcs_ext : (void *const *)a->reduce.srcs;
        memset(r, 0, sizeof(*r));
        if (a->reduce.n_srcs > EC_MAX_SRCS) return -1;
        r->dst = a->reduce.dst; for (int i = 0; i < a->reduce.n_srcs; i++) r->srcs[i] = srcs[i];
        r->n_srcs = a->reduce.n_srcs; r->count = a->reduce.count; r->dt = to_ec_dt(a->reduce.dt); r->op = ec_op_index(a->reduce.op); r->with_alpha = with_alpha; r->alpha = a->reduce.alpha;
        r->avg_n = with_alpha ? ucc_ec_avg_divisor(r->alpha) : 0;
        if (r->dt < 0 || r->op < 0 || !ec_dt_supports_op(r->dt, r->op) || (a->reduce.op == UCC_OP_AVG && !with_alpha)) return -1;
        return EC_TASK_REDUCE; }
    case UCC_EE_EXECUTOR_TASK_REDUCE_STRIDED: {
        ec_reduce_args_t *r = &d->u.reduce; memset(r, 0, sizeof(*r));
        r->dst = a->reduce_strided.dst; r->srcs[0] = a->reduce_strided.src1; r->src2 = a->reduce_strided.src2; r->stride = a->reduce_strided.stride; r->strided = 1;
        r->n_srcs = a->reduce_strided.n_src2 + 1; r->count = a->reduce_strided.count; r->dt = to_ec_dt(a->reduce_strided.dt); r->op = ec_op_index(a->reduce_strided.op);
        r->with_alpha = with_alpha; r->alpha = a->reduce_strided.alpha; r->avg_n = with_alpha ? ucc_ec_avg_divisor(r->alpha) : 0;
        if (r->dt < 0 || r->op < 0 || !ec_dt_supports_op(r->dt, r->op) || (a->reduce_strided.op == UCC_OP_AVG && !with_alpha)) return -1;
        return EC_TASK_REDUCE; }
    case UCC_EE_EXECUTOR_TASK_REDUCE_MULTI_DST: {
        ec_reduce_multi_dst_args_t *m = &d->u.rmd; memset(m, 0, sizeof(*m));
        m->n_bufs = a->reduce_multi_dst.n_bufs; m->dt = to_ec_dt(a->reduce_multi_dst.dt); m->op = ec_op_index(a->reduce_multi_dst.op);
        /* (AVG: the task has no alpha to scale by, so it would silently be a SUM) */
        if (m->n_bufs > EC_MULTI_BUFS || m->dt < 0 || m->op < 0 || !ec_dt_supports_op(m->dt, m->op) || a->reduce_multi_dst.op == UCC_OP_AVG) return -1;
        for (int j = 0; j < m->n_bufs; j++) { m->dst[j] = a->reduce_multi_dst.dst[j]; m->src1[j] = a->reduce_multi_dst.src1[j]; m->src2[j] = a->reduce_multi_dst.src2[j]; m->counts[j] = a->reduce_multi_dst.counts[j]; }
        return EC_TASK_REDUCE_MULTI_DST; }
    case UCC_EE_EXECUTOR_TASK_COPY: {
        ec_copy_multi_args_t *c = &d->u.copy; memset(c, 0, sizeof(*c)); c->n = 1; c->dst[0] = a->copy.dst; c->src[0] = a->copy.src; c->bytes[0] = a->copy.len; return EC_TASK_COPY; }
    case UCC_EE_EXECUTOR_TASK_COPY_MULTI: {
        ec_copy_multi_args_t *c = &d->u.copy; memset(c, 0, sizeof(*c)); c->n = (int)a->copy_multi.num_vectors;
        if (c->n > EC_MULTI_BUFS) return -1;
        for (int j = 0; j < c->n; j++) { c->dst[j] = a->copy_multi.dst[j]; c->src[j] = a->copy_multi.src[j]; c->bytes[j] = a->copy_multi.counts[j]; }
        return EC_TASK_COPY_MULTI; }
    default: return -1;
    }
}

static ucc_status_t launch_on_stream(int kind, ec_ring_slot_t *d, cudaStream_t s)
{
    unsigned nt = EC_CFG->reduce_num_threads; cudaError_t e = cudaSuccess;
    if (nt < 32 || nt > 1024) nt = 512;
    switch (kind) {
    case EC_TASK_REDUCE: {
        size_t nb = EC_CFG->reduce_num_blocks;
        if (nb == UCC_UUNITS_AUTO || nb == 0) { nb = (d->u.reduce.count + nt * 8 - 1) / (nt * 8); if (nb < 1) nb = 1; if (nb > 592) nb = 592; }
        e = ec_launch_reduce(&d->u.reduce, (int)nb, (int)nt, s); break; }
    case EC_TASK_REDUCE_MULTI_DST: e = ec_launch_reduce_multi_dst(&d->u.rmd, (int)nt, s); break;
    case EC_TASK_COPY: e = cudaMemcpyAsync(d->u.copy.dst[0], d->u.copy.src[0], d->u.copy.bytes[0], cudaMemcpyDefault, s); break;
    case EC_TASK_COPY_MULTI: {
        int large = 0;
        for (int j = 0; j < d->u.copy.n; j++) if (d->u.copy.bytes[j] >= EC_CFG->exec_copy_thresh) large = 1;
        if (large) { for (int j = 0; j < d->u.copy.n && e == cudaSuccess; j++) e = cudaMemcpyAsync(d->u.copy.dst[j], d->u.copy.src[j], d->u.copy.bytes[j], cudaMemcpyDefault, s); }
        else e = ec_launch_copy_multi(&d->u.copy, 1024, s);
        break; }
    default: return UCC_ERR_INVALID_PARAM;
    }
    if (e != cudaSuccess) { (void)cudaGetLastError(); ec_error("executor task launch failed: %s", cudaGetErrorString(e)); return UCC_ERR_NO_MESSAGE; }
    return UCC_OK;
}

/* ---- executor ---- */
static ucc_status_t exec_init(const ucc_ee_executor_params_t *p, ucc_ee_executor_t **xp)
{
    ucc_ec_cuda_executor_t *x = (ucc_ec_cuda_executor_t *)ucc_mpool_get(&ucc_ec_cuda.executors);
    if (!x) return UCC_ERR_NO_MEMORY;
    memset(x, 0, sizeof(*x));
    x->super.ee_type = UCC_EE_CUDA_STREAM; x->super.ee_context = NULL; x->state = EXEC_INITIALIZED; x->mode = EXEC_MODE_INTERRUPTIBLE;
    x->task_types = (p->mask & UCC_EE_EXECUTOR_PARAM_FIELD_TASK_TYPES) ? p->task_types : (uint64_t)-1;
    *xp = &x->super;
    return UCC_OK;
}
static ucc_status_t exec_status(const ucc_ee_executor_t *xe)
{
    const ucc_ec_cuda_executor_t *x = (const ucc_ec_cuda_executor_t *)xe;
    switch (x->state) {
    case EXEC_INITIALIZED: return UCC_OPERATION_INITIALIZED;
    case EXEC_POSTED: if (x->mode == EXEC_MODE_PERSISTENT && x->ring->started) { ((ucc_ec_cuda_executor_t *)x)->state = EXEC_STARTED; return UCC_OK; } return x->mode == EXEC_MODE_PERSISTENT ? UCC_INPROGRESS : UCC_OK;
    default: return UCC_OK;
    }
}
static ucc_status_t exec_start(ucc_ee_executor_t *xe, void *ee_context)
{
    ucc_ec_cuda_executor_t *x = (ucc_ec_cuda_executor_t *)xe;
    x->super.ee_context = ee_context;
    if (!ee_context) { x->mode = EXEC_MODE_INTERRUPTIBLE; x->state = EXEC_STARTED; return UCC_OK; }
    if (x->task_types == 0) { /* nothing to execute: just keep the stream busy until stop() */
        void *dp = NULL;
        x->mode = EXEC_MODE_PERSISTENT_WAIT;
        x->wait_state = (volatile uint32_t *)ec_pin_get(sizeof(ec_ring_t) + (size_t)(EC_CFG->exec_max_tasks ? EC_CFG->exec_max_tasks : 128) * sizeof(ec_ring_slot_t));
        if (!x->wait_state) return UCC_ERR_NO_MEMORY;
        *x->wait_state = 0;
        CUDA_CHECK(cudaHostGetDevicePointer(&dp, (void *)x->wait_state, 0)); x->wait_state_dev = (volatile uint32_t *)dp;
        /* STREAM_TASK_MODE (reference ec_cuda.c:21-36): memops parks the stream on a stream memory operation - no SM, no thread - when the
         * driver exports it; kernel (and auto) launch the one-thread wait kernel */
        if (EC_CFG->stream_task_mode == EC_CUDA_TASK_MEMOPS && ucc_cu_api_load() == UCC_OK && ucc_cu.cuStreamWaitValue32 &&
            ucc_cu.cuStreamWaitValue32((CUstream)ee_context, (CUdeviceptr)(uintptr_t)x->wait_state_dev, 1, 0 /* CU_STREAM_WAIT_VALUE_GEQ */) == CUDA_SUCCESS) {
            x->state = EXEC_STARTED;
            return UCC_OK;
        }
        if (ec_launch_wait(x->wait_state_dev, (cudaStream_t)ee_context) != cudaSuccess) { (void)cudaGetLastError(); return UCC_ERR_NO_MESSAGE; }
        x->state = EXEC_STARTED;
        return UCC_OK;
    }
    {
        unsigned n = EC_CFG->exec_max_tasks ? EC_CFG->exec_max_tasks : 128; size_t sz = sizeof(ec_ring_t) + (size_t)n * sizeof(ec_ring_slot_t);
        void *dp = NULL;
        x->mode = EXEC_MODE_PERSISTENT;
        x->ring = (ec_ring_t *)ec_pin_get(sz);
        if (!x->ring) return UCC_ERR_NO_MEMORY;
        memset(x->ring, 0, sz); x->ring->n_slots = n; x->pidx = 0;
        CUDA_CHECK(cudaHostGetDevicePointer(&dp, x->ring, 0)); x->ring_dev = (ec_ring_t *)dp;
        if (ec_launch_persistent(x->ring_dev, (int)EC_CFG->exec_num_workers, (int)ucc_min(EC_CFG->exec_num_threads, 1024u), EC_CFG->use_cooperative_launch, (cudaStream_t)ee_context) != cudaSuccess) {
            (void)cudaGetLastError(); ec_pin_put(x->ring); x->ring = NULL; return UCC_ERR_NO_MESSAGE; }
        x->state = EXEC_POSTED;
    }
    return UCC_OK;
}
static ucc_status_t exec_stop(ucc_ee_executor_t *xe)
{
    ucc_ec_cuda_executor_t *x = (ucc_ec_cuda_executor_t *)xe;
    if (x->mode == EXEC_MODE_PERSISTENT && x->ring) {
        x->ring->shutdown = 1; ucc_memory_cpu_store_fence();
        cudaStreamSynchronize((cudaStream_t)x->super.ee_context); /* the worker kernel observes the flag and retires */
        ec_pin_put(x->ring); x->ring = NULL;
    } else if (x->mode == EXEC_MODE_PERSISTENT_WAIT && x->wait_state) {
        *x->wait_state = 1; ucc_memory_cpu_store_fence();
        cudaStreamSynchronize((cudaStream_t)x->super.ee_context);
        ec_pin_put((void *)x->wait_state); x->wait_state = NULL;
    }
    x->state = EXEC_INITIALIZED; x->super.ee_context = NULL; x->mode = EXEC_MODE_INTERRUPTIBLE;
    return UCC_OK;
}
static ucc_status_t exec_finalize(ucc_ee_executor_t *xe) { ucc_ec_cuda_executor_t *x = (ucc_ec_cuda_executor_t *)xe; if (x->state != EXEC_INITIALIZED) exec_stop(xe); ucc_mpool_put(x); return UCC_OK; }

static ucc_status_t exec_task_post(ucc_ee_executor_t *xe, const ucc_ee_executor_task_args_t *a, ucc_ee_executor_task_t **tp)
{
    ucc_ec_cuda_executor_t *x = (ucc_ec_cuda_executor_t *)xe;
    ucc_ec_cuda_task_t *t = (ucc_ec_cuda_task_t *)ucc_mpool_get(&ucc_ec_cuda.tasks);
    ucc_status_t st;
    int kind;
    if (!t) return UCC_ERR_NO_MEMORY;
    t->super.eee = xe; t->super.args = *a; t->super.status = UCC_INPROGRESS; t->super.handle = NULL; t->event = NULL; t->slot = NULL;
    if (x->mode == EXEC_MODE_PERSISTENT) {
        ec_ring_slot_t *slot = &x->ring->slots[x->pidx % x->ring->n_slots];
        if (slot->state != EC_SLOT_FREE) { ucc_mpool_put(t); return UCC_ERR_NO_RESOURCE; } /* ring full: the oldest task is not finalized */
        kind = describe(a, slot);
        if (kind < 0) { ucc_mpool_put(t); return UCC_ERR_NOT_SUPPORTED; }
        slot->kind = (uint32_t)kind;
        slot->seq = x->pidx; /* the worker that serves task pidx takes this slot only for it, not for a task of another lap */
        ucc_memory_cpu_store_fence();
        slot->state = EC_SLOT_POSTED;
        x->pidx++; t->slot = slot;
    } else {
        ec_ring_slot_t d; cudaStream_t s; cudaEvent_t *e;
        kind = describe(a, &d);
        if (kind < 0) { ucc_mpool_put(t); return UCC_ERR_NOT_SUPPORTED; }
        st = next_stream(&s);
        if (st == UCC_OK) st = launch_on_stream(kind, &d, s);
        if (st != UCC_OK) { ucc_mpool_put(t); return st; }
        e = (cudaEvent_t *)ucc_mpool_get(&ucc_ec_cuda.events);
        if (!e || !*e || cudaEventRecord(*e, s) != cudaSuccess) { (void)cudaGetLastError(); if (e) ucc_mpool_put(e); ucc_mpool_put(t); return UCC_ERR_NO_RESOURCE; }
        t->super.handle = e; t->event = *e;
    }
    *tp = &t->super;
    return UCC_OK;
}
static ucc_status_t exec_task_test(const ucc_ee_executor_task_t *te)
{
    ucc_ec_cuda_task_t *t = (ucc_ec_cuda_task_t *)te;
    cudaError_t e;
    if (t->slot) return t->slot->state == EC_SLOT_DONE ? UCC_OK : UCC_INPROGRESS;
    e = cudaEventQuery(t->event);
    if (e == cudaErrorNotReady) { (void)cudaGetLastError(); return UCC_INPROGRESS; }
    return ucc_cuda_error_to_status(e);
}
static ucc_status_t exec_task_finalize(ucc_ee_executor_task_t *te)
{
    ucc_ec_cuda_task_t *t = (ucc_ec_cuda_task_t *)te;
    if (t->slot) t->slot->state = EC_SLOT_FREE;
    if (t->super.handle) ucc_mpool_put(t->super.handle);
    ucc_mpool_put(t);
    return UCC_OK;
}

ucc_ec_cuda_t ucc_ec_cuda = {
    .super = {.super = {.name = "cuda", .score = 2}, .ref_cnt = 0, .type = UCC_EE_CUDA_STREAM,
              .config_table = {"CUDA execution component", "EC_CUDA_", ucc_ec_cuda_config_table, sizeof(ucc_ec_cuda_config_t), {NULL, NULL}},
              .init = ec_cuda_init, .get_attr = ec_cuda_get_attr, .finalize = ec_cuda_finalize,
              .ops = {ev_create, ev_destroy, ev_post, ev_test},
              .executor_ops = {exec_init, exec_status, exec_start, exec_stop, exec_finalize, exec_task_post, exec_task_test, exec_task_finalize}}};
static void UCC_CTOR ec_cuda_cfg_register(void) { ucc_config_table_register(&ucc_ec_cuda.super.config_table); }
