/* ec/cuda device code interface (sm_90a): reduce / strided reduce / multi-dst reduce /
 * copy / multi copy kernels, the persistent executor kernel and the wait kernel
 * (capabilities of reference ec/cuda/kernel/*.cu, K6-K11 in SURVEY.md §2.10). */
#ifndef UCC_EC_CUDA_KERNELS_H_
#define UCC_EC_CUDA_KERNELS_H_
#include <stdint.h>
#include <stddef.h>
#include <cuda_runtime_api.h>

#define EC_MAX_SRCS 16
#define EC_MULTI_BUFS 7
typedef enum { EC_DT_I8, EC_DT_I16, EC_DT_I32, EC_DT_I64, EC_DT_U8, EC_DT_U16, EC_DT_U32, EC_DT_U64, EC_DT_F16, EC_DT_F32, EC_DT_F64,
               EC_DT_BF16, EC_DT_C64, EC_DT_C128, EC_DT_I128, EC_DT_U128, EC_DT_LAST } ec_dt_t;
typedef enum { EC_OP_SUM, EC_OP_PROD, EC_OP_MAX, EC_OP_MIN, EC_OP_LAND, EC_OP_LOR, EC_OP_LXOR, EC_OP_BAND, EC_OP_BOR, EC_OP_BXOR, EC_OP_LAST } ec_op_t;
typedef enum { EC_TASK_NONE, EC_TASK_REDUCE, EC_TASK_REDUCE_MULTI_DST, EC_TASK_COPY, EC_TASK_COPY_MULTI } ec_task_kind_t;

typedef struct ec_reduce_args {
    void       *dst;
    const void *srcs[EC_MAX_SRCS];   /* plain form */
    const void *src2;                /* strided form: srcs[0] + src2 + k*stride, k < n_srcs-1 */
    size_t      stride;
    int         strided, n_srcs;
    size_t      count;
    int         dt, op, with_alpha;
    int         avg_n;               /* alpha == 1.0 / avg_n exactly (AVG): integer types divide by it; 0: scale by alpha */
    double      alpha;
} ec_reduce_args_t;
typedef struct ec_reduce_multi_dst_args {
    void *dst[EC_MULTI_BUFS]; const void *src1[EC_MULTI_BUFS], *src2[EC_MULTI_BUFS]; size_t counts[EC_MULTI_BUFS]; int n_bufs, dt, op;
} ec_reduce_multi_dst_args_t;
typedef struct ec_copy_multi_args { void *dst[EC_MULTI_BUFS]; const void *src[EC_MULTI_BUFS]; size_t bytes[EC_MULTI_BUFS]; int n; } ec_copy_multi_args_t;

/* one slot of the persistent executor's task ring (lives in host-pinned, device-mapped memory) */
typedef enum { EC_SLOT_FREE = 0, EC_SLOT_POSTED = 1, EC_SLOT_DONE = 2 } ec_slot_state_t;
typedef struct ec_ring_slot {
    volatile uint32_t state;
    uint32_t          kind;
    volatile uint32_t seq;           /* global index of the task in the slot, written before state becomes POSTED */
    uint32_t          pad;
    union { ec_reduce_args_t reduce; ec_reduce_multi_dst_args_t rmd; ec_copy_multi_args_t copy; } u;
} ec_ring_slot_t;
typedef struct ec_ring { volatile uint32_t shutdown; volatile uint32_t started; uint32_t n_slots; uint32_t pad; ec_ring_slot_t slots[1]; } ec_ring_t;

#ifdef __cplusplus
extern "C" {
#endif
int         ec_dt_supports_op(int dt, int op);
size_t      ec_dt_size(int dt);
cudaError_t ec_launch_reduce(const ec_reduce_args_t *a, int nblocks, int nthreads, cudaStream_t s);
cudaError_t ec_launch_reduce_multi_dst(const ec_reduce_multi_dst_args_t *a, int nthreads, cudaStream_t s);
cudaError_t ec_launch_copy_multi(const ec_copy_multi_args_t *a, int nthreads, cudaStream_t s);
cudaError_t ec_launch_persistent(ec_ring_t *ring_dev, int nworkers, int nthreads, int cooperative, cudaStream_t s);
cudaError_t ec_launch_wait(volatile uint32_t *state_dev, cudaStream_t s); /* blocks the stream until *state != 0 */
#ifdef __cplusplus
}
#endif
#endif
