/* Execution component interface: events + executor (reduce / copy tasks).
 * Task vocabulary follows reference ec/base/ucc_ec_base.h:47-208 so TLs and
 * tests can express the same operations. */
#ifndef UCC_EC_BASE_H_
#define UCC_EC_BASE_H_
#include <ucc/api/ucc.h>
#include "utils/ucc_component.h"
#include "utils/ucc_parser.h"

typedef struct ucc_ec_params { ucc_thread_mode_t thread_mode; } ucc_ec_params_t;
typedef struct ucc_ec_attr { uint64_t field_mask; size_t max_executors_bufs; } ucc_ec_attr_t;
typedef struct ucc_ec_config { ucc_log_component_config_t log_component; } ucc_ec_config_t;
extern ucc_config_field_t ucc_ec_config_table[];

typedef struct ucc_ec_ops {
    ucc_status_t (*create_event)(void **event);
    ucc_status_t (*destroy_event)(void *event);
    ucc_status_t (*event_post)(void *ee_context, void *event);
    ucc_status_t (*event_test)(void *event);
} ucc_ec_ops_t;

typedef enum {
    UCC_EE_EXECUTOR_TASK_REDUCE = UCC_BIT(0),
    UCC_EE_EXECUTOR_TASK_REDUCE_STRIDED = UCC_BIT(1),
    UCC_EE_EXECUTOR_TASK_REDUCE_MULTI_DST = UCC_BIT(2),
    UCC_EE_EXECUTOR_TASK_COPY = UCC_BIT(3),
    UCC_EE_EXECUTOR_TASK_COPY_MULTI = UCC_BIT(4),
    UCC_EE_EXECUTOR_TASK_LAST = UCC_BIT(5)
} ucc_ee_executor_task_type_t;

#define UCC_EE_EXECUTOR_NUM_BUFS 9
#define UCC_EE_EXECUTOR_MULTI_OP_NUM_BUFS 7
#define UCC_EEE_TASK_FLAG_REDUCE_WITH_ALPHA UCC_BIT(0)
#define UCC_EEE_TASK_FLAG_REDUCE_SRCS_EXT   UCC_BIT(1)

/* AVG passes alpha = 1.0 / n for the n contributions it averages.  Returns that n when alpha is exactly 1.0 / n for an integer
 * n >= 1, else 0.  Integer types divide the sum by n (truncating): scaling by alpha in double drops the low bits of sums above 2^53. */
static inline int ucc_ec_avg_divisor(double alpha)
{
    int n;
    if (!(alpha > 0.0 && alpha <= 1.0) || 1.0 / alpha > 2147483647.0) return 0;
    n = (int)(1.0 / alpha + 0.5);
    return 1.0 / (double)n == alpha ? n : 0;
}

typedef struct ucc_ee_executor_params { uint64_t mask; ucc_ee_type_t ee_type; uint64_t task_types; } ucc_ee_executor_params_t;
enum { UCC_EE_EXECUTOR_PARAM_FIELD_TYPE = UCC_BIT(0), UCC_EE_EXECUTOR_PARAM_FIELD_TASK_TYPES = UCC_BIT(1) };
typedef struct ucc_ee_executor { ucc_ee_type_t ee_type; void *ee_context; } ucc_ee_executor_t;

typedef struct ucc_eee_task_reduce {
    void *dst;
    union { void *srcs[UCC_EE_EXECUTOR_NUM_BUFS]; void **srcs_ext; };
    size_t count; double alpha; ucc_datatype_t dt; ucc_reduction_op_t op; uint16_t n_srcs;
} ucc_eee_task_reduce_t;
typedef struct ucc_eee_task_reduce_strided {
    void *dst, *src1, *src2; size_t stride, count; double alpha; ucc_datatype_t dt; ucc_reduction_op_t op; uint16_t n_src2;
} ucc_eee_task_reduce_strided_t;
typedef struct ucc_eee_task_reduce_multi_dst {
    void *dst[UCC_EE_EXECUTOR_MULTI_OP_NUM_BUFS], *src1[UCC_EE_EXECUTOR_MULTI_OP_NUM_BUFS], *src2[UCC_EE_EXECUTOR_MULTI_OP_NUM_BUFS];
    size_t counts[UCC_EE_EXECUTOR_MULTI_OP_NUM_BUFS]; ucc_datatype_t dt; ucc_reduction_op_t op; uint16_t n_bufs;
} ucc_eee_task_reduce_multi_dst_t;
typedef struct ucc_eee_task_copy { void *dst; const void *src; size_t len; } ucc_eee_task_copy_t;
typedef struct ucc_eee_task_copy_multi {
    const void *src[UCC_EE_EXECUTOR_MULTI_OP_NUM_BUFS]; void *dst[UCC_EE_EXECUTOR_MULTI_OP_NUM_BUFS];
    size_t counts[UCC_EE_EXECUTOR_MULTI_OP_NUM_BUFS]; size_t num_vectors;
} ucc_eee_task_copy_multi_t;

typedef struct ucc_ee_executor_task_args {
    uint16_t task_type; uint16_t flags;
    union {
        ucc_eee_task_reduce_t reduce; ucc_eee_task_reduce_strided_t reduce_strided;
        ucc_eee_task_reduce_multi_dst_t reduce_multi_dst; ucc_eee_task_copy_t copy; ucc_eee_task_copy_multi_t copy_multi;
    };
} ucc_ee_executor_task_args_t;

typedef struct ucc_ee_executor_task {
    ucc_ee_executor_t          *eee;
    ucc_ee_executor_task_args_t args;
    ucc_status_t                status;
    void                       *handle;
} ucc_ee_executor_task_t;

typedef struct ucc_ee_executor_ops {
    ucc_status_t (*init)(const ucc_ee_executor_params_t *params, ucc_ee_executor_t **executor);
    ucc_status_t (*status)(const ucc_ee_executor_t *executor);
    ucc_status_t (*start)(ucc_ee_executor_t *executor, void *ee_context);
    ucc_status_t (*stop)(ucc_ee_executor_t *executor);
    ucc_status_t (*finalize)(ucc_ee_executor_t *executor);
    ucc_status_t (*task_post)(ucc_ee_executor_t *executor, const ucc_ee_executor_task_args_t *task_args, ucc_ee_executor_task_t **task);
    ucc_status_t (*task_test)(const ucc_ee_executor_task_t *task);
    ucc_status_t (*task_finalize)(ucc_ee_executor_task_t *task);
} ucc_ee_executor_ops_t;

typedef struct ucc_ec_base {
    ucc_component_iface_t          super;
    uint32_t                       ref_cnt;
    ucc_ee_type_t                  type;
    ucc_ec_config_t               *config;
    ucc_config_global_list_entry_t config_table;
    ucc_status_t (*init)(const ucc_ec_params_t *ec_params);
    ucc_status_t (*get_attr)(ucc_ec_attr_t *ec_attr);
    ucc_status_t (*finalize)(void);
    ucc_ec_ops_t                   ops;
    ucc_ee_executor_ops_t          executor_ops;
} ucc_ec_base_t;
#endif
