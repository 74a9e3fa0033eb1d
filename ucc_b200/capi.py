"""ctypes view of the UCC-compatible C API exported by ``libucc.so``.

Struct layouts mirror ``include/ucc/api/ucc.h`` field by field.  Nothing here
adds behaviour: it is the thinnest possible binding, used by the test
harness (:mod:`ucc_b200.harness`), the torch integration and ``bench.py``.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# UCC_B200_LIB points the binding at another build of the library (e.g. the ASAN one from `make asan`)
LIB_PATH = os.environ.get("UCC_B200_LIB") or os.path.join(_HERE, "lib", "libucc.so")


def _load():
    # PyTorch ships its own libnccl.so.2; let it map that copy first so the tl/nccl plugin re-uses it instead
    # of mapping the (older) system NCCL under the same soname
    try:
        import torch  # noqa: F401
    except Exception:
        pass
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `make -C {os.path.dirname(_HERE)}` "
            "or `python -c 'import __graft_entry__ as g; g.build()'`")
    return C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)


lib = _load()

# ----------------------------------------------------------------- enums
UCC_OK, UCC_INPROGRESS, UCC_OPERATION_INITIALIZED = 0, 1, 2
UCC_ERR_NOT_SUPPORTED, UCC_ERR_NOT_IMPLEMENTED, UCC_ERR_INVALID_PARAM = -1, -2, -3
UCC_ERR_NO_MEMORY, UCC_ERR_NO_RESOURCE, UCC_ERR_NO_MESSAGE, UCC_ERR_NOT_FOUND = -4, -5, -6, -7
UCC_ERR_TIMED_OUT, UCC_ERR_IO_ERROR, UCC_ERR_LAST = -8, -9, -100


def BIT(i):
    return 1 << i


COLL_NAMES = ["allgather", "allgatherv", "allreduce", "alltoall", "alltoallv", "barrier", "bcast", "fanin", "fanout",
              "gather", "gatherv", "reduce", "reduce_scatter", "reduce_scatterv", "scatter", "scatterv"]
COLL = {n: BIT(i) for i, n in enumerate(COLL_NAMES)}
(UCC_COLL_TYPE_ALLGATHER, UCC_COLL_TYPE_ALLGATHERV, UCC_COLL_TYPE_ALLREDUCE, UCC_COLL_TYPE_ALLTOALL,
 UCC_COLL_TYPE_ALLTOALLV, UCC_COLL_TYPE_BARRIER, UCC_COLL_TYPE_BCAST, UCC_COLL_TYPE_FANIN, UCC_COLL_TYPE_FANOUT,
 UCC_COLL_TYPE_GATHER, UCC_COLL_TYPE_GATHERV, UCC_COLL_TYPE_REDUCE, UCC_COLL_TYPE_REDUCE_SCATTER,
 UCC_COLL_TYPE_REDUCE_SCATTERV, UCC_COLL_TYPE_SCATTER, UCC_COLL_TYPE_SCATTERV) = [BIT(i) for i in range(16)]

(UCC_MEMORY_TYPE_HOST, UCC_MEMORY_TYPE_CUDA, UCC_MEMORY_TYPE_CUDA_MANAGED, UCC_MEMORY_TYPE_ROCM,
 UCC_MEMORY_TYPE_ROCM_MANAGED, UCC_MEMORY_TYPE_UNKNOWN) = range(6)

DT_NAMES = ["int8", "int16", "int32", "int64", "int128", "uint8", "uint16", "uint32", "uint64", "uint128",
            "float16", "float32", "float64", "bfloat16", "float128", "float32_complex", "float64_complex",
            "float128_complex"]
DT = {n: (i << 3) for i, n in enumerate(DT_NAMES)}
DT_SIZE = {"int8": 1, "int16": 2, "int32": 4, "int64": 8, "int128": 16, "uint8": 1, "uint16": 2, "uint32": 4,
           "uint64": 8, "uint128": 16, "float16": 2, "float32": 4, "float64": 8, "bfloat16": 2, "float128": 16,
           "float32_complex": 8, "float64_complex": 16, "float128_complex": 32}

OP_NAMES = ["sum", "prod", "max", "min", "land", "lor", "lxor", "band", "bor", "bxor", "maxloc", "minloc", "avg"]
OP = {n: i for i, n in enumerate(OP_NAMES)}

UCC_THREAD_SINGLE, UCC_THREAD_FUNNELED, UCC_THREAD_MULTIPLE = 0, 1, 2

UCC_LIB_PARAM_FIELD_THREAD_MODE = BIT(0)
UCC_CONTEXT_PARAM_FIELD_TYPE, UCC_CONTEXT_PARAM_FIELD_SYNC_TYPE, UCC_CONTEXT_PARAM_FIELD_OOB = BIT(0), BIT(1), BIT(2)
UCC_CONTEXT_ATTR_FIELD_CTX_ADDR, UCC_CONTEXT_ATTR_FIELD_CTX_ADDR_LEN, UCC_CONTEXT_ATTR_FIELD_WORK_BUFFER_SIZE = BIT(2), BIT(3), BIT(4)
(UCC_TEAM_PARAM_FIELD_ORDERING, UCC_TEAM_PARAM_FIELD_OUTSTANDING_COLLS, UCC_TEAM_PARAM_FIELD_EP,
 UCC_TEAM_PARAM_FIELD_EP_LIST, UCC_TEAM_PARAM_FIELD_EP_RANGE, UCC_TEAM_PARAM_FIELD_TEAM_SIZE,
 UCC_TEAM_PARAM_FIELD_SYNC_TYPE, UCC_TEAM_PARAM_FIELD_OOB, UCC_TEAM_PARAM_FIELD_P2P_CONN,
 UCC_TEAM_PARAM_FIELD_MEM_PARAMS, UCC_TEAM_PARAM_FIELD_EP_MAP, UCC_TEAM_PARAM_FIELD_ID,
 UCC_TEAM_PARAM_FIELD_FLAGS) = [BIT(i) for i in range(13)]
UCC_TEAM_ATTR_FIELD_EP, UCC_TEAM_ATTR_FIELD_SIZE = BIT(2), BIT(6)
UCC_COLLECTIVE_EP_RANGE_CONTIG = 0
UCC_EP_MAP_FULL, UCC_EP_MAP_STRIDED, UCC_EP_MAP_ARRAY, UCC_EP_MAP_CB = 1, 2, 3, 4

(UCC_COLL_ARGS_FLAG_IN_PLACE, UCC_COLL_ARGS_FLAG_PERSISTENT, UCC_COLL_ARGS_FLAG_COUNT_64BIT,
 UCC_COLL_ARGS_FLAG_DISPLACEMENTS_64BIT, UCC_COLL_ARGS_FLAG_CONTIG_SRC_BUFFER, UCC_COLL_ARGS_FLAG_CONTIG_DST_BUFFER,
 UCC_COLL_ARGS_FLAG_TIMEOUT, UCC_COLL_ARGS_FLAG_MEM_MAPPED_BUFFERS) = [BIT(i) for i in range(8)]
(UCC_COLL_ARGS_FIELD_FLAGS, UCC_COLL_ARGS_FIELD_TAG, UCC_COLL_ARGS_FIELD_CB, UCC_COLL_ARGS_FIELD_GLOBAL_WORK_BUFFER,
 UCC_COLL_ARGS_FIELD_ACTIVE_SET) = [BIT(i) for i in range(5)]
UCC_COLL_ARGS_FIELD_MEM_MAP_SRC_MEMH, UCC_COLL_ARGS_FIELD_MEM_MAP_DST_MEMH = BIT(5), BIT(6)
UCC_COLL_ARGS_FLAG_SRC_MEMH_GLOBAL, UCC_COLL_ARGS_FLAG_DST_MEMH_GLOBAL = BIT(8), BIT(9)
# hints in ucc_coll_args_t.flags (with UCC_COLL_ARGS_FIELD_FLAGS); tl/nvl honours OVERLAP_GPU (docs/user_guide.md)
(UCC_COLL_ARGS_HINT_OPTIMIZE_OVERLAP_CPU, UCC_COLL_ARGS_HINT_OPTIMIZE_OVERLAP_GPU,
 UCC_COLL_ARGS_HINT_OPTIMIZE_LATENCY) = BIT(24), BIT(25), BIT(26)

UCC_EE_CUDA_STREAM, UCC_EE_CPU_THREAD = 0, 1
UCC_EVENT_COLLECTIVE_POST, UCC_EVENT_COLLECTIVE_COMPLETE, UCC_EVENT_COMPUTE_COMPLETE = BIT(0), BIT(1), BIT(2)
UCC_MEM_MAP_MODE_EXPORT, UCC_MEM_MAP_MODE_IMPORT = 0, 1

# --------------------------------------------------------------- structs
ucc_status_t = C.c_int
handle = C.c_void_p

OOB_ALLGATHER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_void_p))
OOB_REQ_FN = C.CFUNCTYPE(C.c_int, C.c_void_p)
COLL_CB_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_int)


class ucc_lib_params_t(C.Structure):
    _fields_ = [("mask", C.c_uint64), ("thread_mode", C.c_int), ("coll_types", C.c_uint64),
                ("reduction_types", C.c_uint64), ("sync_type", C.c_int)]


class ucc_lib_attr_t(C.Structure):
    _fields_ = ucc_lib_params_t._fields_


class ucc_oob_coll_t(C.Structure):
    _fields_ = [("allgather", OOB_ALLGATHER_FN), ("req_test", OOB_REQ_FN), ("req_free", OOB_REQ_FN),
                ("coll_info", C.c_void_p), ("n_oob_eps", C.c_uint32), ("oob_ep", C.c_uint32)]


class ucc_mem_map_t(C.Structure):
    _fields_ = [("address", C.c_void_p), ("len", C.c_size_t)]


class ucc_mem_map_params_t(C.Structure):
    _fields_ = [("segments", C.POINTER(ucc_mem_map_t)), ("n_segments", C.c_uint64)]


class ucc_context_params_t(C.Structure):
    _fields_ = [("mask", C.c_uint64), ("type", C.c_int), ("sync_type", C.c_int), ("oob", ucc_oob_coll_t),
                ("ctx_id", C.c_uint64), ("mem_params", ucc_mem_map_params_t)]


class ucc_context_attr_t(C.Structure):
    _fields_ = [("mask", C.c_uint64), ("type", C.c_int), ("sync_type", C.c_int), ("ctx_addr", C.c_void_p),
                ("ctx_addr_len", C.c_size_t), ("global_work_buffer_size", C.c_uint64)]


class ucc_team_p2p_conn_t(C.Structure):
    _fields_ = [("conn_info_lookup", C.c_void_p), ("conn_info_release", C.c_void_p), ("conn_ctx", C.c_void_p),
                ("req_test", C.c_void_p), ("req_free", C.c_void_p)]


class _ep_map_strided(C.Structure):
    _fields_ = [("start", C.c_uint64), ("stride", C.c_int64)]


class _ep_map_array(C.Structure):
    _fields_ = [("map", C.c_void_p), ("elem_size", C.c_size_t)]


class _ep_map_cb(C.Structure):
    _fields_ = [("cb", C.c_void_p), ("cb_ctx", C.c_void_p)]


class _ep_map_u(C.Union):
    _fields_ = [("strided", _ep_map_strided), ("array", _ep_map_array), ("cb", _ep_map_cb)]


class ucc_ep_map_t(C.Structure):
    _anonymous_ = ("u",)
    _fields_ = [("type", C.c_int), ("ep_num", C.c_uint64), ("u", _ep_map_u)]


class ucc_team_params_t(C.Structure):
    _fields_ = [("mask", C.c_uint64), ("flags", C.c_uint64), ("ordering", C.c_int), ("outstanding_colls", C.c_uint64),
                ("ep", C.c_uint64), ("ep_list", C.POINTER(C.c_uint64)), ("ep_range", C.c_int), ("team_size", C.c_uint64),
                ("sync_type", C.c_int), ("oob", ucc_oob_coll_t), ("p2p_conn", ucc_team_p2p_conn_t),
                ("mem_params", ucc_mem_map_params_t), ("ep_map", ucc_ep_map_t), ("id", C.c_uint64)]


class ucc_team_attr_t(C.Structure):
    _fields_ = [("mask", C.c_uint64), ("ordering", C.c_int), ("outstanding_colls", C.c_uint64), ("ep", C.c_uint64),
                ("ep_range", C.c_int), ("sync_type", C.c_int), ("mem_params", ucc_mem_map_params_t),
                ("size", C.c_uint32), ("eps", C.POINTER(C.c_uint64))]


class ucc_coll_buffer_info_t(C.Structure):
    _fields_ = [("buffer", C.c_void_p), ("count", C.c_uint64), ("datatype", C.c_uint64), ("mem_type", C.c_int)]


class ucc_coll_buffer_info_v_t(C.Structure):
    _fields_ = [("buffer", C.c_void_p), ("counts", C.c_void_p), ("displacements", C.c_void_p),
                ("datatype", C.c_uint64), ("mem_type", C.c_int)]


class _buf_u(C.Union):
    _fields_ = [("info", ucc_coll_buffer_info_t), ("info_v", ucc_coll_buffer_info_v_t)]


class ucc_coll_callback_t(C.Structure):
    _fields_ = [("cb", COLL_CB_FN), ("data", C.c_void_p)]


class _active_set(C.Structure):
    _fields_ = [("start", C.c_uint64), ("stride", C.c_int64), ("size", C.c_uint64)]


class _memh_u(C.Union):
    _fields_ = [("local_memh", C.c_void_p), ("global_memh", C.POINTER(C.c_void_p))]


class ucc_coll_args_t(C.Structure):
    _fields_ = [("mask", C.c_uint64), ("coll_type", C.c_int), ("src", _buf_u), ("dst", _buf_u), ("op", C.c_int),
                ("flags", C.c_uint64), ("root", C.c_uint64), ("error_type", C.c_int), ("tag", C.c_uint16),
                ("global_work_buffer", C.c_void_p), ("cb", ucc_coll_callback_t), ("timeout", C.c_double),
                ("active_set", _active_set), ("src_memh", _memh_u), ("dst_memh", _memh_u)]


class ucc_coll_req_t(C.Structure):
    _fields_ = [("status", C.c_int)]


class ucc_ee_params_t(C.Structure):
    _fields_ = [("ee_type", C.c_int), ("ee_context", C.c_void_p), ("ee_context_size", C.c_size_t)]


class ucc_ev_t(C.Structure):
    _fields_ = [("ev_type", C.c_int), ("ev_context", C.c_void_p), ("ev_context_size", C.c_size_t), ("req", C.c_void_p)]


class ucc_proc_info_t(C.Structure):
    _fields_ = [("host_hash", C.c_uint64), ("socket_id", C.c_uint8), ("numa_id", C.c_uint8), ("host_id", C.c_uint64),
                ("pid", C.c_int)]


# ------------------------------------------------------------ prototypes
def _proto(name, restype, *argtypes):
    fn = getattr(lib, name)
    fn.restype = restype
    fn.argtypes = list(argtypes)
    return fn


ucc_status_string = _proto("ucc_status_string", C.c_char_p, C.c_int)
ucc_lib_config_read = _proto("ucc_lib_config_read", C.c_int, C.c_char_p, C.c_char_p, C.POINTER(handle))
ucc_lib_config_release = _proto("ucc_lib_config_release", None, handle)
ucc_lib_config_modify = _proto("ucc_lib_config_modify", C.c_int, handle, C.c_char_p, C.c_char_p)
ucc_init_version = _proto("ucc_init_version", C.c_int, C.c_uint, C.c_uint, C.POINTER(ucc_lib_params_t), handle, C.POINTER(handle))
ucc_finalize = _proto("ucc_finalize", C.c_int, handle)
ucc_lib_get_attr = _proto("ucc_lib_get_attr", C.c_int, handle, C.POINTER(ucc_lib_attr_t))
ucc_get_version_string = _proto("ucc_get_version_string", C.c_char_p)
ucc_context_config_read = _proto("ucc_context_config_read", C.c_int, handle, C.c_char_p, C.POINTER(handle))
ucc_context_config_release = _proto("ucc_context_config_release", None, handle)
ucc_context_config_modify = _proto("ucc_context_config_modify", C.c_int, handle, C.c_char_p, C.c_char_p, C.c_char_p)
ucc_context_create = _proto("ucc_context_create", C.c_int, handle, C.POINTER(ucc_context_params_t), handle, C.POINTER(handle))
ucc_context_create_proc_info = _proto("ucc_context_create_proc_info", C.c_int, handle, C.POINTER(ucc_context_params_t),
                                      handle, C.POINTER(handle), C.POINTER(ucc_proc_info_t))
ucc_context_progress = _proto("ucc_context_progress", C.c_int, handle)
ucc_context_destroy = _proto("ucc_context_destroy", C.c_int, handle)
ucc_context_get_attr = _proto("ucc_context_get_attr", C.c_int, handle, C.POINTER(ucc_context_attr_t))
ucc_team_create_post = _proto("ucc_team_create_post", C.c_int, C.POINTER(handle), C.c_uint32, C.POINTER(ucc_team_params_t), C.POINTER(handle))
ucc_team_create_test = _proto("ucc_team_create_test", C.c_int, handle)
ucc_team_destroy = _proto("ucc_team_destroy", C.c_int, handle)
ucc_team_get_attr = _proto("ucc_team_get_attr", C.c_int, handle, C.POINTER(ucc_team_attr_t))
ucc_collective_init = _proto("ucc_collective_init", C.c_int, C.POINTER(ucc_coll_args_t), C.POINTER(C.POINTER(ucc_coll_req_t)), handle)
ucc_collective_post = _proto("ucc_collective_post", C.c_int, C.POINTER(ucc_coll_req_t))
ucc_collective_finalize = _proto("ucc_collective_finalize", C.c_int, C.POINTER(ucc_coll_req_t))
ucc_collective_init_and_post = _proto("ucc_collective_init_and_post", C.c_int, C.POINTER(ucc_coll_args_t), C.POINTER(C.POINTER(ucc_coll_req_t)), handle)
ucc_collective_triggered_post = _proto("ucc_collective_triggered_post", C.c_int, handle, C.POINTER(ucc_ev_t))
ucc_ee_create = _proto("ucc_ee_create", C.c_int, handle, C.POINTER(ucc_ee_params_t), C.POINTER(handle))
ucc_ee_destroy = _proto("ucc_ee_destroy", C.c_int, handle)
ucc_ee_get_event = _proto("ucc_ee_get_event", C.c_int, handle, C.POINTER(C.POINTER(ucc_ev_t)))
ucc_ee_ack_event = _proto("ucc_ee_ack_event", C.c_int, handle, C.POINTER(ucc_ev_t))
ucc_ee_set_event = _proto("ucc_ee_set_event", C.c_int, handle, C.POINTER(ucc_ev_t))
ucc_dt_create_generic = _proto("ucc_dt_create_generic", C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64))
ucc_dt_destroy = _proto("ucc_dt_destroy", None, C.c_uint64)

UCC_API_MAJOR, UCC_API_MINOR = 1, 9


def status_str(st):
    return ucc_status_string(st).decode()


class UccError(RuntimeError):
    def __init__(self, st, what=""):
        self.status = st
        super().__init__(f"{what}: {status_str(st)} ({st})")


def check(st, what=""):
    if st < 0:
        raise UccError(st, what)
    return st
