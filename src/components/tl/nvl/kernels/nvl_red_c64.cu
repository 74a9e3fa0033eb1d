/* tl/nvl reduction kernels instantiated for complex float */
#include "nvl_reduce_impl.cuh"
NVL_INSTANTIATE_REDUCE(nvl_c64, c64)
