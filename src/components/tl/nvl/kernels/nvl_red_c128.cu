/* tl/nvl reduction kernels instantiated for complex double */
#include "nvl_reduce_impl.cuh"
NVL_INSTANTIATE_REDUCE(nvl_c128, c128)
