/* tl/nvl reduction kernels instantiated for int128 */
#include "nvl_reduce_impl.cuh"
NVL_INSTANTIATE_REDUCE(nvl_i128, i128)
