/* tl/nvl reduction kernels instantiated for uint128 */
#include "nvl_reduce_impl.cuh"
NVL_INSTANTIATE_REDUCE(nvl_u128, u128)
