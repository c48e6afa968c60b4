// The halo-tile and x-packed halo-tile kernels (conv_halo_kernel, conv_halox_kernel), both element types,
// one per compiled N tile.
#include "conv_kernels.cuh"

namespace occd_conv {
template int run_halo_family<float>(const occd_conv_plan*, cudaStream_t);
template int run_halo_family<__nv_bfloat16>(const occd_conv_plan*, cudaStream_t);
}  // namespace occd_conv
