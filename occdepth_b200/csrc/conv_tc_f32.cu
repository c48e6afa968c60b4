// The per-tap and x-packed per-tap kernels (conv_tc_kernel), TF32, one per compiled N tile.
#include "conv_kernels.cuh"

namespace occd_conv {
template int run_tc_family<float>(const occd_conv_plan*, cudaStream_t);
}  // namespace occd_conv
