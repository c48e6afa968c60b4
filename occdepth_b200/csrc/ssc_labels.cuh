// Decoding of semantic scene completion labels, shared by the metrics (metrics.cu) and the loss sums (losses.cu).
// Labels arrive as float32 (KITTI targets), uint8 (NYU targets) or int64; 255 means "ignore".
#pragma once
#include <stdint.h>

namespace ssc_labels {

constexpr int kIgnore = -1, kInvalid = -2;

// label -> class in [0, C), kIgnore (255) or kInvalid (anything else, including a float that is not an integer)
__device__ __forceinline__ int label_class(uint8_t v, int C) { return v == 255 ? kIgnore : (v < C ? (int)v : kInvalid); }
__device__ __forceinline__ int label_class(long long v, int C) {
  return v == 255 ? kIgnore : ((unsigned long long)v < (unsigned long long)C ? (int)v : kInvalid);
}
__device__ __forceinline__ int label_class(float v, int C) {
  return v == 255.f ? kIgnore : ((v >= 0.f && v < (float)C && v == truncf(v)) ? (int)v : kInvalid);  // NaN: invalid
}

}  // namespace ssc_labels
