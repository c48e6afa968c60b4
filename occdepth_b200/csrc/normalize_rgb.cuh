// Image pre-processing of the datasets (data/semantic_kitti/kitti_dataset.py:372-403, same in data/NYU): PIL RGB
// uint8 -> `np.array(img, float32) / 255.0` -> crop to (img_H, img_W) -> ToTensor (HWC -> CHW) ->
// Normalize(mean, std) = (x - mean) / std, all in float32 with IEEE rounding.  One thread per output pixel;
// __host__ __device__ bodies (tests/host_emul/ runs them on the CPU against torchvision / numpy, bit for bit).
#pragma once
#include <string.h>
#include "common.cuh"

namespace nrm {

#define NRM_HD __host__ __device__ __forceinline__

struct Args {
  const unsigned char* in;  // [H0][W0][3] RGB, row stride W0 * 3
  float* out;               // [3][H][W]
  int W0, H, W;
  float mean[3], stdv[3];
};

NRM_HD float sub_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
NRM_HD float div_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}

// one channel value: (u8 / 255 - mean) / std in float32
NRM_HD float normalize1(unsigned char u, float mean, float stdv) {
  return div_rn(sub_rn(div_rn((float)u, 255.0f), mean), stdv);
}

NRM_HD void body(const Args& a, long long i) {
  const int x = (int)(i % a.W), y = (int)(i / a.W);
  const unsigned char* p = a.in + ((long long)y * a.W0 + x) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) a.out[((long long)c * a.H + y) * a.W + x] = normalize1(p[c], a.mean[c], a.stdv[c]);
}

// ---- the forward's input staging: n uint8 images -> channels-last [n][H][W][cstride] of the activation type ----
// The values are those of occd_planar_to_cl(body(...)): normalize1, then TF32 (cvt.rna) or bf16 (round to nearest
// even) rounding; channels [3, cstride) are written as zeros.
struct StageArgs {
  const unsigned char* in;        // image 0, pixel (0, 0), channel 0
  long long img_stride, row_stride;  // bytes between images / rows; pixels are 3 contiguous bytes
  void* out;                      // [n][H][W][cstride], float (TF32 values) or __nv_bfloat16
  int H, W, cstride;
  float mean[3], stdv[3];
};

// cvt.rna.tf32.f32: round the 13 dropped mantissa bits to nearest, ties away from zero (finite inputs)
NRM_HD float tf32_rna(float v) {
#ifdef __CUDA_ARCH__
  return round_tf32(v);
#else
  uint32_t u;
  memcpy(&u, &v, 4);
  u = (u + 0x1000u) & ~0x1fffu;
  float r;
  memcpy(&r, &u, 4);
  return r;
#endif
}

template <typename OT> NRM_HD OT to_act(float v);
template <> NRM_HD float to_act<float>(float v) { return tf32_rna(v); }
template <> NRM_HD __nv_bfloat16 to_act<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// i: output pixel over [n][H][W]
template <typename OT>
NRM_HD void stage_body(const StageArgs& a, long long i) {
  const long long hw = (long long)a.H * a.W;
  const long long img = i / hw, r = i - img * hw;
  const long long y = r / a.W, x = r - y * a.W;
  const unsigned char* p = a.in + img * a.img_stride + y * a.row_stride + x * 3;
  OT* o = static_cast<OT*>(a.out) + i * a.cstride;
  float v[8];
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = normalize1(p[c], a.mean[c], a.stdv[c]);
#pragma unroll
  for (int c = 3; c < 8; ++c) v[c] = 0.f;
#ifdef __CUDA_ARCH__
  // cstride is a multiple of 8: one 8-channel vector per store
  if constexpr (sizeof(OT) == 2) {
    *reinterpret_cast<uint4*>(o) = pack8(v);
    for (int c = 8; c < a.cstride; c += 8) *reinterpret_cast<uint4*>(o + c) = make_uint4(0, 0, 0, 0);
  } else {
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = round_tf32(v[c]);
    st256_f(reinterpret_cast<float*>(o), v);
    const float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int c = 8; c < a.cstride; c += 8) st256_f(reinterpret_cast<float*>(o + c), z);
  }
#else
  for (int c = 0; c < a.cstride; ++c) o[c] = to_act<OT>(c < 8 ? v[c] : 0.f);
#endif
}

// NYU's load_depth (data/NYU/nyu_dataset.py:42-48): (u16 / divisor) in float64, rounded to float32, clamped to
// [0, max_depth] in float32
NRM_HD float depth_u16(unsigned short u, double divisor, float max_depth) {
  float d = (float)((double)u / divisor);
  if (d > max_depth) d = max_depth;
  if (d < 0.f) d = 0.f;
  return d;
}

#ifdef __CUDACC__
__global__ void __launch_bounds__(256) normalize_rgb_kernel(const Args a, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) body(a, i);
}

template <typename OT>
__global__ void __launch_bounds__(256) stage_rgb_kernel(const StageArgs a, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) stage_body<OT>(a, i);
}

__global__ void __launch_bounds__(256) depth_u16_kernel(const unsigned short* __restrict__ in, float* __restrict__ out,
                                                        long long n, double divisor, float max_depth) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = depth_u16(in[i], divisor, max_depth);
}
#endif

}  // namespace nrm
