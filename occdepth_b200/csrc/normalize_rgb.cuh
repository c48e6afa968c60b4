// Image pre-processing of the datasets (data/semantic_kitti/kitti_dataset.py:372-403, same in data/NYU): PIL RGB
// uint8 -> `np.array(img, float32) / 255.0` -> crop to (img_H, img_W) -> ToTensor (HWC -> CHW) ->
// Normalize(mean, std) = (x - mean) / std, all in float32 with IEEE rounding.  One thread per output pixel;
// __host__ __device__ bodies (tests/host_emul/ runs them on the CPU against torchvision / numpy, bit for bit).
#pragma once
#include <math.h>
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
// even) rounding; channels [3, cstride) are written as zeros.  The camera formats (occd_stage_camera_u8_cl) first
// make the RGB pixel OpenCV would: cv::cvtColor (COLOR_BGR2RGB, COLOR_YUV2RGB_NV12), and with maps then cv::remap
// (INTER_LINEAR, BORDER_CONSTANT 0) of the converted image, in OpenCV's fixed-point arithmetic.
enum { PIX_RGB = 0, PIX_BGR = 1, PIX_NV12 = 2 };  // OCCD_PIX_*

struct StageArgs {
  const unsigned char* in;        // image 0, pixel (0, 0), channel 0
  long long img_stride, row_stride;  // bytes between images / rows; RGB / BGR pixels are 3 contiguous bytes
  void* out;                      // [n][H][W][cstride], float (TF32 values) or __nv_bfloat16
  int H, W, cstride;
  float mean[3], stdv[3];
  // the camera formats only
  long long uv_offset;            // NV12: image i's interleaved U, V plane starts at in + i*img_stride + uv_offset
  int H0, W0;                     // raw size: a remap tap outside it reads 0
  const float* maps;              // [n][2][H][W] float32 (source x, then y) per output pixel; image i's at
  long long map_stride;           // maps + i*map_stride floats
};

// cv::remap's INTER_LINEAR table (imgproc initInterTab2D): per fraction cell (fy, fx) of 1/32 pixel the weights of the
// taps (y, x), (y, x+1), (y+1, x), (y+1, x+1), each rint(float32 weight * 32768); a sum other than 32768 is fixed on
// the largest (sum < 32768) or smallest (sum > 32768) tap.  Built at compile time, for the device's __constant__ copy
// and the host emulation alike.
struct RemapTab {
  unsigned short w[1024][4];
};

constexpr int rint_pos(float v) {  // round half to even, v >= 0
  const int f = (int)v;
  const float r = v - (float)f;
  return r > 0.5f || (r == 0.5f && (f & 1)) ? f + 1 : f;
}

constexpr RemapTab make_remap_tab() {
  RemapTab t{};
  for (int fy = 0; fy < 32; ++fy)
    for (int fx = 0; fx < 32; ++fx) {
      const float ty[2] = {1.f - fy * (1.f / 32), fy * (1.f / 32)}, tx[2] = {1.f - fx * (1.f / 32), fx * (1.f / 32)};
      int w[4] = {}, sum = 0, lo = 0, hi = 0;
      for (int k = 0; k < 4; ++k) {
        w[k] = rint_pos(ty[k >> 1] * tx[k & 1] * 32768.f);
        sum += w[k];
        if (w[k] < w[lo]) lo = k;
        if (w[k] > w[hi]) hi = k;
      }
      if (sum < 32768) w[hi] += 32768 - sum;
      if (sum > 32768) w[lo] -= sum - 32768;
      for (int k = 0; k < 4; ++k) t.w[fy * 32 + fx][k] = (unsigned short)w[k];
    }
  return t;
}

#ifdef __CUDACC__
static __constant__ RemapTab kRemapTabDev = make_remap_tab();
#endif
static constexpr RemapTab kRemapTabHost = make_remap_tab();

// cv::saturate_cast<int>(m * 32), OpenCV's rounding of a float map entry (half to even); NaN, +-inf and values beyond
// int give INT_MIN, as x86's cvtss2si does, so every tap of such an entry lands outside the image
NRM_HD int remap_fixed(float m) {
  const float s = m * 32.f;
  if (!(s >= -2147483648.f && s < 2147483648.f)) return (int)0x80000000u;
#ifdef __CUDA_ARCH__
  return __float2int_rn(s);
#else
  return (int)nearbyintf(s);
#endif
}

// OpenCV's YUV420sp2RGB (COLOR_YUV2RGB_NV12): BT.601 limited range in 20-bit fixed point
NRM_HD void nv12_to_rgb(int Y, int U, int V, int* rgb) {
  const int c = max(Y - 16, 0) * 1220542, u = U - 128, v = V - 128;
  rgb[0] = min(max((c + 1673527 * v + (1 << 19)) >> 20, 0), 255);
  rgb[1] = min(max((c - 852492 * v - 409993 * u + (1 << 19)) >> 20, 0), 255);
  rgb[2] = min(max((c + 2116026 * u + (1 << 19)) >> 20, 0), 255);
}

// the RGB colour of raw pixel (yy, xx) of the image at `img`
template <int FMT>
NRM_HD void rgb_at(const StageArgs& a, const unsigned char* img, long long yy, long long xx, int* rgb) {
  if constexpr (FMT == PIX_NV12) {
    const unsigned char* uv = img + a.uv_offset + (yy >> 1) * a.row_stride + (xx & ~1LL);
    nv12_to_rgb(img[yy * a.row_stride + xx], uv[0], uv[1], rgb);
  } else {
    const unsigned char* p = img + yy * a.row_stride + xx * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) rgb[c] = p[FMT == PIX_BGR ? 2 - c : c];
  }
}

// cv::remap of the converted image at output pixel (y, x) of image i: four taps, each converted before the weighting
template <int FMT>
NRM_HD void remap_at(const StageArgs& a, const unsigned char* img, long long i, long long y, long long x, int* rgb) {
  const float* m = a.maps + i * a.map_stride + y * a.W + x;
  const int X = remap_fixed(m[0]), Y = remap_fixed(m[(long long)a.H * a.W]);
#ifdef __CUDA_ARCH__
  const unsigned short* w = kRemapTabDev.w[(Y & 31) * 32 + (X & 31)];
#else
  const unsigned short* w = kRemapTabHost.w[(Y & 31) * 32 + (X & 31)];
#endif
  int acc[3] = {1 << 14, 1 << 14, 1 << 14};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int ty = (Y >> 5) + (k >> 1), tx = (X >> 5) + (k & 1);
    if (ty < 0 || ty >= a.H0 || tx < 0 || tx >= a.W0) continue;  // BORDER_CONSTANT: 0 in every channel
    int t[3];
    rgb_at<FMT>(a, img, ty, tx, t);
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] += (int)w[k] * t[c];
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) rgb[c] = min(max(acc[c] >> 15, 0), 255);
}

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

// i: output pixel over [n][H][W].  RGB without maps reads the pixel as the datasets' route does
template <typename OT, int FMT = PIX_RGB, bool MAPS = false>
NRM_HD void stage_body(const StageArgs& a, long long i) {
  const long long hw = (long long)a.H * a.W;
  const long long img = i / hw, r = i - img * hw;
  const long long y = r / a.W, x = r - y * a.W;
  float v[8];
  OT* o;
  if constexpr (FMT == PIX_RGB && !MAPS) {
    const unsigned char* p = a.in + img * a.img_stride + y * a.row_stride + x * 3;
    o = static_cast<OT*>(a.out) + i * a.cstride;
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = normalize1(p[c], a.mean[c], a.stdv[c]);
  } else {
    o = static_cast<OT*>(a.out) + i * a.cstride;
    int rgb[3];
    if constexpr (MAPS) remap_at<FMT>(a, a.in + img * a.img_stride, img, y, x, rgb);
    else rgb_at<FMT>(a, a.in + img * a.img_stride, y, x, rgb);
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = normalize1((unsigned char)rgb[c], a.mean[c], a.stdv[c]);
  }
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

template <typename OT, int FMT, bool MAPS>
__global__ void __launch_bounds__(256) stage_camera_kernel(const StageArgs a, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) stage_body<OT, FMT, MAPS>(a, i);
}

__global__ void __launch_bounds__(256) depth_u16_kernel(const unsigned short* __restrict__ in, float* __restrict__ out,
                                                        long long n, double divisor, float max_depth) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = depth_u16(in[i], divisor, max_depth);
}
#endif

}  // namespace nrm
