// Data-pipeline kernels (SURVEY 8f row 2).
// occd_vox2pix_fwd: the data pipeline's voxel -> pixel index generation on the device (SURVEY 8f row 2);
// occd_vox2pix_range_fwd: one window of the same voxel order (a rank's X-slab under the slab partition).
// replaces occdepth/data/utils/helpers.py:94-169 (vox2pix) as called per view and per scale by the datasets
// (data/semantic_kitti/kitti_dataset.py, data/NYU/nyu_dataset.py).
#include <stdio.h>
#include "vox2pix.cuh"
#include "normalize_rgb.cuh"
#include "../../include/occdepth_b200.h"

namespace {

template <typename T>
int run(const void* cam_E, const float* cam_k, const float* vox_origin, double voxel_size, int X, int Y, int Z,
        int img_W, int img_H, const int* pattern, int P, long long* pix, unsigned char* fov, void* pix_z,
        long long v0, long long n, cudaStream_t st) {
  v2p::Args<T> a;
  for (int i = 0; i < 12; ++i) a.E[i] = static_cast<const T*>(cam_E)[i];
  a.fx = cam_k[0]; a.fy = cam_k[4]; a.cx = cam_k[2]; a.cy = cam_k[5];
  for (int i = 0; i < 3; ++i) a.origin[i] = vox_origin[i];
  a.voxel_size = voxel_size;
  a.X = X; a.Y = Y; a.Z = Z; a.W = img_W; a.H = img_H; a.P = P;
  for (int p = 0; p < P; ++p) { a.pat[p][0] = pattern[2 * p]; a.pat[p][1] = pattern[2 * p + 1]; }
  a.pix = pix; a.fov = fov; a.pix_z = static_cast<T*>(pix_z);
  a.v0 = v0;
  v2p::vox2pix_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, n);
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

// voxels [v0, v0 + n) of the X*Y*Z grid; `who` names the entry point in the refusals
int vox2pix_window(const char* who, const void* cam_E, int pose_is_f32, const float* cam_k, const float* vox_origin,
                   double voxel_size, int X, int Y, int Z, int img_W, int img_H, const int* pattern, int P,
                   long long* pix, unsigned char* fov, void* pix_z, long long v0, long long n, void* stream) {
  auto refuse = [&](const char* what) {
    char msg[160];                        // occd_set_last_error keeps a copy
    snprintf(msg, sizeof msg, "%s: %s", who, what);
    occd_set_last_error(msg);
    return OCCD_ERR_ARG;
  };
  if (!(cam_E && cam_k && vox_origin && pattern && fov)) return refuse("null argument");  // pix may be NULL
  if (!(X > 0 && Y > 0 && Z > 0 && img_W > 0 && img_H > 0 && voxel_size > 0)) return refuse("dims");
  if (!(P >= 1 && P <= v2p::kMaxPattern)) return refuse("pattern size must be 1..25");
  const long long N = (long long)X * Y * Z;
  if (!(v0 >= 0 && n >= 1 && v0 <= N - n)) return refuse("the window [v0, v0 + n) must lie inside the X*Y*Z grid");
  if ((n + 255) / 256 > 2147483647LL) return refuse("too many voxels");
  cudaStream_t st = (cudaStream_t)stream;
  return pose_is_f32 ? run<float>(cam_E, cam_k, vox_origin, voxel_size, X, Y, Z, img_W, img_H, pattern, P, pix, fov,
                                  pix_z, v0, n, st)
                     : run<double>(cam_E, cam_k, vox_origin, voxel_size, X, Y, Z, img_W, img_H, pattern, P, pix, fov,
                                   pix_z, v0, n, st);
}

}  // namespace

extern "C" int occd_vox2pix_fwd(const void* cam_E, int pose_is_f32, const float* cam_k, const float* vox_origin,
                                double voxel_size, int X, int Y, int Z, int img_W, int img_H, const int* pattern,
                                int P, long long* pix, unsigned char* fov, void* pix_z, void* stream) {
  const long long N = X > 0 && Y > 0 && Z > 0 ? (long long)X * Y * Z : 1;
  return vox2pix_window("occd_vox2pix_fwd", cam_E, pose_is_f32, cam_k, vox_origin, voxel_size, X, Y, Z, img_W, img_H,
                        pattern, P, pix, fov, pix_z, 0, N, stream);
}

extern "C" int occd_vox2pix_range_fwd(const void* cam_E, int pose_is_f32, const float* cam_k,
                                      const float* vox_origin, double voxel_size, int X, int Y, int Z, int img_W,
                                      int img_H, const int* pattern, int P, long long* pix, unsigned char* fov,
                                      void* pix_z, long long v0, long long n, void* stream) {
  return vox2pix_window("occd_vox2pix_range_fwd", cam_E, pose_is_f32, cam_k, vox_origin, voxel_size, X, Y, Z, img_W,
                        img_H, pattern, P, pix, fov, pix_z, v0, n, stream);
}

// occd_normalize_rgb_u8: uint8 HWC image -> cropped, normalised float32 CHW (the datasets' `normalize_rgb`,
// data/semantic_kitti/kitti_dataset.py:164-171,376-402)
extern "C" int occd_normalize_rgb_u8(const void* in, float* out, int H0, int W0, int H, int W, const float* mean,
                                     const float* stdv, void* stream) {
  OCCD_CHECK_ARG(in && out && mean && stdv, "occd_normalize_rgb_u8: null argument");
  OCCD_CHECK_ARG(H > 0 && W > 0 && H <= H0 && W <= W0, "occd_normalize_rgb_u8: the crop must lie inside the image");
  nrm::Args a;
  a.in = (const unsigned char*)in; a.out = out; a.W0 = W0; a.H = H; a.W = W;
  for (int c = 0; c < 3; ++c) { a.mean[c] = mean[c]; a.stdv[c] = stdv[c]; }
  const long long total = (long long)H * W;
  nrm::normalize_rgb_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, total);
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

namespace {

// the staging launcher of every pixel format; `who` names the entry point in the refusals
template <int FMT, bool MAPS>
int stage_camera(const char* who, const void* in, long long img_stride, long long row_stride, long long uv_offset,
                 int n, int H0, int W0, int H, int W, const float* maps, long long map_stride, const float* mean,
                 const float* stdv, void* out, int out_dtype, int cstride, void* stream) {
  auto refuse = [&](const char* what) {
    char msg[160];
    snprintf(msg, sizeof msg, "%s: %s", who, what);
    occd_set_last_error(msg);
    return OCCD_ERR_ARG;
  };
  if (!(in && out && mean && stdv)) return refuse("null argument");
  if (!(n > 0 && H > 0 && W > 0 && H0 > 0 && W0 > 0 && (MAPS || (H <= H0 && W <= W0))))
    return refuse("the crop must lie inside the image");
  if (FMT == nrm::PIX_NV12) {
    if (H0 % 2 || W0 % 2) return refuse("an NV12 image has an even height and width");
    // luma rows [0, H0), then H0 / 2 chroma rows of W0 bytes from uv_offset
    const long long luma = (long long)(H0 - 1) * row_stride + W0, chroma = (long long)(H0 / 2 - 1) * row_stride + W0;
    if (!(row_stride >= W0 && uv_offset >= luma && (n == 1 || img_stride >= uv_offset + chroma)))
      return refuse("the chroma plane overlaps the luma rows, or the strides overlap the rows / images");
  } else if (!(row_stride >= 3LL * W0 && (n == 1 || img_stride >= (long long)(H0 - 1) * row_stride + 3LL * W0))) {
    return refuse("strides overlap the rows / images");
  }
  if (MAPS) {
    if (reinterpret_cast<uintptr_t>(maps) % 4 != 0) return refuse("maps must be 4-byte aligned float32");
    if (!(n == 1 || map_stride >= 2LL * H * W)) return refuse("map_stride overlaps the images' maps");
    if (H0 >= 32767 || W0 >= 32767) return refuse("a remapped image is under 32767 pixels a side");
  }
  if (!(cstride >= 8 && cstride % 8 == 0)) return refuse("cstride must be a multiple of 8");
  if (reinterpret_cast<uintptr_t>(out) % 16 != 0) return refuse("out must be 16-byte aligned");
  nrm::StageArgs a;
  a.in = (const unsigned char*)in; a.img_stride = img_stride; a.row_stride = row_stride;
  a.out = out; a.H = H; a.W = W; a.cstride = cstride;
  for (int c = 0; c < 3; ++c) { a.mean[c] = mean[c]; a.stdv[c] = stdv[c]; }
  a.uv_offset = uv_offset; a.H0 = H0; a.W0 = W0; a.maps = maps; a.map_stride = map_stride;
  const long long total = (long long)n * H * W;
  if ((total + 255) / 256 > 2147483647LL) return refuse("too many pixels");
  const unsigned grid = (unsigned)((total + 255) / 256);
  cudaStream_t st = (cudaStream_t)stream;
  if (out_dtype == OCCD_DTYPE_BF16) nrm::stage_camera_kernel<__nv_bfloat16, FMT, MAPS><<<grid, 256, 0, st>>>(a, total);
  else if (out_dtype == OCCD_DTYPE_F32) nrm::stage_camera_kernel<float, FMT, MAPS><<<grid, 256, 0, st>>>(a, total);
  else return refuse("dtype");
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

}  // namespace

// occd_stage_rgb_u8_cl: n uint8 HWC images -> the forward's channels-last input [n][H][W][cstride], equal to
// occd_planar_to_cl(occd_normalize_rgb_u8(image)) in one pass
extern "C" int occd_stage_rgb_u8_cl(const void* in, long long img_stride, long long row_stride, int n, int H0, int W0,
                                    int H, int W, const float* mean, const float* stdv, void* out, int out_dtype,
                                    int cstride, void* stream) {
  return stage_camera<nrm::PIX_RGB, false>("occd_stage_rgb_u8_cl", in, img_stride, row_stride, 0, n, H0, W0, H, W,
                                           nullptr, 0, mean, stdv, out, out_dtype, cstride, stream);
}

// occd_stage_camera_u8_cl: the same staging of RGB, BGR or NV12 images, optionally rectified by per-image maps
extern "C" int occd_stage_camera_u8_cl(const void* in, int format, long long img_stride, long long row_stride,
                                       long long uv_offset, int n, int H0, int W0, int H, int W, const float* maps,
                                       long long map_stride, const float* mean, const float* stdv, void* out,
                                       int out_dtype, int cstride, void* stream) {
  static const char* who = "occd_stage_camera_u8_cl";
#define OCCD_STAGE_FMT(F)                                                                                           \
  return maps ? stage_camera<F, true>(who, in, img_stride, row_stride, uv_offset, n, H0, W0, H, W, maps, map_stride, \
                                      mean, stdv, out, out_dtype, cstride, stream)                                 \
              : stage_camera<F, false>(who, in, img_stride, row_stride, uv_offset, n, H0, W0, H, W, nullptr, 0,    \
                                       mean, stdv, out, out_dtype, cstride, stream)
  switch (format) {
    case OCCD_PIX_RGB: OCCD_STAGE_FMT(nrm::PIX_RGB);
    case OCCD_PIX_BGR: OCCD_STAGE_FMT(nrm::PIX_BGR);
    case OCCD_PIX_NV12: OCCD_STAGE_FMT(nrm::PIX_NV12);
  }
#undef OCCD_STAGE_FMT
  occd_set_last_error("occd_stage_camera_u8_cl: format must be OCCD_PIX_RGB, OCCD_PIX_BGR or OCCD_PIX_NV12");
  return OCCD_ERR_ARG;
}

// occd_depth_u16_to_f32: NYU's load_depth (data/NYU/nyu_dataset.py:42-48) of a decoded uint16 depth PNG
extern "C" int occd_depth_u16_to_f32(const void* in, float* out, long long n, double divisor, float max_depth,
                                     void* stream) {
  OCCD_CHECK_ARG(in && out && n > 0 && divisor > 0, "occd_depth_u16_to_f32: bad args");
  OCCD_CHECK_ARG((n + 255) / 256 <= 2147483647LL, "occd_depth_u16_to_f32: too many pixels");
  nrm::depth_u16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (const unsigned short*)in, out, n, divisor, max_depth);
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}
