// Camera views of a class map: one ray per pixel through a uint16 class map, walked voxel by voxel (Amanatides-Woo,
// render.cuh) to the first voxel whose class is neither `empty` nor `ignore`, with its class, entry depth and element
// offset.  The visibility query under the views the visualisation scripts draw from, on maps that never leave the
// device.
//
// One thread per pixel, consecutive threads on consecutive u, so neighbouring rays walk neighbouring voxels; one
// block row per image row and grid.z over the B x V cameras, which travel by value in the kernel parameters (no
// host-to-device copy, so the launch captures into a CUDA graph).  Each thread writes only its own pixel: the same
// inputs give the same bytes.
//
// Soft views (occd_render_probs): the same walk over a float16 probability field, each ray composited front to back
// (render.cuh, composite_ray) into the class, expected depth, opacity and per-pixel channel distribution.  The C
// running sums stay in registers: instantiations for C <= 16, 32 and 64.  Blocks of 16 x 8 pixels: a KITTI field's
// probabilities (84 MB) do not stay in L2 as the class map does, and square tiles keep a block's rays on fewer
// lines of each class plane than one-row blocks (DESIGN section 7).
#include "render.cuh"
#include "../../include/occdepth_b200.h"

namespace {

constexpr int kThreads = 128;
constexpr int kMaxCameras = OCCD_RENDER_MAX_CAMERAS;

struct Cameras {
  rnd::Camera c[kMaxCameras];
};

__global__ void __launch_bounds__(kThreads) render_kernel(const uint16_t* __restrict__ map, long long N, int V, int W,
                                                          int H, const rnd::Grid g,
                                                          const __grid_constant__ Cameras cams,
                                                          uint16_t* __restrict__ cls, float* __restrict__ depth,
                                                          int32_t* __restrict__ index) {
  const int u = blockIdx.x * kThreads + threadIdx.x;
  if (u >= W) return;
  const int v = blockIdx.y, cam = blockIdx.z;
  const rnd::Hit h = rnd::cast_ray(cams.c[cam], g, map + (long long)(cam / V) * N, u, v);
  const long long p = ((long long)cam * H + v) * W + u;
  if (cls) cls[p] = (uint16_t)h.cls;
  if (depth) depth[p] = (float)h.t;
  if (index) index[p] = (int32_t)h.off;
}

constexpr int kMaxClasses = 64;
constexpr int kTileX = 16, kTileY = 8;

struct SoftParams {
  rnd::Camera c[kMaxCameras];
  uint16_t lut[kMaxClasses];
};

template <int CMAX>
__global__ void __launch_bounds__(kTileX * kTileY, CMAX <= 32 ? 4 : 3)
    render_probs_kernel(const __half* __restrict__ probs, const uint16_t* __restrict__ cmap, int C, long long N,
                        int V, int W, int H, float t_min, int use_lut, const rnd::Grid g,
                        const __grid_constant__ SoftParams prm, uint16_t* __restrict__ cls,
                        float* __restrict__ depth, float* __restrict__ opacity, __half* __restrict__ probs_out) {
  const int u = blockIdx.x * kTileX + threadIdx.x % kTileX;
  const int v = blockIdx.y * kTileY + threadIdx.x / kTileX;
  if (u >= W || v >= H) return;
  const int cam = blockIdx.z, b = cam / V;
  rnd::SoftIn in;
  in.probs = probs + (long long)b * C * N;
  in.cstride = N;
  in.cmap = cmap ? cmap + (long long)b * N : nullptr;
  in.C = C;
  in.t_min = t_min;
  in.lut = use_lut ? prm.lut : nullptr;
  const long long HW = (long long)H * W, p = (long long)cam * HW + (long long)v * W + u;
  rnd::composite_ray<CMAX>(prm.c[cam], g, in, u, v, cls ? cls + p : nullptr, depth ? depth + p : nullptr,
                           opacity ? opacity + p : nullptr,
                           probs_out ? probs_out + (long long)cam * C * HW + (long long)v * W + u : nullptr, HW);
}

bool finite_all(const double* a, int n) {
  for (int i = 0; i < n; ++i)
    if (!isfinite(a[i])) return false;
  return true;
}

}  // namespace

extern "C" int occd_render_classes(const uint16_t* class_map, int B, int GX, int GY, int GZ, const long long* strides,
                                   const double* origin, double voxel, int V, const double* cameras, int W, int H,
                                   int empty, int ignore, double near_t, double far_t, uint16_t* cls, float* depth,
                                   int32_t* index, void* stream) {
  OCCD_CHECK_ARG(class_map && strides && origin && cameras,
                 "occd_render_classes: class_map, strides, origin and cameras are required");
  OCCD_CHECK_ARG(cls || depth || index, "occd_render_classes: at least one of cls, depth and index is required");
  OCCD_CHECK_ARG(B >= 1 && V >= 1 && (long long)B * V <= kMaxCameras,
                 "occd_render_classes: B >= 1 maps with V >= 1 cameras each, at most 32 cameras per call");
  OCCD_CHECK_ARG(GX > 0 && GY > 0 && GZ > 0, "occd_render_classes: grid dims must be positive");
  const long long N = (long long)GX * GY * GZ;
  OCCD_CHECK_ARG(N <= 2147483647LL, "occd_render_classes: a map holds at most 2^31 - 1 voxels");
  OCCD_CHECK_ARG(strides[0] >= 0 && strides[0] <= N && strides[1] >= 0 && strides[1] <= N && strides[2] >= 0 &&
                     strides[2] <= N && (GX - 1) * strides[0] + (GY - 1) * strides[1] + (GZ - 1) * strides[2] < N,
                 "occd_render_classes: strides must be non-negative and keep every voxel inside its map");
  OCCD_CHECK_ARG(W > 0 && H > 0 && H <= 65535 && (long long)W * H <= 2147483647LL,
                 "occd_render_classes: W and H must be positive, H <= 65535 and W * H < 2^31");
  OCCD_CHECK_ARG(isfinite(voxel) && voxel > 0.0 && finite_all(origin, 3),
                 "occd_render_classes: voxel must be finite and positive, origin finite");
  OCCD_CHECK_ARG(finite_all(cameras, 12 * B * V), "occd_render_classes: cameras must be finite");
  OCCD_CHECK_ARG(empty >= 0 && empty <= 65535 && ignore >= 0 && ignore <= 65535,
                 "occd_render_classes: empty and ignore must be uint16 class ids");
  OCCD_CHECK_ARG(isfinite(near_t) && near_t >= 0.0 && far_t > near_t,
                 "occd_render_classes: near must be finite and >= 0, far > near");
  OCCD_CHECK_ARG((uintptr_t)class_map % 2 == 0 && (uintptr_t)cls % 2 == 0 && (uintptr_t)depth % 4 == 0 &&
                     (uintptr_t)index % 4 == 0,
                 "occd_render_classes: a pointer is not aligned to its element size");
  rnd::Grid g;
  for (int a = 0; a < 3; ++a) {
    g.origin[a] = origin[a];
    g.s[a] = strides[a];
  }
  g.voxel = voxel;
  g.G[0] = GX;
  g.G[1] = GY;
  g.G[2] = GZ;
  g.empty = empty;
  g.ignore = ignore;
  g.near_t = near_t;
  g.far_t = far_t;
  Cameras cams;
  for (int c = 0; c < kMaxCameras; ++c)
    for (int i = 0; i < 12; ++i) {
      const double x = c < B * V ? cameras[12 * c + i] : 0.0;
      if (i < 9)
        cams.c[c].M[i] = x;
      else
        cams.c[c].o[i - 9] = x;
    }
  const dim3 grid((unsigned)((W + kThreads - 1) / kThreads), (unsigned)H, (unsigned)(B * V));
  render_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(class_map, N, V, W, H, g, cams, cls, depth, index);
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

extern "C" int occd_render_probs(const void* probs, int B, int C, int GX, int GY, int GZ, const long long* strides,
                                 const uint16_t* class_map, int ignore, int empty, const double* origin, double voxel,
                                 int V, const double* cameras, int W, int H, double near_t, double far_t, float t_min,
                                 const int* lut, uint16_t* cls, float* depth, float* opacity, void* probs_out,
                                 void* stream) {
  OCCD_CHECK_ARG(probs && strides && origin && cameras,
                 "occd_render_probs: probs, strides, origin and cameras are required");
  OCCD_CHECK_ARG(cls || depth || opacity || probs_out,
                 "occd_render_probs: at least one of cls, depth, opacity and probs_out is required");
  OCCD_CHECK_ARG(B >= 1 && V >= 1 && (long long)B * V <= kMaxCameras,
                 "occd_render_probs: B >= 1 maps with V >= 1 cameras each, at most 32 cameras per call");
  OCCD_CHECK_ARG(C >= 1 && C <= kMaxClasses, "occd_render_probs: C must be in [1, 64]");
  OCCD_CHECK_ARG(empty >= 0 && empty < C, "occd_render_probs: empty must be a channel index below C");
  OCCD_CHECK_ARG(GX > 0 && GY > 0 && GZ > 0, "occd_render_probs: grid dims must be positive");
  const long long N = (long long)GX * GY * GZ;
  OCCD_CHECK_ARG(N <= 2147483647LL, "occd_render_probs: a map holds at most 2^31 - 1 voxels");
  OCCD_CHECK_ARG(strides[0] >= 0 && strides[0] <= N && strides[1] >= 0 && strides[1] <= N && strides[2] >= 0 &&
                     strides[2] <= N && (GX - 1) * strides[0] + (GY - 1) * strides[1] + (GZ - 1) * strides[2] < N,
                 "occd_render_probs: strides must be non-negative and keep every voxel inside its map");
  OCCD_CHECK_ARG(W > 0 && H > 0 && H <= 65535 && (long long)W * H <= 2147483647LL,
                 "occd_render_probs: W and H must be positive, H <= 65535 and W * H < 2^31");
  OCCD_CHECK_ARG(isfinite(voxel) && voxel > 0.0 && finite_all(origin, 3),
                 "occd_render_probs: voxel must be finite and positive, origin finite");
  OCCD_CHECK_ARG(finite_all(cameras, 12 * B * V), "occd_render_probs: cameras must be finite");
  OCCD_CHECK_ARG(ignore >= 0 && ignore <= 65535, "occd_render_probs: ignore must be a uint16 class id");
  OCCD_CHECK_ARG(isfinite(near_t) && near_t >= 0.0 && far_t > near_t,
                 "occd_render_probs: near must be finite and >= 0, far > near");
  OCCD_CHECK_ARG(t_min >= 0.f && t_min < 1.f, "occd_render_probs: t_min must be in [0, 1)");
  OCCD_CHECK_ARG((uintptr_t)probs % 2 == 0 && (uintptr_t)class_map % 2 == 0 && (uintptr_t)cls % 2 == 0 &&
                     (uintptr_t)depth % 4 == 0 && (uintptr_t)opacity % 4 == 0 && (uintptr_t)probs_out % 2 == 0,
                 "occd_render_probs: a pointer is not aligned to its element size");
  rnd::Grid g;
  for (int a = 0; a < 3; ++a) {
    g.origin[a] = origin[a];
    g.s[a] = strides[a];
  }
  g.voxel = voxel;
  g.G[0] = GX;
  g.G[1] = GY;
  g.G[2] = GZ;
  g.empty = empty;
  g.ignore = ignore;
  g.near_t = near_t;
  g.far_t = far_t;
  SoftParams prm;
  for (int c = 0; c < kMaxCameras; ++c)
    for (int i = 0; i < 12; ++i) {
      const double x = c < B * V ? cameras[12 * c + i] : 0.0;
      if (i < 9)
        prm.c[c].M[i] = x;
      else
        prm.c[c].o[i - 9] = x;
    }
  for (int c = 0; c < kMaxClasses; ++c) prm.lut[c] = (lut && c < C) ? (uint16_t)lut[c] : 0;  // .astype(np.uint16)
  const dim3 grid((unsigned)((W + kTileX - 1) / kTileX), (unsigned)((H + kTileY - 1) / kTileY), (unsigned)(B * V));
  cudaStream_t st = (cudaStream_t)stream;
  const __half* p = static_cast<const __half*>(probs);
  __half* po = static_cast<__half*>(probs_out);
#define RND_LAUNCH(CM)                                                                                              \
  render_probs_kernel<CM><<<grid, kTileX * kTileY, 0, st>>>(p, class_map, C, N, V, W, H, t_min, lut ? 1 : 0, g, prm, \
                                                            cls, depth, opacity, po)
  if (C <= 16)
    RND_LAUNCH(16);
  else if (C <= 32)
    RND_LAUNCH(32);
  else
    RND_LAUNCH(64);
#undef RND_LAUNCH
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}
