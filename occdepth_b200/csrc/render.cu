// Camera views of a class map: one ray per pixel through a uint16 class map, walked voxel by voxel (Amanatides-Woo,
// render.cuh) to the first voxel whose class is neither `empty` nor `ignore`, with its class, entry depth and element
// offset.  The visibility query under the views the visualisation scripts draw from, on maps that never leave the
// device.
//
// One thread per pixel, consecutive threads on consecutive u, so neighbouring rays walk neighbouring voxels; one
// block row per image row and grid.z over the B x V cameras, which travel by value in the kernel parameters (no
// host-to-device copy, so the launch captures into a CUDA graph).  Each thread writes only its own pixel: the same
// inputs give the same bytes.
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
