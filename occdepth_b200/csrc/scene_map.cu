// Scene maps: a frame's float16 class probabilities summed as log-probabilities into a persistent, axis-aligned voxel
// map (naive-Bayes fusion; the accumulator is a logits tensor the class-map kernels read as they are), the whole-voxel
// shift of a streaming map, and the `unknown` mark of voxels no frame observed.
//
// Integrate: one thread per map voxel of the caller's box, consecutive threads along the contiguous MZ axis.  A voxel
// that falls in the frame grid (scene_map.cuh), inside the FOV mask and with no NaN probability is observed: its C
// float16 gathers are issued together, then its C accumulators are read together, then acc[c] += logf(max(p_c,
// min_prob)) and count += 1.  One writer per voxel and frame: no atomics, the same inputs give the same bytes.
#include <cuda_fp16.h>

#include "scene_map.cuh"
#include "../../include/occdepth_b200.h"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxClasses = 64;

template <int CMAX>
__global__ void __launch_bounds__(kThreads) integrate_kernel(float* __restrict__ acc, int* __restrict__ count,
                                                             const __half* __restrict__ probs, long long cstride,
                                                             const uint8_t* __restrict__ fov, int C, long long MV,
                                                             int MY, int MZ, int i0, int j0, int k0, int bj, int bk,
                                                             long long n, float min_prob, const smap::Geom g) {
  const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (t >= n) return;
  const long long r = t / bk;
  const int k = k0 + (int)(t - r * bk);
  const int j = j0 + (int)(r % bj);
  const int i = i0 + (int)(r / bj);
  const long long off = smap::frame_offset(g, i, j, k);
  if (off < 0 || (fov && !fov[off])) return;
  // every gather in flight before the first use; two classes per register
  __half2 p[CMAX / 2];
#pragma unroll
  for (int c = 0; c < CMAX; c += 2) {
    const __half lo = c < C ? probs[c * cstride + off] : __float2half(0.f);
    const __half hi = c + 1 < C ? probs[(c + 1) * cstride + off] : __float2half(0.f);
    p[c / 2] = __halves2half2(lo, hi);
  }
  bool nan = false;
#pragma unroll
  for (int c = 0; c < CMAX / 2; ++c) {
    const __half2 n2 = __hisnan2(p[c]);
    nan |= __low2float(n2) != 0.f || __high2float(n2) != 0.f;
  }
  if (nan) return;
  const long long v = ((long long)i * MY + j) * MZ + k;
  // the accumulators in groups of kGroup loads, each group's read-modify-writes after its loads
  constexpr int kGroup = 8;
#pragma unroll
  for (int c0 = 0; c0 < CMAX; c0 += kGroup) {
    if (c0 >= C) break;
    float a[kGroup];
#pragma unroll
    for (int u = 0; u < kGroup; ++u)
      if (c0 + u < C) a[u] = acc[(c0 + u) * MV + v];
#pragma unroll
    for (int u = 0; u < kGroup; ++u) {
      const int c = c0 + u;
      if (c < C) {
        const float pc = (c & 1) ? __high2float(p[c / 2]) : __low2float(p[c / 2]);
        acc[c * MV + v] = a[u] + logf(fmaxf(pc, min_prob));
      }
    }
  }
  count[v] += 1;
}

// planes [0, C) of acc and the count plane (blockIdx.y == C): out[idx] = in[idx + d], 0 where idx + d leaves the map
__global__ void __launch_bounds__(kThreads) shift_kernel(const float* __restrict__ acc, const int* __restrict__ count,
                                                         float* __restrict__ acc_out, int* __restrict__ count_out,
                                                         int C, int MX, int MY, int MZ, int dx, int dy, int dz,
                                                         long long MV) {
  const long long v = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (v >= MV) return;
  const int plane = blockIdx.y;
  const long long r = v / MZ;
  const int k = (int)(v - r * MZ) + dz, j = (int)(r % MY) + dy, i = (int)(r / MY) + dx;
  const bool in = i >= 0 && i < MX && j >= 0 && j < MY && k >= 0 && k < MZ;
  const long long s = ((long long)i * MY + j) * MZ + k;
  if (plane < C)
    acc_out[plane * MV + v] = in ? acc[plane * MV + s] : 0.f;
  else
    count_out[v] = in ? count[s] : 0;
}

__global__ void __launch_bounds__(kThreads) mark_kernel(unsigned short* __restrict__ map, const int* __restrict__ count,
                                                        long long n, unsigned short unknown) {
  const long long v = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (v < n && count[v] == 0) map[v] = unknown;
}

bool finite_all(const double* a, int n) {
  for (int i = 0; i < n; ++i)
    if (!isfinite(a[i])) return false;
  return true;
}

}  // namespace

extern "C" int occd_scene_map_integrate(float* acc, int32_t* count, int n_classes, int MX, int MY, int MZ,
                                        double voxel, const double* origin, const void* probs,
                                        const long long* strides, const uint8_t* fov_mask, int GX, int GY, int GZ,
                                        const double* grid_origin, double grid_voxel, const double* R, float min_prob,
                                        const int* box, void* stream) {
  OCCD_CHECK_ARG(acc && count && probs && origin && strides && grid_origin && R && box,
                 "occd_scene_map_integrate: acc, count, probs, origin, strides, grid_origin, R and box are required");
  OCCD_CHECK_ARG(n_classes >= 1 && n_classes <= kMaxClasses, "occd_scene_map_integrate: n_classes must be in [1, 64]");
  OCCD_CHECK_ARG(MX > 0 && MY > 0 && MZ > 0 && GX > 0 && GY > 0 && GZ > 0,
                 "occd_scene_map_integrate: map and frame grid dims must be positive");
  OCCD_CHECK_ARG(isfinite(voxel) && voxel > 0.0 && isfinite(grid_voxel) && grid_voxel > 0.0,
                 "occd_scene_map_integrate: voxel sizes must be finite and positive");
  OCCD_CHECK_ARG(finite_all(origin, 3) && finite_all(grid_origin, 3),
                 "occd_scene_map_integrate: origin and grid_origin must be finite");
  OCCD_CHECK_ARG(finite_all(R, 12), "occd_scene_map_integrate: R (inverse(T), rows 0..2) must be finite");
  OCCD_CHECK_ARG(min_prob > 0.f && min_prob <= 1.f, "occd_scene_map_integrate: min_prob must be in (0, 1]");
  OCCD_CHECK_ARG(strides[0] >= 0 && strides[1] >= 0 && strides[2] >= 0 && strides[3] >= 0,
                 "occd_scene_map_integrate: strides must be non-negative");
  OCCD_CHECK_ARG(box[0] >= 0 && box[0] <= box[1] && box[1] <= MX && box[2] >= 0 && box[2] <= box[3] &&
                     box[3] <= MY && box[4] >= 0 && box[4] <= box[5] && box[5] <= MZ,
                 "occd_scene_map_integrate: box must lie inside the map (0 <= lo <= hi <= dim per axis)");
  OCCD_CHECK_ARG((uintptr_t)acc % 4 == 0 && (uintptr_t)count % 4 == 0 && (uintptr_t)probs % 2 == 0,
                 "occd_scene_map_integrate: a pointer is not aligned to its element size");
  const long long bi = box[1] - box[0], bj = box[3] - box[2], bk = box[5] - box[4];
  const long long n = bi * bj * bk;
  if (n == 0) return OCCD_OK;
  smap::Geom g;
  for (int i = 0; i < 12; ++i) g.R[i] = R[i];
  for (int a = 0; a < 3; ++a) {
    g.origin[a] = origin[a];
    g.g[a] = grid_origin[a];
    g.s[a] = strides[1 + a];
  }
  g.voxel = voxel;
  g.vf = grid_voxel;
  g.G[0] = GX;
  g.G[1] = GY;
  g.G[2] = GZ;
  const long long MV = (long long)MX * MY * MZ;
  const unsigned blocks = (unsigned)((n + kThreads - 1) / kThreads);
  cudaStream_t st = (cudaStream_t)stream;
  const __half* p = static_cast<const __half*>(probs);
#define SMAP_LAUNCH(CM)                                                                                             \
  integrate_kernel<CM><<<blocks, kThreads, 0, st>>>(acc, count, p, strides[0], fov_mask, n_classes, MV, MY, MZ,     \
                                                     box[0], box[2], box[4], (int)bj, (int)bk, n, min_prob, g)
  if (n_classes <= 16)
    SMAP_LAUNCH(16);
  else if (n_classes <= 32)
    SMAP_LAUNCH(32);
  else
    SMAP_LAUNCH(64);
#undef SMAP_LAUNCH
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

extern "C" int occd_scene_map_shift(const float* acc, const int32_t* count, float* acc_out, int32_t* count_out,
                                    int n_classes, int MX, int MY, int MZ, const int* d, void* stream) {
  OCCD_CHECK_ARG(acc && count && acc_out && count_out && d,
                 "occd_scene_map_shift: acc, count, acc_out, count_out and d are required");
  OCCD_CHECK_ARG(n_classes >= 1 && n_classes <= kMaxClasses, "occd_scene_map_shift: n_classes must be in [1, 64]");
  OCCD_CHECK_ARG(MX > 0 && MY > 0 && MZ > 0, "occd_scene_map_shift: map dims must be positive");
  OCCD_CHECK_ARG(acc != acc_out && count != count_out, "occd_scene_map_shift: the copy is out of place");
  OCCD_CHECK_ARG((uintptr_t)acc % 4 == 0 && (uintptr_t)count % 4 == 0 && (uintptr_t)acc_out % 4 == 0 &&
                     (uintptr_t)count_out % 4 == 0,
                 "occd_scene_map_shift: a pointer is not aligned to its element size");
  const long long MV = (long long)MX * MY * MZ;
  // a shift of a whole dim or more leaves nothing: clamp so the index arithmetic stays in int
  int dd[3];
  const int M[3] = {MX, MY, MZ};
  for (int a = 0; a < 3; ++a) dd[a] = d[a] > M[a] ? M[a] : (d[a] < -M[a] ? -M[a] : d[a]);
  const dim3 grid((unsigned)((MV + kThreads - 1) / kThreads), (unsigned)(n_classes + 1));
  shift_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(acc, count, acc_out, count_out, n_classes, MX, MY, MZ,
                                                            dd[0], dd[1], dd[2], MV);
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

extern "C" int occd_scene_map_mark_unobserved(void* map, const int32_t* count, long long n, int unknown,
                                              void* stream) {
  OCCD_CHECK_ARG(map && count, "occd_scene_map_mark_unobserved: map and count are required");
  OCCD_CHECK_ARG(n > 0, "occd_scene_map_mark_unobserved: n must be positive");
  OCCD_CHECK_ARG(unknown >= 0 && unknown <= 65535, "occd_scene_map_mark_unobserved: unknown must be a uint16 id");
  OCCD_CHECK_ARG((uintptr_t)map % 2 == 0 && (uintptr_t)count % 4 == 0,
                 "occd_scene_map_mark_unobserved: a pointer is not aligned to its element size");
  mark_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      static_cast<unsigned short*>(map), count, n, (unsigned short)unknown);
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}
