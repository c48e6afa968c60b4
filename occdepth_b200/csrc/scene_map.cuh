// Scene maps: the index math that places a map voxel in a frame's output grid (include/occdepth_b200.h, "Scene
// maps").  For map voxel (i, j, k):
//   c_a = ((idx_a + 0.5) * voxel) + origin_a                                      (float64)
//   q_r = ((R[r][0] * c_x + R[r][1] * c_y) + R[r][2] * c_z) + R[r][3]             (float64, in this order, no FMA)
//   f_a = floor((q_a - g_a) / v_f)                                                (a true division)
// R = inverse(T), T the frame grid's frame -> map frame.  Every operation is one correctly rounded IEEE step, so the
// device, the host build in tests/host_emul/ and numpy's element-wise float64 restatement give the same bits.
#pragma once
#include <math.h>
#include "common.cuh"

namespace smap {

#define SMAP_HD __host__ __device__ __forceinline__

struct Geom {
  double R[12];               // rows 0..2 of inverse(T), row-major: map frame -> the frame grid's frame
  double origin[3], voxel;    // the map
  double g[3], vf;            // the frame grid: origin and voxel edge
  int G[3];                   // the frame grid's dims along its x, y, z
  long long s[3];             // element strides of x, y, z inside one class plane
};

SMAP_HD double mul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
SMAP_HD double add_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
SMAP_HD double sub_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
SMAP_HD double div_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
// the float32 twins: one correctly rounded IEEE single operation each, never contracted into an FMA
SMAP_HD float fmul_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
SMAP_HD float fadd_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
SMAP_HD float fsub_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
SMAP_HD float fdiv_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}

// element offset inside a class plane of the frame voxel that map voxel (i, j, k) falls in, or -1 when its centre
// lies outside the frame grid.  f[3] receives the frame index (also when outside; NaN-free since R is finite)
SMAP_HD long long frame_offset(const Geom& a, int i, int j, int k, double* f = nullptr) {
  const int idx[3] = {i, j, k};
  double c[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) c[d] = add_rn(mul_rn((double)idx[d] + 0.5, a.voxel), a.origin[d]);
  long long off = 0;
  bool in = true;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double* R = a.R + 4 * r;
    const double q = add_rn(add_rn(add_rn(mul_rn(R[0], c[0]), mul_rn(R[1], c[1])), mul_rn(R[2], c[2])), R[3]);
    const double fr = floor(div_rn(sub_rn(q, a.g[r]), a.vf));
    if (f) f[r] = fr;
    // compared as a double first: a far-away centre must not overflow the integer conversion
    in = in && fr >= 0.0 && fr < (double)a.G[r];
    if (in) off += (long long)fr * a.s[r];
  }
  return in ? off : -1;
}

}  // namespace smap
