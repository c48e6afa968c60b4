// Voxel-centre -> pixel projection of the data pipeline (occdepth/data/utils/helpers.py:94-169 `vox2pix`, with
// fusion.py:201-217 `vox2world`, :518-522 `rigid_transform`, :236-343 `cam2allpixs`), bit for bit:
//   centre_j = float32( origin32_j + voxel_size * idx_j + voxel_size * 0.5 )          (float64 arithmetic, one cast)
//   cam_r    = fma(E_r3, 1, fma(E_r2, z, fma(E_r1, y, E_r0 * x)))                      (np.dot of the 4x4 pose with
//              [centre 1]: the sequential-FMA accumulation of OpenBLAS' gemm kernels; in the POSE's precision --
//              float64 for the KITTI calibration, float32 when the caller hands a float32 pose)
//   xc       = int64(rint(cam_0 * fx32 / cam_2 + cx32)), yc likewise                   (same precision; np.round =
//              half to even)
//   pix[p]   = (xc + pattern[p].x, yc + pattern[p].y);  fov[p] = 0 <= x < W && 0 <= y < H && cam_2 > 0
// Voxel order: C order over (X, Y, Z) (np.meshgrid(..., indexing="ij") flattened).  One thread per voxel.  A window
// [v0, v0 + n) of that order (an X-slab of the grid) writes its voxels to outputs [0, n); the whole grid is v0 = 0.
// __host__ __device__ body: tests/host_emul/ runs it on the CPU against the reference itself.
#pragma once
#include <math.h>
#include "common.cuh"

namespace v2p {

constexpr int kMaxPattern = 25;
#define V2P_HD __host__ __device__ __forceinline__

template <typename T>
struct Args {
  T E[12];               // rows 0..2 of the 4x4 pose (cam_E), row-major, in the caller's precision
  float fx, fy, cx, cy;  // intrinsics AFTER the reference's .astype(float32)
  float origin[3];       // vox_origin AFTER .astype(float32)
  double voxel_size;
  int X, Y, Z, W, H, P;
  int pat[kMaxPattern][2];
  long long* pix;        // [n][P][2] (x, y), or null: only the mask (and pix_z) is written
  unsigned char* fov;    // [n][P] (numpy bool)
  T* pix_z;              // [n] or null
  long long v0 = 0;      // flat index of the window's first voxel; output i holds voxel v0 + i
};

V2P_HD double mul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
V2P_HD double add_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
V2P_HD double div_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
V2P_HD double fma_rn(double a, double b, double c) {
#ifdef __CUDA_ARCH__
  return __fma_rn(a, b, c);
#else
  return fma(a, b, c);
#endif
}
V2P_HD float mul_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
V2P_HD float add_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
V2P_HD float div_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
V2P_HD float fma_rn(float a, float b, float c) {
#ifdef __CUDA_ARCH__
  return __fmaf_rn(a, b, c);
#else
  return fmaf(a, b, c);
#endif
}

// int(np.round(v)) of the numba-compiled reference: rint, then the x86 float -> int64 conversion (which yields
// INT64_MIN for NaN / out-of-range values, e.g. a voxel centre exactly in the camera plane)
V2P_HD long long to_pix(double v) {
  const double r = rint(v);
  if (!(r >= -9223372036854775808.0 && r < 9223372036854775808.0)) return (long long)0x8000000000000000ULL;
  return (long long)r;
}
V2P_HD long long to_pix(float v) { return to_pix((double)rintf(v)); }

// output n of the window: voxel a.v0 + n
template <typename T>
V2P_HD void body(const Args<T>& a, long long n) {
  const long long v = a.v0 + n;
  const int k = (int)(v % a.Z);
  const int j = (int)((v / a.Z) % a.Y);
  const int i = (int)(v / ((long long)a.Z * a.Y));
  const int idx[3] = {i, j, k};
  T c[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    // vol_origin[j] + (vox_size * vox_coords[i, j]) + vox_size * offsets[j] in float64, stored to a float32 array
    const double v = add_rn(add_rn((double)a.origin[d], mul_rn(a.voxel_size, (double)(float)idx[d])),
                            mul_rn(a.voxel_size, 0.5));
    c[d] = (T)(float)v;
  }
  T cam[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const T* e = a.E + 4 * r;
    cam[r] = fma_rn(e[3], (T)1, fma_rn(e[2], c[2], fma_rn(e[1], c[1], mul_rn(e[0], c[0]))));
  }
  const long long xc = to_pix(add_rn(div_rn(mul_rn(cam[0], (T)a.fx), cam[2]), (T)a.cx));
  const long long yc = to_pix(add_rn(div_rn(mul_rn(cam[1], (T)a.fy), cam[2]), (T)a.cy));
  for (int p = 0; p < a.P; ++p) {
    const long long x = xc + a.pat[p][0], y = yc + a.pat[p][1];
    if (a.pix) {
      a.pix[(n * a.P + p) * 2] = x;
      a.pix[(n * a.P + p) * 2 + 1] = y;
    }
    a.fov[n * a.P + p] = (x >= 0 && x < a.W && y >= 0 && y < a.H && cam[2] > (T)0) ? 1 : 0;
  }
  if (a.pix_z) a.pix_z[n] = cam[2];
}

#ifdef __CUDACC__
template <typename T>
__global__ void __launch_bounds__(256) vox2pix_kernel(const Args<T> a, long long N) {
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n < N) body(a, n);
}
#endif

}  // namespace v2p
