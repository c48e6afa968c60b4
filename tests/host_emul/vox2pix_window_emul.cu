// CPU emulation harness for the windowed form of csrc/vox2pix.cuh: v2p::body over outputs [0, n) of the window
// that starts at voxel v0, exactly as vox2pix_kernel runs it for occd_vox2pix_range_fwd.
#include "vox2pix.cuh"

extern "C" void occd_set_last_error(const char*) {}

template <typename T>
static int run(const void* cam_E, const float* cam_k, const float* vox_origin, double voxel_size, int X, int Y, int Z,
               int img_W, int img_H, const int* pattern, int P, long long* pix, unsigned char* fov, void* pix_z,
               long long v0, long long n) {
  v2p::Args<T> a;
  for (int i = 0; i < 12; ++i) a.E[i] = static_cast<const T*>(cam_E)[i];
  a.fx = cam_k[0]; a.fy = cam_k[4]; a.cx = cam_k[2]; a.cy = cam_k[5];
  for (int i = 0; i < 3; ++i) a.origin[i] = vox_origin[i];
  a.voxel_size = voxel_size;
  a.X = X; a.Y = Y; a.Z = Z; a.W = img_W; a.H = img_H; a.P = P;
  for (int p = 0; p < P; ++p) { a.pat[p][0] = pattern[2 * p]; a.pat[p][1] = pattern[2 * p + 1]; }
  a.pix = pix; a.fov = fov; a.pix_z = static_cast<T*>(pix_z);
  a.v0 = v0;
  for (long long i = 0; i < n; ++i) v2p::body(a, i);
  return 0;
}

extern "C" int vox2pix_window_emulate(const void* cam_E, int pose_is_f32, const float* cam_k, const float* vox_origin,
                                      double voxel_size, int X, int Y, int Z, int img_W, int img_H, const int* pattern,
                                      int P, long long* pix, unsigned char* fov, void* pix_z, long long v0,
                                      long long n) {
  if (P < 1 || P > v2p::kMaxPattern || v0 < 0 || n < 1 || v0 + n > (long long)X * Y * Z) return 1;
  return pose_is_f32 ? run<float>(cam_E, cam_k, vox_origin, voxel_size, X, Y, Z, img_W, img_H, pattern, P, pix, fov,
                                  pix_z, v0, n)
                     : run<double>(cam_E, cam_k, vox_origin, voxel_size, X, Y, Z, img_W, img_H, pattern, P, pix, fov,
                                   pix_z, v0, n);
}
