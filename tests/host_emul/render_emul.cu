// CPU emulation harness for csrc/render.cuh: the ray walk is __host__ __device__ IEEE double arithmetic with one
// rounding per operation, so running it on the host reproduces the device's class, depth and index per pixel.
#include "render.cuh"

extern "C" void occd_set_last_error(const char*) {}

// n pixels (u[i], v[i]) of one camera through one map: cls, depth (float32 of the entry time), index (-1 on a miss)
extern "C" int render_emulate(const uint16_t* map, const int* G, const long long* s, const double* origin, double voxel,
                              const double* camera, int empty, int ignore, double near_t, double far_t, long long n,
                              const int* u, const int* v, uint16_t* cls, float* depth, int32_t* index) {
  rnd::Grid g;
  for (int a = 0; a < 3; ++a) {
    g.origin[a] = origin[a];
    g.G[a] = G[a];
    g.s[a] = s[a];
  }
  g.voxel = voxel;
  g.empty = empty;
  g.ignore = ignore;
  g.near_t = near_t;
  g.far_t = far_t;
  rnd::Camera c;
  for (int i = 0; i < 9; ++i) c.M[i] = camera[i];
  for (int i = 0; i < 3; ++i) c.o[i] = camera[9 + i];
  for (long long p = 0; p < n; ++p) {
    const rnd::Hit h = rnd::cast_ray(c, g, map, u[p], v[p]);
    cls[p] = (uint16_t)h.cls;
    depth[p] = (float)h.t;
    index[p] = (int32_t)h.off;
  }
  return 0;
}
