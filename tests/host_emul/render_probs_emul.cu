// CPU emulation harness for the soft views of csrc/render.cuh: the walk is __host__ __device__ IEEE double arithmetic
// and the compositing IEEE float arithmetic, one rounding per operation, so running composite_ray on the host
// reproduces the device's class, depth, opacity and channels per pixel.
#include "render.cuh"

extern "C" void occd_set_last_error(const char*) {}

// n pixels (u[i], v[i]) of one camera through one item: probs float16 [C][plane] (planes cstride apart), class_map
// (or NULL), lut (C ids, or NULL); outputs cls, depth, opacity [n] and probs_out float16 [n][C]
extern "C" int render_probs_emulate(const __half* probs, int C, long long cstride, const uint16_t* class_map,
                                    const int* G, const long long* s, const double* origin, double voxel,
                                    const double* camera, int empty, int ignore, double near_t, double far_t,
                                    float t_min, const uint16_t* lut, long long n, const int* u, const int* v,
                                    uint16_t* cls, float* depth, float* opacity, __half* probs_out) {
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
  rnd::SoftIn in;
  in.probs = probs;
  in.cstride = cstride;
  in.cmap = class_map;
  in.C = C;
  in.t_min = t_min;
  in.lut = lut;
  for (long long p = 0; p < n; ++p) {
    if (C <= 16)
      rnd::composite_ray<16>(c, g, in, u[p], v[p], cls + p, depth + p, opacity + p, probs_out + p * C, 1);
    else if (C <= 32)
      rnd::composite_ray<32>(c, g, in, u[p], v[p], cls + p, depth + p, opacity + p, probs_out + p * C, 1);
    else
      rnd::composite_ray<64>(c, g, in, u[p], v[p], cls + p, depth + p, opacity + p, probs_out + p * C, 1);
  }
  return 0;
}
