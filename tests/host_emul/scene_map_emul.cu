// CPU emulation harness for csrc/scene_map.cuh: the index function is __host__ __device__ IEEE double arithmetic with
// one rounding per operation, so running it on the host reproduces the device's frame index and observed flag.
#include "scene_map.cuh"

extern "C" void occd_set_last_error(const char*) {}

// for every voxel of an MX x MY x MZ map (C order): off[v] = frame_offset (-1 outside), f[v][3] = the frame index
extern "C" int scene_map_index_emulate(const double* R, const double* origin, double voxel, int MX, int MY, int MZ,
                                       const double* grid_origin, double grid_voxel, const int* G, const long long* s,
                                       long long* off, double* f) {
  smap::Geom g;
  for (int i = 0; i < 12; ++i) g.R[i] = R[i];
  for (int a = 0; a < 3; ++a) {
    g.origin[a] = origin[a];
    g.g[a] = grid_origin[a];
    g.G[a] = G[a];
    g.s[a] = s[a];
  }
  g.voxel = voxel;
  g.vf = grid_voxel;
  long long v = 0;
  for (int i = 0; i < MX; ++i)
    for (int j = 0; j < MY; ++j)
      for (int k = 0; k < MZ; ++k, ++v) off[v] = smap::frame_offset(g, i, j, k, f + 3 * v);
  return 0;
}
