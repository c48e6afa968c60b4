// Occupied-voxel list of a class map: the rows the reference's visualisation scripts select on the host
// (scripts/visualization/kitti_vis_pred.py:69-89: voxel centres from get_grid_coords, the class attached, split by
// fov_mask, rows with 0 < class < 255 kept) compacted on the device, in numpy's boolean-indexing order (ascending flat
// index, in-FOV voxels first), so only the occupied rows ever leave the device.
//
// Three launches over tiles of kTile voxels: count (per-tile in / out of FOV counts, the class histogram), scan (one
// block per frame turns the tile counts into exclusive offsets and writes the frame's totals), write (re-reads the
// tile -- 6 bytes per voxel, resident in L2 after the first pass -- and stores each occupied voxel at tile offset +
// its rank inside the tile).  Positions depend only on the map, never on scheduling: two runs write the same bytes.
#include <string.h>

#include "common.cuh"
#include "../../include/occdepth_b200.h"

namespace {

constexpr int kThreads = 256;
constexpr int kGroup = 8;                 // voxels per thread: one 16-byte load of the map, one 8-byte load of the mask
constexpr int kTile = kThreads * kGroup;
static_assert(kTile == OCCD_VOXEL_TILE, "the header's workspace formula assumes this tile");
constexpr int kMaxClasses = 64;
constexpr int kScanThreads = 1024;

// this thread's kGroup voxels of frame-local tile `tile`: bit k of `occ` = voxel e + k is occupied
// (empty < class < ignore), bit k of `in` = it is inside the FOV (every voxel when there is no mask)
struct Group {
  unsigned short c[kGroup];
  unsigned occ, in;
  int e;
};

__device__ __forceinline__ Group load_group(const unsigned short* __restrict__ map, const uint8_t* __restrict__ fov,
                                            int N, int tile, int empty, int ignore) {
  Group g;
  g.e = tile * kTile + (int)threadIdx.x * kGroup;
  g.occ = 0u;
  g.in = fov ? 0u : 0xffu;
  if (g.e >= N) return g;
  // the frame's base pointers decide (uniformly for the block) whether full groups take vector loads
  const bool vec = ((uintptr_t)map & 15) == 0 && ((uintptr_t)fov & 7) == 0 && g.e + kGroup <= N;
  if (vec) {
    const uint4 r = *reinterpret_cast<const uint4*>(map + g.e);
    memcpy(g.c, &r, sizeof(r));
    if (fov) {
      const uint2 m = *reinterpret_cast<const uint2*>(fov + g.e);
      uint8_t b[kGroup];
      memcpy(b, &m, sizeof(m));
#pragma unroll
      for (int k = 0; k < kGroup; ++k) g.in |= (b[k] ? 1u : 0u) << k;
    }
  } else {
#pragma unroll
    for (int k = 0; k < kGroup; ++k) {
      const bool ok = g.e + k < N;
      g.c[k] = ok ? map[g.e + k] : (unsigned short)empty;
      if (fov && ok && fov[g.e + k]) g.in |= 1u << k;
    }
  }
#pragma unroll
  for (int k = 0; k < kGroup; ++k) g.occ |= ((int)g.c[k] > empty && (int)g.c[k] < ignore ? 1u : 0u) << k;
  return g;
}

// work[(b*T + tile)] = (occupied in FOV, occupied out of FOV) of the tile; hist[b][class] += occupied voxels
__global__ void __launch_bounds__(kThreads) voxel_count_kernel(const unsigned short* __restrict__ map,
                                                               const uint8_t* __restrict__ fov, int N, int empty,
                                                               int ignore, int C, uint2* __restrict__ work,
                                                               unsigned int* __restrict__ hist) {
  __shared__ unsigned int s_hist[kMaxClasses];
  __shared__ unsigned int s_cnt[2];
  const int b = blockIdx.y, T = gridDim.x;
  if (threadIdx.x < kMaxClasses) s_hist[threadIdx.x] = 0u;
  if (threadIdx.x < 2) s_cnt[threadIdx.x] = 0u;
  __syncthreads();
  const Group g = load_group(map + (long long)b * N, fov ? fov + (long long)b * N : nullptr, N, blockIdx.x, empty,
                             ignore);
#pragma unroll
  for (int k = 0; k < kGroup; ++k)
    if ((g.occ >> k & 1u) && g.c[k] < C) atomicAdd(&s_hist[g.c[k]], 1u);
  const unsigned n_in = __reduce_add_sync(0xffffffffu, (unsigned)__popc(g.occ & g.in));
  const unsigned n_out = __reduce_add_sync(0xffffffffu, (unsigned)__popc(g.occ & ~g.in));
  if ((threadIdx.x & 31) == 0) {
    if (n_in) atomicAdd(&s_cnt[0], n_in);
    if (n_out) atomicAdd(&s_cnt[1], n_out);
  }
  __syncthreads();
  if (threadIdx.x == 0) work[(long long)b * T + blockIdx.x] = make_uint2(s_cnt[0], s_cnt[1]);
  if (threadIdx.x < C && s_hist[threadIdx.x]) atomicAdd(&hist[b * C + threadIdx.x], s_hist[threadIdx.x]);
}

// exclusive scan of a block's values (x and y independently); `total` receives the block's sums.  Every thread of the
// block calls it; `s` holds one uint2 per warp
template <int THREADS>
__device__ __forceinline__ uint2 block_exclusive_scan(uint2 v, uint2* s, uint2& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint2 inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned ax = __shfl_up_sync(0xffffffffu, inc.x, d), ay = __shfl_up_sync(0xffffffffu, inc.y, d);
    if (lane >= d) {
      inc.x += ax;
      inc.y += ay;
    }
  }
  if (lane == 31) s[warp] = inc;
  __syncthreads();
  uint2 pre = make_uint2(0u, 0u);
  total = make_uint2(0u, 0u);
#pragma unroll
  for (int w = 0; w < THREADS / 32; ++w) {
    const uint2 t = s[w];
    if (w < warp) {
      pre.x += t.x;
      pre.y += t.y;
    }
    total.x += t.x;
    total.y += t.y;
  }
  __syncthreads();                      // s is reused by the caller's next round
  return make_uint2(pre.x + inc.x - v.x, pre.y + inc.y - v.y);
}

// one block per frame: work[b][*] becomes the exclusive prefix of the tile counts; count[b] = the frame's totals
__global__ void __launch_bounds__(kScanThreads) voxel_scan_kernel(uint2* __restrict__ work, int T,
                                                                  unsigned int* __restrict__ count) {
  __shared__ uint2 s[kScanThreads / 32];
  uint2* w = work + (long long)blockIdx.x * T;
  uint2 carry = make_uint2(0u, 0u);
  for (int base = 0; base < T; base += kScanThreads) {
    const int i = base + (int)threadIdx.x;
    const uint2 v = i < T ? w[i] : make_uint2(0u, 0u);
    uint2 total;
    const uint2 ex = block_exclusive_scan<kScanThreads>(v, s, total);
    if (i < T) w[i] = make_uint2(carry.x + ex.x, carry.y + ex.y);
    carry.x += total.x;
    carry.y += total.y;
  }
  if (threadIdx.x == 0) {
    count[2 * blockIdx.x] = carry.x;
    count[2 * blockIdx.x + 1] = carry.y;
  }
}

struct Coords {
  double res, half, origin[3];
  int YZ, Z, index0;
};

// rows [0, cap) of frame b: the in-FOV voxels from row 0, the others from row count[b][0], each in ascending index
template <bool XYZ>
__global__ void __launch_bounds__(kThreads) voxel_write_kernel(const unsigned short* __restrict__ map,
                                                               const uint8_t* __restrict__ fov, int N, int empty,
                                                               int ignore, unsigned int cap,
                                                               const uint2* __restrict__ work,
                                                               const unsigned int* __restrict__ count,
                                                               int* __restrict__ index,
                                                               unsigned short* __restrict__ cls,
                                                               float* __restrict__ xyz, Coords cg) {
  __shared__ uint2 s[kThreads / 32];
  const int b = blockIdx.y, T = gridDim.x;
  const Group g = load_group(map + (long long)b * N, fov ? fov + (long long)b * N : nullptr, N, blockIdx.x, empty,
                             ignore);
  uint2 total;
  const uint2 ex = block_exclusive_scan<kThreads>(
      make_uint2((unsigned)__popc(g.occ & g.in), (unsigned)__popc(g.occ & ~g.in)), s, total);
  if (total.x + total.y == 0u) return;
  const uint2 off = work[(long long)b * T + blockIdx.x];
  unsigned p_in = off.x + ex.x, p_out = count[2 * b] + off.y + ex.y;
  const long long row0 = (long long)b * cap;
#pragma unroll
  for (int k = 0; k < kGroup; ++k) {
    if (!(g.occ >> k & 1u)) continue;
    const unsigned p = (g.in >> k & 1u) ? p_in++ : p_out++;
    if (p >= cap) continue;
    const int gi = cg.index0 + g.e + k;
    index[row0 + p] = gi;
    cls[row0 + p] = g.c[k];
    if constexpr (XYZ) {
      // numpy's float64 `idx * resolution + resolution / 2` (a product, then a sum: no fused multiply-add), the
      // origin added to that, then one rounding to float32
      const int r = gi % cg.YZ;
      const int v[3] = {gi / cg.YZ, r / cg.Z, r % cg.Z};
      float* o = xyz + (row0 + p) * 3;
#pragma unroll
      for (int a = 0; a < 3; ++a)
        o[a] = (float)__dadd_rn(__dadd_rn(__dmul_rn((double)v[a], cg.res), cg.half), cg.origin[a]);
    }
  }
}

}  // namespace

extern "C" int occd_occupied_voxels(const uint16_t* class_map, const uint8_t* fov_mask, int B, int X, int Y, int Z,
                                    int index0, int empty, int ignore, int n_classes, int cap, uint32_t* count,
                                    uint32_t* hist, int32_t* index, uint16_t* cls, float* xyz, double voxel_size,
                                    const double* origin, uint32_t* work, long long work_len, void* stream) {
  OCCD_CHECK_ARG(class_map && count && hist && work, "occd_occupied_voxels: class_map, count, hist and work are required");
  OCCD_CHECK_ARG(B > 0 && X > 0 && Y > 0 && Z > 0 && index0 >= 0, "occd_occupied_voxels: B, X, Y, Z must be positive, index0 >= 0");
  const long long N = (long long)X * Y * Z;
  OCCD_CHECK_ARG(N + index0 <= 2147483647LL && B <= 65535, "occd_occupied_voxels: flat indices must fit int32, B <= 65535");
  OCCD_CHECK_ARG(n_classes > 0 && n_classes <= kMaxClasses, "occd_occupied_voxels: n_classes must be in [1, 64]");
  OCCD_CHECK_ARG(empty >= 0 && ignore >= 0 && empty <= 65535 && ignore <= 65535,
                 "occd_occupied_voxels: empty / ignore must be uint16 class ids");
  OCCD_CHECK_ARG(cap >= 0 && (cap == 0 || (index && cls)), "occd_occupied_voxels: cap >= 0, and index / cls when cap > 0");
  OCCD_CHECK_ARG(!xyz || voxel_size > 0.0, "occd_occupied_voxels: voxel_size must be positive when xyz is written");
  const int T = (int)((N + kTile - 1) / kTile);
  OCCD_CHECK_ARG(work_len >= OCCD_VOXEL_WORK_LEN(B, N), "occd_occupied_voxels: work is shorter than OCCD_VOXEL_WORK_LEN(B, N)");
  OCCD_CHECK_ARG((uintptr_t)class_map % 2 == 0 && (uintptr_t)work % 8 == 0 && (uintptr_t)count % 4 == 0 &&
                     (uintptr_t)hist % 4 == 0 && (uintptr_t)index % 4 == 0 && (uintptr_t)cls % 2 == 0 &&
                     (uintptr_t)xyz % 4 == 0,
                 "occd_occupied_voxels: a pointer is not aligned to its element size (work: 8 bytes)");
  cudaStream_t st = (cudaStream_t)stream;
  if (cudaMemsetAsync(hist, 0, (size_t)B * n_classes * sizeof(uint32_t), st) != cudaSuccess) {
    occd_set_last_error("occd_occupied_voxels: clearing hist failed");
    return OCCD_ERR_CUDA;
  }
  uint2* w = reinterpret_cast<uint2*>(work);
  const dim3 grid((unsigned)T, (unsigned)B);
  voxel_count_kernel<<<grid, kThreads, 0, st>>>(class_map, fov_mask, (int)N, empty, ignore, n_classes, w, hist);
  OCCD_CHECK_LAUNCH();
  voxel_scan_kernel<<<(unsigned)B, kScanThreads, 0, st>>>(w, T, count);
  OCCD_CHECK_LAUNCH();
  if (cap == 0) return OCCD_OK;
  Coords cg;
  cg.res = voxel_size;
  cg.half = voxel_size / 2;
  for (int a = 0; a < 3; ++a) cg.origin[a] = origin ? origin[a] : 0.0;
  cg.YZ = Y * Z;
  cg.Z = Z;
  cg.index0 = index0;
  if (xyz)
    voxel_write_kernel<true><<<grid, kThreads, 0, st>>>(class_map, fov_mask, (int)N, empty, ignore, (unsigned)cap, w,
                                                        count, index, cls, xyz, cg);
  else
    voxel_write_kernel<false><<<grid, kThreads, 0, st>>>(class_map, fov_mask, (int)N, empty, ignore, (unsigned)cap,
                                                         w, count, index, cls, xyz, cg);
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}
