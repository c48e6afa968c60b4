// FlospDepth occupancy prior: frustum grid generation fused with trilinear sampling of the depth distribution.
// replaces FrustumGridGenerator.forward/transform_grid (occdepth/models/f2v/frustum_grid_generator.py:70-152),
// bin_depths LID (f2v/utils/depth_utils.py:24-26), normalize_coords (f2v/utils/grid_utils.py:4-19),
// Sampler / F.grid_sample 5-D bilinear zeros align_corners=False (f2v/sampler.py:49-65) for the depth volume AND
// the all-ones mask volume, and the per-camera masked mean of FlospDepth.forward (flosp_depth.py:563-602).
// The grid is never materialised: each thread computes its voxel's sampling coordinate on the fly.
// Also: channel softmax (flosp_depth.py:548), small FC layers of DepthNet's Mlp/SELayer (:159-199), channel gate.
#include "common.cuh"
#include "../../include/occdepth_b200.h"

namespace {

struct FrustumCam {
  float T[12];    // rows 0..2 of lidar_to_cam @ grid_to_lidar (voxel index+0.5 -> camera)
  float K[12];    // cam_to_img 3x4
  float ida[16];  // 4x4
};

__device__ __forceinline__ float dehom(float z) {  // kornia 0.5.0 convert_points_from_homogeneous scale
  return fabsf(z) > 1e-8f ? 1.f / (z + 1e-8f) : 1.f;
}

// GIVEN: the normalised sampling coordinates are read from `grids` ([V][N][3] = (x, y, z) of F.grid_sample's grid:
// the reference's infer_mode / ONNX route feeds pre-computed grids, OccDepth.py:310-317, flosp_depth.py:564-565)
// instead of being computed from the camera tables.
// X window: the thread grid covers planes [xw0, xw0 + Xl) of the X-plane grid and writes them densely in the local
// voxel order (perm_xzy applied inside the window); the voxel coordinate and the index of a given grid are those of
// the full grid, so a window computes exactly the values of the matching slice of the whole grid.
template <bool GIVEN>
__global__ void frustum_sample_kernel(const float* __restrict__ depth, const FrustumCam* __restrict__ cams,
                                      const float* __restrict__ grids, int V,
                                      int Dn, int h, int w, int X, int Y, int Z, int xw0, int Xl, float img_w,
                                      float img_h, float dmin, float bin_size, int mean_mode,
                                      float* __restrict__ out, int perm_xzy) {
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // local voxel index
  const long long N = (long long)X * Y * Z;
  if (n >= (long long)Xl * Y * Z) return;
  const int k = (int)(n % Z), j = (int)((n / Z) % Y), il = (int)(n / ((long long)Z * Y));
  const int i = xw0 + il;
  const long long nf = n + (long long)xw0 * Y * Z;                         // full-grid voxel index
  const float px = i + 0.5f, py = j + 0.5f, pz = k + 0.5f;
  float fsum = 0.f, msum = 0.f;
  for (int v = 0; v < V; ++v) {
    float nx, ny, nz;
    if constexpr (GIVEN) {
      const float* g = grids + ((long long)v * N + nf) * 3;
      nx = g[0]; ny = g[1]; nz = g[2];
    } else {
    const FrustumCam& c = cams[v];
    // camera point (homogeneous w == 1 -> scale 1/(1+1e-8) == 1 in fp32)
    const float cx = c.T[0] * px + c.T[1] * py + c.T[2] * pz + c.T[3];
    const float cy = c.T[4] * px + c.T[5] * py + c.T[6] * pz + c.T[7];
    const float cz = c.T[8] * px + c.T[9] * py + c.T[10] * pz + c.T[11];
    const float ix = c.K[0] * cx + c.K[1] * cy + c.K[2] * cz + c.K[3];
    const float iy = c.K[4] * cx + c.K[5] * cy + c.K[6] * cz + c.K[7];
    const float iz = c.K[8] * cx + c.K[9] * cy + c.K[10] * cz + c.K[11];
    const float sc = dehom(iz);
    const float u = ix * sc, vv = iy * sc;
    const float dep = iz - c.K[11];
    const float bin = -0.5f + 0.5f * sqrtf(1.f + 8.f * (dep - dmin) / bin_size);
    // ida (4x4) on (u, v, bin, 1), de-homogenised
    const float gx = c.ida[0] * u + c.ida[1] * vv + c.ida[2] * bin + c.ida[3];
    const float gy = c.ida[4] * u + c.ida[5] * vv + c.ida[6] * bin + c.ida[7];
    const float gz = c.ida[8] * u + c.ida[9] * vv + c.ida[10] * bin + c.ida[11];
    const float gw = c.ida[12] * u + c.ida[13] * vv + c.ida[14] * bin + c.ida[15];
    const float s2 = dehom(gw);
    nx = gx * s2 / (img_w - 1.f) * 2.f - 1.f;
    ny = gy * s2 / (img_h - 1.f) * 2.f - 1.f;
    nz = gz * s2 / ((float)Dn - 1.f) * 2.f - 1.f;
    if (!isfinite(nx)) nx = -2.f;
    if (!isfinite(ny)) ny = -2.f;
    if (!isfinite(nz)) nz = -2.f;
    }
    // grid_sample, align_corners=False: pixel = ((g + 1) * size - 1) / 2
    const float fx = ((nx + 1.f) * w - 1.f) * 0.5f;
    const float fy = ((ny + 1.f) * h - 1.f) * 0.5f;
    const float fz = ((nz + 1.f) * Dn - 1.f) * 0.5f;
    const float x0f = floorf(fx), y0f = floorf(fy), z0f = floorf(fz);
    const int x0 = (int)x0f, y0 = (int)y0f, z0 = (int)z0f;
    const float tx = fx - x0f, ty = fy - y0f, tz = fz - z0f;
    const float* vol = depth + (long long)v * Dn * h * w;
    float f = 0.f, m = 0.f;
#pragma unroll
    for (int dz = 0; dz < 2; ++dz)
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          const int xx = x0 + dx, yy = y0 + dy, zz = z0 + dz;
          if (xx >= 0 && xx < w && yy >= 0 && yy < h && zz >= 0 && zz < Dn) {
            const float wgt = (dx ? tx : 1.f - tx) * (dy ? ty : 1.f - ty) * (dz ? tz : 1.f - tz);
            f += wgt * __ldg(vol + ((long long)zz * h + yy) * w + xx);
            m += wgt;
          }
        }
    fsum += f;
    msum += m;
  }
  float r = fsum;
  if (V > 1 && mean_mode && msum > 0.f) r = fsum / msum;
  long long no = n;
  if (perm_xzy) no = ((long long)il * Z + k) * Y + j;  // x3ds_depth.permute(0,1,2,4,3) (OccDepth.py:337)
  out[no] = r;
}

// softmax over C planar channels per position: in/out [B][C][S] fp32
__global__ void softmax_planar_kernel(const float* __restrict__ in, float* __restrict__ out, int C, long long S,
                                      long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long b = i / S, s = i % S;
  const float* p = in + b * C * S + s;
  float* o = out + b * C * S + s;
  float m = -INFINITY;
  for (int c = 0; c < C; ++c) m = fmaxf(m, p[(long long)c * S]);
  float sum = 0.f;
  for (int c = 0; c < C; ++c) sum += expf(p[(long long)c * S] - m);
  const float inv = 1.f / sum;
  for (int c = 0; c < C; ++c) o[(long long)c * S] = expf(p[(long long)c * S] - m) * inv;
}

// out[b][o] = act(bias[o] + sum_i w[o][i] * in[b][i]); one warp per output
__global__ void fc_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                          float* __restrict__ out, int n_in, int n_out, int act) {
  const int o = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  if (o >= n_out) return;
  float s = 0.f;
  for (int i = lane; i < n_in; i += 32) s = fmaf(w[(long long)o * n_in + i], in[(long long)b * n_in + i], s);
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
  if (lane == 0) out[(long long)b * n_out + o] = apply_act(s + bias[o], act);
}

// x[b][pos][c] *= gate[b][c]  (channels-last, C % 8 == 0)
template <typename T>
__global__ void channel_scale_kernel(T* __restrict__ x, const float* __restrict__ gate, long long S, int C,
                                     int cstride, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int cv = (int)(i % (C / 8));
  const long long pos = i / (C / 8);
  const long long b = pos / S;
  T* p = x + pos * cstride + cv * 8;
  float v[8];
  Elem<T>::ld8(p, v);
  const float* g = gate + b * C + cv * 8;
#pragma unroll
  for (int k = 0; k < 8; ++k) v[k] *= g[k];
  Elem<T>::st8(p, v);
}

}  // namespace

namespace {
int frustum_window(const float* depth, const float* cams, const float* grids, int V, int Dn, int h, int w, int X,
                   int Y, int Z, int xw0, int Xl, float img_w, float img_h, float dmin, float dmax, int mean_mode,
                   float* out, int perm_xzy, void* stream) {
  const long long N = (long long)Xl * Y * Z;
  OCCD_CHECK_ARG((N + 255) / 256 <= 2147483647LL, "frustum sampling: too many voxels");
  if (grids) {
    frustum_sample_kernel<true><<<(unsigned)((N + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        depth, nullptr, grids, V, Dn, h, w, X, Y, Z, xw0, Xl, 0.f, 0.f, 0.f, 1.f, mean_mode, out, perm_xzy);
  } else {
    const float bin_size = 2.f * (dmax - dmin) / ((float)Dn * (1.f + (float)Dn));
    frustum_sample_kernel<false><<<(unsigned)((N + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        depth, reinterpret_cast<const FrustumCam*>(cams), nullptr, V, Dn, h, w, X, Y, Z, xw0, Xl, img_w, img_h, dmin,
        bin_size, mean_mode, out, perm_xzy);
  }
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}
}  // namespace

extern "C" int occd_frustum_sample_fwd(const float* depth, const float* cams, int V, int Dn, int h, int w, int X, int Y,
                                       int Z, float img_w, float img_h, float dmin, float dmax, int mean_mode,
                                       float* out, int perm_xzy, void* stream) {
  OCCD_CHECK_ARG(depth && cams && out && V >= 1 && Dn > 1 && h > 0 && w > 0 && X > 0 && Y > 0 && Z > 0,
                 "occd_frustum_sample_fwd: args");
  return frustum_window(depth, cams, nullptr, V, Dn, h, w, X, Y, Z, 0, X, img_w, img_h, dmin, dmax, mean_mode, out,
                        perm_xzy, stream);
}

extern "C" int occd_frustum_sample_window_fwd(const float* depth, const float* cams, int V, int Dn, int h, int w,
                                              int X, int Y, int Z, int x0, int Xl, float img_w, float img_h,
                                              float dmin, float dmax, int mean_mode, float* out, int perm_xzy,
                                              void* stream) {
  OCCD_CHECK_ARG(depth && cams && out && V >= 1 && Dn > 1 && h > 0 && w > 0 && X > 0 && Y > 0 && Z > 0,
                 "occd_frustum_sample_window_fwd: args");
  OCCD_CHECK_ARG(Xl > 0 && x0 >= 0 && x0 <= X - Xl, "occd_frustum_sample_window_fwd: the window [x0, x0 + Xl) must "
                 "hold at least one plane and lie inside the X planes of the grid");
  return frustum_window(depth, cams, nullptr, V, Dn, h, w, X, Y, Z, x0, Xl, img_w, img_h, dmin, dmax, mean_mode, out,
                        perm_xzy, stream);
}

extern "C" int occd_grid_sample_prior_fwd(const float* depth, const float* grids, int V, int Dn, int h, int w, int X,
                                          int Y, int Z, int mean_mode, float* out, int perm_xzy, void* stream) {
  OCCD_CHECK_ARG(depth && grids && out && V >= 1 && Dn > 1 && h > 0 && w > 0 && X > 0 && Y > 0 && Z > 0,
                 "occd_grid_sample_prior_fwd: args");
  return frustum_window(depth, nullptr, grids, V, Dn, h, w, X, Y, Z, 0, X, 0.f, 0.f, 0.f, 0.f, mean_mode, out,
                        perm_xzy, stream);
}

extern "C" int occd_grid_sample_prior_window_fwd(const float* depth, const float* grids, int V, int Dn, int h, int w,
                                                 int X, int Y, int Z, int x0, int Xl, int mean_mode, float* out,
                                                 int perm_xzy, void* stream) {
  OCCD_CHECK_ARG(depth && grids && out && V >= 1 && Dn > 1 && h > 0 && w > 0 && X > 0 && Y > 0 && Z > 0,
                 "occd_grid_sample_prior_window_fwd: args");
  OCCD_CHECK_ARG(Xl > 0 && x0 >= 0 && x0 <= X - Xl, "occd_grid_sample_prior_window_fwd: the window [x0, x0 + Xl) "
                 "must hold at least one plane and lie inside the X planes of the grid");
  return frustum_window(depth, nullptr, grids, V, Dn, h, w, X, Y, Z, x0, Xl, 0.f, 0.f, 0.f, 0.f, mean_mode, out,
                        perm_xzy, stream);
}

extern "C" int occd_softmax_planar(const float* in, float* out, long long B, int C, long long S, void* stream) {
  OCCD_CHECK_ARG(in && out && B > 0 && C > 0 && S > 0, "occd_softmax_planar: args");
  const long long total = B * S;
  softmax_planar_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(in, out, C, S, total);
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

extern "C" int occd_fc_fwd(const float* in, const float* w, const float* bias, float* out, int B, int n_in, int n_out,
                           int act, void* stream) {
  OCCD_CHECK_ARG(in && w && bias && out && B > 0 && n_in > 0 && n_out > 0, "occd_fc_fwd: args");
  fc_kernel<<<dim3((n_out + 3) / 4, B), 128, 0, (cudaStream_t)stream>>>(in, w, bias, out, n_in, n_out, act);
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

extern "C" int occd_channel_scale(void* x, const float* gate, int dtype, long long B, long long S, int C, int cstride,
                                  void* stream) {
  OCCD_CHECK_ARG(x && gate && B > 0 && S > 0 && C > 0 && C % 8 == 0 && cstride % 8 == 0 && cstride >= C,
                 "occd_channel_scale: args");
  const long long total = B * S * (C / 8);
  OCCD_DISPATCH_DTYPE(dtype, T, (channel_scale_kernel<T><<<(unsigned)((total + 255) / 256), 256, 0,
                                                            (cudaStream_t)stream>>>((T*)x, gate, S, C, cstride,
                                                                                    total)));
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

namespace {
// Virtual right view from the left features and a depth map (NYU "virtual stereo"):
// replaces OccDepth.generate_virtual_img (occdepth/models/OccDepth.py:233-260): F.interpolate(depth, bilinear,
// align_corners=False) -> disparity bf/scale / depth (inf -> 0) -> base grid arange(-1,1,2/h) (pixel-CORNER
// coordinates) shifted by disparity*2/w -> F.grid_sample(bilinear, border, align_corners=False).
// The reference uses batch item 0's disparity for every item (:257): depth_stride 0.  A batch of independent camera
// frames gives item b the depth map at depth + b * depth_stride.
template <typename T>
__global__ void virtual_view_kernel(const T* __restrict__ in, T* __restrict__ out,
                                    const float* __restrict__ depth, int B, int h, int w, int CV, int cs_in,
                                    int cs_out, int dh, int dw, float bf_scale, long long depth_stride) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)B * h * w * CV;
  if (i >= total) return;
  const int cv = (int)(i % CV);
  long long p = i / CV;
  const int x = (int)(p % w); p /= w;
  const int y = (int)(p % h); p /= h;
  const int b = (int)p;
  depth += b * depth_stride;
  // depth at (y, x) of the feature map: bilinear, align_corners=False (area_pixel_compute_source_index)
  const float sy = fmaxf(((float)y + 0.5f) * ((float)dh / (float)h) - 0.5f, 0.f);
  const float sx = fmaxf(((float)x + 0.5f) * ((float)dw / (float)w) - 0.5f, 0.f);
  const int y0 = min((int)sy, dh - 1), x0 = min((int)sx, dw - 1);
  const int y1 = min(y0 + 1, dh - 1), x1 = min(x0 + 1, dw - 1);
  const float ly = sy - y0, lx = sx - x0;
  const float d = (1.f - ly) * ((1.f - lx) * depth[(long long)y0 * dw + x0] + lx * depth[(long long)y0 * dw + x1]) +
                  ly * ((1.f - lx) * depth[(long long)y1 * dw + x0] + lx * depth[(long long)y1 * dw + x1]);
  float dx = bf_scale / d;
  if (isinf(dx)) dx = 0.f;
  // grid = (-1 + 2x/w + dx*2/w, -1 + 2y/h); unnormalise (align_corners=False): ((g+1)*size - 1)/2
  const float gx = -1.f + (float)x * (2.f / (float)w) + dx * 2.f / (float)w;
  const float gy = -1.f + (float)y * (2.f / (float)h);
  float fx = ((gx + 1.f) * (float)w - 1.f) * 0.5f;
  float fy = ((gy + 1.f) * (float)h - 1.f) * 0.5f;
  fx = fminf(fmaxf(fx, 0.f), (float)(w - 1));   // padding_mode="border": clip coordinates
  fy = fminf(fmaxf(fy, 0.f), (float)(h - 1));
  const int ix0 = (int)floorf(fx), iy0 = (int)floorf(fy);
  const int ix1 = min(ix0 + 1, w - 1), iy1 = min(iy0 + 1, h - 1);
  const float tx = fx - ix0, ty = fy - iy0;
  const T* base = in + (long long)b * h * w * cs_in + cv * 8;
  float a[8], bb[8], c[8], dd[8], o[8];
  Elem<T>::ld8_nc(base + ((long long)iy0 * w + ix0) * cs_in, a);
  Elem<T>::ld8_nc(base + ((long long)iy0 * w + ix1) * cs_in, bb);
  Elem<T>::ld8_nc(base + ((long long)iy1 * w + ix0) * cs_in, c);
  Elem<T>::ld8_nc(base + ((long long)iy1 * w + ix1) * cs_in, dd);
#pragma unroll
  for (int k = 0; k < 8; ++k)
    o[k] = (1.f - ty) * ((1.f - tx) * a[k] + tx * bb[k]) + ty * ((1.f - tx) * c[k] + tx * dd[k]);
  Elem<T>::st8(out + (((long long)b * h + y) * w + x) * cs_out + cv * 8, o);
}
}  // namespace

namespace {
int virtual_view(const void* in, void* out, const float* depth, int dtype, int B, int h, int w, int C, int cs_in,
                 int cs_out, int dh, int dw, float bf_scale, long long depth_stride, void* stream) {
  const int CV = (C + 7) / 8;
  const long long total = (long long)B * h * w * CV;
  OCCD_DISPATCH_DTYPE(dtype, T, (virtual_view_kernel<T><<<(unsigned)((total + 255) / 256), 256, 0,
                                                           (cudaStream_t)stream>>>(
                                     (const T*)in, (T*)out, depth, B, h, w, CV, cs_in, cs_out, dh, dw, bf_scale,
                                     depth_stride)));
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}
}  // namespace

extern "C" int occd_virtual_view_fwd(const void* in, void* out, const float* depth, int dtype, int B, int h, int w,
                                     int C, int cs_in, int cs_out, int dh, int dw, float bf_scale, void* stream) {
  OCCD_CHECK_ARG(in && out && depth && B > 0 && h > 0 && w > 0 && C > 0 && dh > 0 && dw > 0 && cs_in % 8 == 0 &&
                 cs_out % 8 == 0, "occd_virtual_view_fwd: args");
  OCCD_CHECK_ARG((C + 7) / 8 * 8 <= cs_in && (C + 7) / 8 * 8 <= cs_out, "occd_virtual_view_fwd: channel window");
  return virtual_view(in, out, depth, dtype, B, h, w, C, cs_in, cs_out, dh, dw, bf_scale, 0, stream);
}

extern "C" int occd_virtual_view_items_fwd(const void* in, void* out, const float* depth, int dtype, int B, int h,
                                           int w, int C, int cs_in, int cs_out, int dh, int dw, float bf_scale,
                                           long long depth_stride, void* stream) {
  OCCD_CHECK_ARG(in && out && depth && B > 0 && h > 0 && w > 0 && C > 0 && dh > 0 && dw > 0 && cs_in % 8 == 0 &&
                 cs_out % 8 == 0, "occd_virtual_view_items_fwd: args");
  OCCD_CHECK_ARG((C + 7) / 8 * 8 <= cs_in && (C + 7) / 8 * 8 <= cs_out, "occd_virtual_view_items_fwd: channel window");
  OCCD_CHECK_ARG(depth_stride == 0 || depth_stride >= (long long)dh * dw,
                 "occd_virtual_view_items_fwd: depth_stride must be 0 (item 0's depth map for every item) or at least "
                 "dh * dw (one map per item)");
  return virtual_view(in, out, depth, dtype, B, h, w, C, cs_in, cs_out, dh, dw, bf_scale, depth_stride, stream);
}
