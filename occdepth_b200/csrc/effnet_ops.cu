// Bandwidth-bound pieces of the 2D backbone (channels-last bf16):
//   depthwise KxK conv + folded BN + SiLU + squeeze (global-average-pool partial sums)
//   squeeze-excite MLP (reduce FC + SiLU + expand FC + sigmoid)
//   SE gate folded into the following 1x1 projection's weights (per image)
//   bilinear resize with align_corners=True (UpSampleBN, unet2d.py:39-44)
//   the same resize applied to the nine per-tap products of UpSampleBN's conv1, summed on the fine grid
// replaces geffnet DepthwiseSeparableConv / InvertedResidual internals (conv_dw, bn, act, se) as iterated by
// Encoder.forward (unet2d.py:188-196) and F.interpolate in UpSampleBN.forward.
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include "common.cuh"
#include "dwconv_tiled.cuh"
#include "../../include/occdepth_b200.h"

namespace {

constexpr int kDwThreads = 256;
constexpr int kDwPX = 4;    // consecutive output pixels per thread (register blocking along W)
constexpr int kDwRows = 4;  // output rows per block (amortises the squeeze atomics)

// blockDim = (CVB, 256/CVB): threadIdx.x owns one 8-channel vector (coalesced CVB*16-byte segments),
// threadIdx.y owns kDwPX consecutive output pixels of one image row.  Per filter row the thread loads the
// (kDwPX-1)*S + K input vectors it needs ONCE and reuses them across the K taps and kDwPX outputs (2.5x fewer
// loads/unpacks than one-pixel-per-thread for K = 5).  CVB in {8,16,32} is picked per layer so narrow layers
// (C = 64) keep every lane busy.  The squeeze (global-average-pool sum) is accumulated in registers, reduced
// across threadIdx.y in shared memory and added to pool[b][c] as a 64-bit FIXED-POINT integer (2^-24 units): integer
// atomics commute exactly, so the SE gates (and everything downstream) are bit-reproducible run to run -- float
// atomics are not.
template <typename T, int K, int S, int CVB>
__global__ void __launch_bounds__(kDwThreads)
dwconv_kernel(const T* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
              T* __restrict__ out, long long* __restrict__ pool, int H, int W, int OH, int OW, int C,
              int cs_in, int cs_out, int pad_top, int pad_left, int act) {
  constexpr int PY = kDwThreads / CVB;
  constexpr int NIN = (kDwPX - 1) * S + K;
  __shared__ float red[PY][CVB * 8 + 1];
  const int tx = threadIdx.x % CVB, ty = threadIdx.x / CVB;
  const int c0 = (blockIdx.y * CVB + tx) * 8;
  const bool cvalid = c0 < C;
  const int row_blocks = (OH + kDwRows - 1) / kDwRows;
  const int b = blockIdx.z / row_blocks;
  const int ox0 = (blockIdx.x * PY + ty) * kDwPX;
  float psum[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) psum[i] = 0.f;
#pragma unroll 1
  for (int ry = 0; ry < kDwRows; ++ry) {
  const int oy = (blockIdx.z % row_blocks) * kDwRows + ry;
  if (cvalid && ox0 < OW && oy < OH) {
    float acc[kDwPX][8];
    {
      float bv[8];
      *reinterpret_cast<float4*>(bv) = __ldg(reinterpret_cast<const float4*>(bias + c0));
      *reinterpret_cast<float4*>(bv + 4) = __ldg(reinterpret_cast<const float4*>(bias + c0 + 4));
#pragma unroll
      for (int p = 0; p < kDwPX; ++p)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[p][i] = bv[i];
    }
    const T* inb = in + (long long)b * H * W * cs_in + c0;
    const float* wc = w + c0;
    const int ix0 = ox0 * S - pad_left;
#pragma unroll
    for (int ky = 0; ky < K; ++ky) {
      const int iy = oy * S - pad_top + ky;
      if (iy < 0 || iy >= H) continue;
      const T* row = inb + (long long)iy * W * cs_in;
      float xin[NIN][8];
#pragma unroll
      for (int j = 0; j < NIN; ++j) {
        const int ix = ix0 + j;
        if (ix >= 0 && ix < W) {
          Elem<T>::ld8_nc(row + (long long)ix * cs_in, xin[j]);
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) xin[j][i] = 0.f;
        }
      }
#pragma unroll
      for (int kx = 0; kx < K; ++kx) {
        float wv[8];
        const float* wp = wc + (long long)(ky * K + kx) * C;
        *reinterpret_cast<float4*>(wv) = __ldg(reinterpret_cast<const float4*>(wp));
        *reinterpret_cast<float4*>(wv + 4) = __ldg(reinterpret_cast<const float4*>(wp + 4));
#pragma unroll
        for (int p = 0; p < kDwPX; ++p)
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[p][i] = fmaf(xin[p * S + kx][i], wv[i], acc[p][i]);
      }
    }
#pragma unroll
    for (int p = 0; p < kDwPX; ++p) {
      const int ox = ox0 + p;
      if (ox >= OW) break;
      apply_act8(acc[p], act);
      // store, and pool what the next layer will actually read (the rounded activation)
      Elem<T>::st8_rb(out + (((long long)b * OH + oy) * OW + ox) * cs_out + c0, acc[p]);
      if (pool) {
#pragma unroll
        for (int i = 0; i < 8; ++i) psum[i] += acc[p][i];
      }
    }
  }
  }
  if (pool) {
#pragma unroll
    for (int i = 0; i < 8; ++i) red[ty][tx * 8 + i] = psum[i];
    __syncthreads();
    if (ty == 0 && cvalid) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float s = 0.f;
#pragma unroll
        for (int y = 0; y < PY; ++y) s += red[y][tx * 8 + i];
        atomicAdd(reinterpret_cast<unsigned long long*>(pool) + (long long)b * C + c0 + i,
                  (unsigned long long)__float2ll_rn(s * 16777216.f));
      }
    }
  }
}

// squeeze-excite MLP in two wide launches (the FC weights are MBs for the late stages: one block cannot stream them)
//   hidden[b][r] = silu(b1[r] + <w1[r], pool[b] / HW>)          grid (R, B), one block per hidden unit
//   gate[b][c]   = sigmoid(b2[c] + sum_r w2t[r][c] hidden[b][r]) grid (ceil(C/256), B); also clears pool
__global__ void __launch_bounds__(128)
se_fc1_kernel(const long long* __restrict__ pool, float inv_hw, const float* __restrict__ w1,
              const float* __restrict__ b1, float* __restrict__ hidden, int C, int R) {
  pdl_wait();
  __shared__ float red[4];
  const int r = blockIdx.x, b = blockIdx.y;
  const float* wr = w1 + (long long)r * C;
  const long long* pb = pool + (long long)b * C;
  float s = 0.f;
  for (int c = threadIdx.x; c < C; c += 128)
    s = fmaf(__ldg(wr + c), (float)((double)pb[c] * (1.0 / 16777216.0)), s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    const float v = (red[0] + red[1] + red[2] + red[3]) * inv_hw + b1[r];
    hidden[(long long)b * R + r] = __fdividef(v, 1.f + __expf(-v));
  }
}

__global__ void __launch_bounds__(256)
se_fc2_kernel(long long* __restrict__ pool, const float* __restrict__ hidden, const float* __restrict__ w2t,
              const float* __restrict__ b2, float* __restrict__ gate, int C, int R) {
  extern __shared__ float hid[];
  const int b = blockIdx.y;
  for (int r = threadIdx.x; r < R; r += 256) hid[r] = hidden[(long long)b * R + r];
  __syncthreads();
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= C) return;
  float s = b2[c];
  for (int r = 0; r < R; ++r) s = fmaf(__ldg(w2t + (long long)r * C + c), hid[r], s);
  gate[(long long)b * C + c] = __fdividef(1.f, 1.f + __expf(-s));
  pool[(long long)b * C + c] = 0;  // ready for the next forward
}

// fused: gate for a strip of 256 input channels (second FC + sigmoid), then that strip of the projection
// weights scaled and packed to bf16 for `rows_per_block` output rows.  grid (ceil(Kpad/256), row blocks)
template <typename T>
__global__ void __launch_bounds__(256)
se_fc2_fold_kernel(long long* __restrict__ pool, const float* __restrict__ hidden, const float* __restrict__ w2t,
                   const float* __restrict__ b2, const float* __restrict__ master, T* __restrict__ out,
                   int C, int R, int rows, int Kpad, int rows_per_block) {
  pdl_wait();
  extern __shared__ float hid[];
  const int img = blockIdx.z;   // one weight set per image
  for (int r = threadIdx.x; r < R; r += 256) hid[r] = hidden[(long long)img * R + r];
  __syncthreads();
  const int k = blockIdx.x * 256 + threadIdx.x;
  if (k >= Kpad) return;
  float g = 0.f;
  if (k < C) {
    float s = b2[k];
    for (int r = 0; r < R; ++r) s = fmaf(__ldg(w2t + (long long)r * C + k), hid[r], s);
    g = __fdividef(1.f, 1.f + __expf(-s));
    if (blockIdx.y == 0) pool[(long long)img * C + k] = 0;  // ready for the next forward
  }
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(rows, r0 + rows_per_block);
  T* o = out + (long long)img * rows * Kpad;
  for (int r = r0; r < r1; ++r)
    o[(long long)r * Kpad + k] = Elem<T>::cvt(__ldg(master + (long long)r * Kpad + k) * g);
}

// out[row][k] = bf16(master[row][k] * gate[k])  (k < C), rows = Cout_pad, row length Kpad
template <typename T>
__global__ void scale_weights_kernel(const float* __restrict__ master, const float* __restrict__ gate,
                                     T* __restrict__ out, int rows, int Kpad, int C) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 8;  // Kpad % 8 == 0
  if (i >= (long long)rows * Kpad) return;
  const int k = (int)(i % Kpad);
  float m[8], g[8];
  *reinterpret_cast<float4*>(m) = __ldg(reinterpret_cast<const float4*>(master + i));
  *reinterpret_cast<float4*>(m + 4) = __ldg(reinterpret_cast<const float4*>(master + i + 4));
#pragma unroll
  for (int j = 0; j < 8; ++j) g[j] = (k + j < C) ? gate[k + j] : 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) m[j] *= g[j];
  Elem<T>::st8(out + i, m);
}

// bilinear, align_corners=True; in [B][h][w][cs_in] -> out [B][OH][OW][cs_out] (channel windows), C % 8 == 0 padded
template <typename T>
__global__ void upsample_bilinear_kernel(const T* __restrict__ in, T* __restrict__ out, int B,
                                         int h, int w, int OH, int OW, int CV, int cs_in, int in_off, int cs_out,
                                         int out_off, float sy, float sx) {
  pdl_wait();
  // grid: x covers one output row's (column, channel-vector) pairs, y = (image, output row): 32-bit index math only
  // (a flat 64-bit index would cost three software 64-bit divisions per 32-byte store)
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (unsigned)(OW * CV)) return;
  const int ox = (int)(i / (unsigned)CV);
  const int cv = (int)(i - (unsigned)ox * (unsigned)CV);
  const int b = (int)(blockIdx.y / (unsigned)OH);
  const int oy = (int)(blockIdx.y - (unsigned)b * (unsigned)OH);
  const float fy = sy * oy, fx = sx * ox;
  int y0 = (int)fy, x0 = (int)fx;
  y0 = min(y0, h - 1); x0 = min(x0, w - 1);
  const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
  const float ly = fy - y0, lx = fx - x0;
  const float hy = 1.f - ly, hx = 1.f - lx;
  const T* base = in + (long long)b * h * w * cs_in + in_off + cv * 8;
  float a[8], bb[8], c[8], d[8], o[8];
  Elem<T>::ld8_nc(base + ((long long)y0 * w + x0) * cs_in, a);
  Elem<T>::ld8_nc(base + ((long long)y0 * w + x1) * cs_in, bb);
  Elem<T>::ld8_nc(base + ((long long)y1 * w + x0) * cs_in, c);
  Elem<T>::ld8_nc(base + ((long long)y1 * w + x1) * cs_in, d);
#pragma unroll
  for (int k = 0; k < 8; ++k) o[k] = hy * (hx * a[k] + lx * bb[k]) + ly * (hx * c[k] + lx * d[k]);
  Elem<T>::st8(out + (((long long)b * OH + oy) * OW + ox) * cs_out + out_off + cv * 8, o);
}

// UpSampleBN conv1 with the resize moved behind the 3x3 taps: bilinear resizing commutes with a channel mix, so the
// up half of the conv runs as one 1x1 GEMM on the coarse map, Y[b][i][j][t*tap_stride + c] = W_t x[b][i][j] for the
// nine taps t = (dy+1)*3 + (dx+1), and this kernel resizes and sums them on the fine grid:
//   out[b][p][c] = act(pre[b][p][c] + sum_t [p+t inside OH x OW] bilinear_ac(Y_t)(p+t)[c])
// The bilinear weights and the padding mask both factor into rows and columns.  A thread owns one (output column,
// channel vector) and walks a strip of output rows; per dy it keeps the column-summed partials
//   H_dy(i) = sum_dx [ox+dx inside] ((1-lx) Y_t[i][x0] + lx Y_t[i][x1])
// of the two coarse rows its current output row reads.  Consecutive output rows share those rows, so each partial
// is built once per strip (6 vector loads) instead of costing 36 loads per output vector.
template <typename T>
__global__ void __launch_bounds__(256)
upsample_tapsum_kernel(const T* __restrict__ y, const T* pre, T* out, int h, int w, int OH, int OW, int CV,
                       int cs_y, int y_off, int tap_stride, int cs_pre, int pre_off, int cs_out, int out_off,
                       int strip_rows, int n_strips, int act, float sy, float sx) {
  pdl_wait();
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (unsigned)(OW * CV)) return;
  const int ox = (int)(i / (unsigned)CV);
  const int cv = (int)(i - (unsigned)ox * (unsigned)CV);
  const int b = (int)(blockIdx.y / (unsigned)n_strips);
  const int oy0 = (int)(blockIdx.y - (unsigned)b * (unsigned)n_strips) * strip_rows;
  const int oy1 = min(oy0 + strip_rows, OH);
  // per dx: offsets of the two coarse columns (the fine column ox+dx is resized from) and their weights
  int xo0[3], xo1[3];
  float wx0[3], wx1[3];
  bool xin[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const int fx = ox + d - 1;
    xin[d] = fx >= 0 && fx < OW;
    const float f = sx * (float)max(fx, 0);
    const int x0 = min((int)f, w - 1), x1 = min(x0 + 1, w - 1);
    wx1[d] = f - (float)x0;
    wx0[d] = 1.f - wx1[d];
    xo0[d] = x0 * cs_y;
    xo1[d] = x1 * cs_y;
  }
  const T* yb = y + (long long)b * h * w * cs_y + y_off + cv * 8;
  // hr[d][k]: H_dy of coarse row row[d] + k (k = 1 clamped to the last row); row[d] = -2: nothing held yet
  float hr[3][2][8];
  int row[3] = {-2, -2, -2};
  auto hsum = [&](int d, int r, float* dst) {
#pragma unroll
    for (int k = 0; k < 8; ++k) dst[k] = 0.f;
    const T* yr = yb + r * w * cs_y + 3 * d * tap_stride;
#pragma unroll
    for (int e = 0; e < 3; ++e) {
      if (!xin[e]) continue;
      float a[8], c[8];
      Elem<T>::ld8_nc(yr + e * tap_stride + xo0[e], a);
      Elem<T>::ld8_nc(yr + e * tap_stride + xo1[e], c);
#pragma unroll
      for (int k = 0; k < 8; ++k) dst[k] += wx0[e] * a[k] + wx1[e] * c[k];
    }
  };
  const int pix0 = b * OH * OW;   // 32-bit: OCCD_CHECK_ARG bounds B*OH*OW*cs
#pragma unroll 1
  for (int oy = oy0; oy < oy1; ++oy) {
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const int fy = oy + d - 1;
      if (fy < 0 || fy >= OH) continue;
      const float f = sy * (float)fy;
      const int y0 = min((int)f, h - 1);
      const float ly = f - (float)y0;
      if (y0 != row[d]) {
        if (y0 == row[d] + 1) {
#pragma unroll
          for (int k = 0; k < 8; ++k) hr[d][0][k] = hr[d][1][k];
        } else {
          hsum(d, y0, hr[d][0]);
        }
        hsum(d, min(y0 + 1, h - 1), hr[d][1]);
        row[d] = y0;
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += (1.f - ly) * hr[d][0][k] + ly * hr[d][1][k];
    }
    const int p = pix0 + oy * OW + ox;
    if (pre) {
      float r[8];
      Elem<T>::ld8(pre + p * cs_pre + pre_off + cv * 8, r);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += r[k];
    }
    apply_act8(acc, act);
    Elem<T>::st8(out + p * cs_out + out_off + cv * 8, acc);
  }
}

}  // namespace

template <typename T>
static int dwconv2d_direct(const void* in, const float* w, const float* bias, void* out, long long* pool, int B,
                           int H, int W, int OH, int OW, int C, int cs_in, int cs_out, int K, int stride,
                           int pad_top, int pad_left, int act, void* stream) {
  OCCD_CHECK_ARG(in && w && bias && out && B > 0 && H > 0 && W > 0 && OH > 0 && OW > 0, "occd_dwconv2d_fwd: args");
  OCCD_CHECK_ARG(C > 0 && C % 8 == 0 && cs_in % 8 == 0 && cs_out % 8 == 0 && cs_in >= C && cs_out >= C,
                 "occd_dwconv2d_fwd: channels must be a multiple of 8");
  OCCD_CHECK_ARG((long long)B * ((OH + kDwRows - 1) / kDwRows) <= 65535, "occd_dwconv2d_fwd: B*OH too large");
  OCCD_CHECK_ARG(K == 3 || K == 5, "occd_dwconv2d_fwd: kernel size must be 3 or 5");
  const int CV = C / 8;
  // lanes per pixel: the candidate in {8,16,32} with the least padding (ties -> widest)
  int cvb = 32, best = -1;
  for (int c = 32; c >= 8; c >>= 1) {
    const int padded = (CV + c - 1) / c * c;
    if (best < 0 || padded < best) { best = padded; cvb = c; }
  }
  OCCD_CHECK_ARG(stride == 1 || stride == 2, "occd_dwconv2d_fwd: stride must be 1 or 2");
  const int py = kDwThreads / cvb;
  dim3 grid((OW + py * kDwPX - 1) / (py * kDwPX), (CV + cvb - 1) / cvb, B * ((OH + kDwRows - 1) / kDwRows)), block(kDwThreads);
  cudaStream_t st = (cudaStream_t)stream;
  const T* i = (const T*)in;
  T* o = (T*)out;
#define OCCD_DW(K_, S_, CVB_)                                                                                   \
  dwconv_kernel<T, K_, S_, CVB_><<<grid, block, 0, st>>>(i, w, bias, o, pool, H, W, OH, OW, C, cs_in, cs_out,   \
                                                          pad_top, pad_left, act)
#define OCCD_DW_CVB(K_, S_)                                                                                     \
  { if (cvb == 8) OCCD_DW(K_, S_, 8); else if (cvb == 16) OCCD_DW(K_, S_, 16); else OCCD_DW(K_, S_, 32); }
  if (K == 3 && stride == 1) OCCD_DW_CVB(3, 1)
  else if (K == 3) OCCD_DW_CVB(3, 2)
  else if (stride == 1) OCCD_DW_CVB(5, 1)
  else OCCD_DW_CVB(5, 2)
#undef OCCD_DW_CVB
#undef OCCD_DW
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

extern "C" int occd_dwconv2d_fwd(const void* in, const float* w, const float* bias, void* out, long long* pool,
                                 int dtype, int B, int H, int W, int OH, int OW, int C, int cs_in, int cs_out, int K,
                                 int stride, int pad_top, int pad_left, int act, void* stream) {
  OCCD_DISPATCH_DTYPE(dtype, T, return dwconv2d_direct<T>(in, w, bias, out, pool, B, H, W, OH, OW, C, cs_in, cs_out, K,
                                                         stride, pad_top, pad_left, act, stream));
}


namespace {

template <typename T, int K, int S, int CVB, int TH, int PXV = 4>
int launch_dw_tiled(const dwt::Args& a, int B, cudaStream_t st) {
  using C_ = dwt::Cfg<T, K, S, CVB, TH, PXV>;
  static bool attr_set[64] = {false};  // per instantiation, per device
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (!attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(dwt::dwconv_tiled_kernel<T, K, S, CVB, TH, PXV>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C_::kSmemBytes);
    if (e != cudaSuccess) { occd_set_last_error(cudaGetErrorString(e)); return OCCD_ERR_CUDA; }
    attr_set[dev] = true;
  }
  const int tiles_y = (a.OH + TH - 1) / TH;
  dim3 grid(a.tiles_x * tiles_y, (a.C + C_::CT - 1) / C_::CT, B);
  OCCD_LAUNCH_CHECKED((dwt::dwconv_tiled_kernel<T, K, S, CVB, TH, PXV>), grid, dim3(C_::NT), C_::kSmemBytes, st, a);
  return OCCD_OK;
}

template <typename T, int K, int S>
int launch_dw_tiled_ks(const dwt::Args& a, int B, dwt::Choice ch, cudaStream_t st) {
  if (ch.cvb == 4) {   // 16 rows per pass: TH = 16 only
    if constexpr (sizeof(T) == 4 && S == 1) {
      // fp32, stride 1: 8 outputs per thread / 128-thread CTAs (the stride-2 layers keep 4; tools/dw_bench.py
      // compares the variants).  OCCD_DW_PX=4 forces 4 (experiment hook)
      static const bool px4 = [] { const char* e = getenv("OCCD_DW_PX"); return e && atoi(e) == 4; }();
      if (!px4) return launch_dw_tiled<T, K, S, 4, 16, 8>(a, B, st);
    }
    return launch_dw_tiled<T, K, S, 4, 16>(a, B, st);
  }
  if constexpr (sizeof(T) == 2) {
    if (ch.th == 16) return launch_dw_tiled<T, K, S, 8, 16>(a, B, st);
    return launch_dw_tiled<T, K, S, 8, 8>(a, B, st);
  }
  occd_set_last_error("occd_dwconv2d_tiled_fwd: internal tile choice");
  return OCCD_ERR_ARG;
}

template <typename T>
int dw_tiled_dispatch(const dwt::Args& a, int B, int K, int stride, dwt::Choice ch, cudaStream_t st) {
  if (K == 3 && stride == 1) return launch_dw_tiled_ks<T, 3, 1>(a, B, ch, st);
  if (K == 3) return launch_dw_tiled_ks<T, 3, 2>(a, B, ch, st);
  if (stride == 1) return launch_dw_tiled_ks<T, 5, 1>(a, B, ch, st);
  return launch_dw_tiled_ks<T, 5, 2>(a, B, ch, st);
}

}  // namespace

// Shared-memory-tiled variant of occd_dwconv2d_fwd (same arguments, same results up to fp32 summation order).
extern "C" int occd_dwconv2d_tiled_fwd(const void* in, const float* w, const float* bias, void* out, long long* pool,
                                       int dtype, int B, int H, int W, int OH, int OW, int C, int cs_in, int cs_out,
                                       int K, int stride, int pad_top, int pad_left, int act, void* stream) {
  OCCD_CHECK_ARG(dtype == OCCD_DTYPE_F32 || dtype == OCCD_DTYPE_BF16, "occd_dwconv2d_tiled_fwd: dtype");
  OCCD_CHECK_ARG(in && w && bias && out && B > 0 && H > 0 && W > 0 && OH > 0 && OW > 0, "occd_dwconv2d_tiled_fwd: args");
  OCCD_CHECK_ARG(C > 0 && C % 8 == 0 && cs_in % 8 == 0 && cs_out % 8 == 0 && cs_in >= C && cs_out >= C,
                 "occd_dwconv2d_tiled_fwd: channels must be a multiple of 8");
  OCCD_CHECK_ARG(K == 3 || K == 5, "occd_dwconv2d_tiled_fwd: kernel size must be 3 or 5");
  OCCD_CHECK_ARG(stride == 1 || stride == 2, "occd_dwconv2d_tiled_fwd: stride must be 1 or 2");
  OCCD_CHECK_ARG(B <= 65535 && (C + 31) / 32 <= 65535, "occd_dwconv2d_tiled_fwd: B/C too large");
  static int n_sms = 0;
  if (n_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n_sms <= 0) n_sms = 132;
  }
  dwt::Args a;
  a.in = in; a.w = w; a.bias = bias; a.out = out; a.pool = pool;
  a.H = H; a.W = W; a.OH = OH; a.OW = OW; a.C = C; a.cs_in = cs_in; a.cs_out = cs_out;
  a.pad_top = pad_top; a.pad_left = pad_left; a.act = act; a.tiles_x = (OW + dwt::kTW - 1) / dwt::kTW;
  const dwt::Choice ch = dwt::choose(B, OH, OW, C, stride, n_sms, dtype == OCCD_DTYPE_F32 ? 4 : 2);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == OCCD_DTYPE_F32) return dw_tiled_dispatch<float>(a, B, K, stride, ch, st);
  return dw_tiled_dispatch<__nv_bfloat16>(a, B, K, stride, ch, st);
}

extern "C" int occd_se_gate_fwd(long long* pool, float inv_hw, const float* w1, const float* b1, const float* w2t,
                                const float* b2, float* gate, int B, int C, int R, void* stream) {
  OCCD_CHECK_ARG(pool && w1 && b1 && w2t && b2 && gate && B > 0 && C > 0 && R > 0, "occd_se_gate_fwd: args");
  OCCD_CHECK_ARG(R <= 8192 && B <= 65535, "occd_se_gate_fwd: R/B too large");
  // hidden activations live right behind the gate: gate buffer must hold B*C + B*R floats
  float* hidden = gate + (long long)B * C;
  se_fc1_kernel<<<dim3(R, B), 128, 0, (cudaStream_t)stream>>>(pool, inv_hw, w1, b1, hidden, C, R);
  OCCD_CHECK_LAUNCH();
  se_fc2_kernel<<<dim3((C + 255) / 256, B), 256, R * sizeof(float), (cudaStream_t)stream>>>(pool, hidden, w2t, b2,
                                                                                             gate, C, R);
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

extern "C" int occd_scale_weights(const float* master, const float* gate, void* out, int wdtype, int rows, int Kpad,
                                  int C, void* stream) {
  OCCD_CHECK_ARG(master && gate && out && rows > 0 && Kpad > 0 && C > 0 && C <= Kpad, "occd_scale_weights: args");
  OCCD_CHECK_ARG(Kpad % 8 == 0, "occd_scale_weights: Kpad must be a multiple of 8");
  const long long total = (long long)rows * Kpad / 8;
  OCCD_DISPATCH_DTYPE(wdtype, T, (scale_weights_kernel<T><<<(unsigned)((total + 255) / 256), 256, 0,
                                                             (cudaStream_t)stream>>>(master, gate, (T*)out, rows,
                                                                                     Kpad, C)));
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

extern "C" int occd_upsample_bilinear_ac(const void* in, void* out, int dtype, int B, int h, int w, int OH, int OW,
                                         int C, int cs_in, int in_off, int cs_out, int out_off, void* stream) {
  OCCD_CHECK_ARG(in && out && B > 0 && h > 0 && w > 0 && OH > 0 && OW > 0 && C > 0, "occd_upsample_bilinear_ac: args");
  OCCD_CHECK_ARG(cs_in % 8 == 0 && cs_out % 8 == 0 && in_off % 8 == 0 && out_off % 8 == 0,
                 "occd_upsample_bilinear_ac: alignment");
  const int CV = (C + 7) / 8;
  OCCD_CHECK_ARG(in_off + CV * 8 <= cs_in && out_off + CV * 8 <= cs_out, "occd_upsample_bilinear_ac: channel window");
  const float sy = OH > 1 ? (float)(h - 1) / (float)(OH - 1) : 0.f;
  const float sx = OW > 1 ? (float)(w - 1) / (float)(OW - 1) : 0.f;
  OCCD_CHECK_ARG((long long)OW * CV < (1LL << 31) && (long long)B * OH <= 65535, "occd_upsample_bilinear_ac: extent");
  OCCD_DISPATCH_DTYPE(dtype, T, OCCD_LAUNCH_CHECKED(upsample_bilinear_kernel<T>,
                                                    dim3((unsigned)((OW * CV + 255) / 256), (unsigned)(B * OH)),
                                                    dim3(256), 0, (cudaStream_t)stream, (const T*)in, (T*)out, B, h, w,
                                                    OH, OW, CV, cs_in, in_off, cs_out, out_off, sy, sx));
  return OCCD_OK;
}

extern "C" int occd_upsample_tapsum_ac(const void* y, const void* pre, void* out, int dtype, int B, int h, int w,
                                       int OH, int OW, int C, int cs_y, int y_off, int tap_stride, int cs_pre,
                                       int pre_off, int cs_out, int out_off, int act, void* stream) {
  OCCD_CHECK_ARG(y && out && B > 0 && h > 0 && w > 0 && OH > 0 && OW > 0 && C > 0, "occd_upsample_tapsum_ac: args");
  OCCD_CHECK_ARG(act >= ACT_NONE && act <= ACT_SIGMOID, "occd_upsample_tapsum_ac: act");
  OCCD_CHECK_ARG(cs_y % 8 == 0 && y_off % 8 == 0 && tap_stride % 8 == 0 && cs_out % 8 == 0 && out_off % 8 == 0 &&
                     (!pre || (cs_pre % 8 == 0 && pre_off % 8 == 0)),
                 "occd_upsample_tapsum_ac: alignment");
  const int CV = (C + 7) / 8;
  OCCD_CHECK_ARG(y_off >= 0 && out_off >= 0 && tap_stride >= CV * 8 &&
                     (long long)y_off + 8LL * tap_stride + CV * 8 <= cs_y && out_off + CV * 8 <= cs_out &&
                     (!pre || (pre_off >= 0 && pre_off + CV * 8 <= cs_pre)),
                 "occd_upsample_tapsum_ac: channel window");
  OCCD_CHECK_ARG((long long)h * w * cs_y < (1LL << 31) && (long long)B * OH * OW * cs_out < (1LL << 31) &&
                     (!pre || (long long)B * OH * OW * cs_pre < (1LL << 31)) && (long long)OW * CV < (1LL << 31),
                 "occd_upsample_tapsum_ac: extent");
  // strips of output rows: long enough that consecutive rows reuse their coarse-row partials, short enough that
  // the grid still fills the GPU a few times over (2^19 threads)
  const long long per_row = (long long)B * OW * CV;
  int n_strips = (int)std::min<long long>(OH, std::max<long long>(1, ((1LL << 19) + per_row - 1) / per_row));
  const int strip_rows = (OH + n_strips - 1) / n_strips;
  n_strips = (OH + strip_rows - 1) / strip_rows;
  OCCD_CHECK_ARG((long long)B * n_strips <= 65535, "occd_upsample_tapsum_ac: extent");
  const float sy = OH > 1 ? (float)(h - 1) / (float)(OH - 1) : 0.f;
  const float sx = OW > 1 ? (float)(w - 1) / (float)(OW - 1) : 0.f;
  OCCD_DISPATCH_DTYPE(dtype, T, OCCD_LAUNCH_CHECKED(upsample_tapsum_kernel<T>,
                                                    dim3((unsigned)((OW * CV + 255) / 256), (unsigned)(B * n_strips)),
                                                    dim3(256), 0, (cudaStream_t)stream, (const T*)y, (const T*)pre,
                                                    (T*)out, h, w, OH, OW, CV, cs_y, y_off, tap_stride, cs_pre, pre_off,
                                                    cs_out, out_off, strip_rows, n_strips, act, sy, sx));
  return OCCD_OK;
}

extern "C" int occd_se_gate_fold_fwd(long long* pool, float inv_hw, const float* w1, const float* b1, const float* w2t,
                                     const float* b2, float* hidden, const float* master, void* wout, int wdtype,
                                     int B, int C, int R, int rows, int Kpad, void* stream) {
  OCCD_CHECK_ARG(pool && w1 && b1 && w2t && b2 && hidden && master && wout && C > 0 && R > 0 && rows > 0 &&
                 Kpad >= C && R <= 8192, "occd_se_gate_fold_fwd: args");
  cudaStream_t st = (cudaStream_t)stream;
  OCCD_CHECK_ARG(B >= 1 && B <= 65535, "occd_se_gate_fold_fwd: B");
  OCCD_LAUNCH_CHECKED(se_fc1_kernel, dim3(R, B), dim3(128), 0, st, (const long long*)pool, inv_hw, w1, b1, hidden, C, R);
  const int kblocks = (Kpad + 255) / 256;
  int rows_per_block = rows;
  while (rows_per_block > 16 && B * kblocks * ((rows + rows_per_block - 1) / rows_per_block) < 296) rows_per_block /= 2;
  dim3 grid(kblocks, (rows + rows_per_block - 1) / rows_per_block, B);
  OCCD_DISPATCH_DTYPE(wdtype, T, OCCD_LAUNCH_CHECKED(se_fc2_fold_kernel<T>, grid, dim3(256), R * sizeof(float), st, pool,
                                                     (const float*)hidden, w2t, b2, master, (T*)wout, C, R, rows, Kpad,
                                                     rows_per_block));
  return OCCD_OK;
}
