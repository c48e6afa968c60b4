// Loss sums of the reference's evaluation step (OccDepth.step, occdepth/models/OccDepth.py:378-533) on the device.
// Every loss the step logs is a ratio of a few sums over voxels, relation entries or depth pixels; these kernels
// accumulate those sums, and occdepth_b200/losses.py forms the losses from them.  The reference instead softmaxes the
// logits, then masks and reduces the whole probability tensor once per class (sem_scal_loss) and once per local
// frustum (the frustum loss); here one pass reads the logits, the labels and the frustum masks once.
//
// Per-element math is fp32.  Each block accumulates its elements in a fixed order (fp32 within a tile, fp64 across
// tiles) and writes one row of partials to the caller's workspace; a second kernel adds the rows in block order to
// the caller's sums.  The grid depends on the shapes only, so the same inputs give bit-identical sums.
#include <math.h>

#include "common.cuh"
#include "ssc_labels.cuh"
#include "../../include/occdepth_b200.h"

namespace {

using namespace ssc_labels;

constexpr int kThreads = 256;                      // also the voxel tile of the SSC kernel
constexpr int kWarps = kThreads / 32;
constexpr int kGrid = OCCD_LOSS_WORK_BLOCKS;
constexpr int kPitch = kThreads + 1;               // probability rows in shared memory, padded against bank conflicts
constexpr int kChunk = 16;                         // per-voxel loads issued together (logit channels, frustum masks)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// sums[k] += sum over b < nblocks of work[b][k], b in order
__global__ void add_partials_kernel(const double* __restrict__ work, int nblocks, int K, double* __restrict__ sums) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < K; k += gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int b = 0; b < nblocks; ++b) s += work[(size_t)b * K + k];
    sums[k] += s;
  }
}

int add_partials(const double* work, int nblocks, int K, double* sums, cudaStream_t st) {
  add_partials_kernel<<<ceil_div(K, kThreads), kThreads, 0, st>>>(work, nblocks, K, sums);
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

// ---- SSC logits against labels ---------------------------------------------------------------------------------
// One tile is kThreads consecutive voxels of one frame, one voxel per thread.  Phase A: each thread softmaxes its
// voxel into shared memory and forms its cross-entropy terms (summed per warp).  Phase B: thread (c, seg) sums class
// c's probabilities over a segment of the tile for the sem-scal sums.  Phase C: for each frustum with a voxel in
// the tile (usually one or two), the same threads sum mask * probability, and thread c adds the segments in order.
struct SscSmem {
  int C, F, nseg;
  size_t facc, red, sp, sg, part, sm, act, bytes;
  __host__ __device__ SscSmem(int C_, int F_) : C(C_), F(F_), nseg(kThreads / C_) {
    facc = 0;                                                         // double [F][C]
    red = facc + sizeof(double) * F * C;                              // double [3][kThreads]
    sp = red + sizeof(double) * 3 * kThreads;                         // float [C][kPitch]
    sg = sp + sizeof(float) * C * kPitch;                             // int [kThreads]
    part = sg + sizeof(int) * kThreads;                               // float [kThreads]
    act = part + sizeof(float) * kThreads;                            // uint32 [2][2]: frustums present, by parity
    sm = act + sizeof(unsigned) * 4;                                  // uint8 [F][kThreads]
    bytes = sm + (size_t)F * kThreads;
  }
};

template <typename L>
__global__ void __launch_bounds__(kThreads) ssc_loss_kernel(
    const float* __restrict__ logits, const L* __restrict__ label, int C, long long S, long long tiles_per_frame,
    long long n_tiles, const float* __restrict__ weight, const float* __restrict__ occ,
    const float* __restrict__ occ_weight, const uint8_t* __restrict__ masks, int F, double* __restrict__ work) {
  extern __shared__ __align__(16) unsigned char smem[];
  const SscSmem L_(C, F);
  double* facc = reinterpret_cast<double*>(smem + L_.facc);
  double* red = reinterpret_cast<double*>(smem + L_.red);
  float* sp = reinterpret_cast<float*>(smem + L_.sp);
  int* sg = reinterpret_cast<int*>(smem + L_.sg);
  float* part = reinterpret_cast<float*>(smem + L_.part);
  unsigned* act = reinterpret_cast<unsigned*>(smem + L_.act);
  uint8_t* sm = smem + L_.sm;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int nseg = L_.nseg, seg_len = (kThreads + nseg - 1) / nseg;
  const bool worker = tid < nseg * C;                    // a (class, segment) pair of phases B and C
  const int my_c = tid / nseg, my_seg = tid % nseg;
  const int v0 = my_seg * seg_len, v1 = min(v0 + seg_len, kThreads);
  for (int i = tid; i < F * C; i += kThreads) facc[i] = 0.0;
  if (tid < 4) act[tid] = 0u;
  double ce = 0.0, ce_w = 0.0, oce = 0.0, oce_w = 0.0;   // lane 0 of each warp
  long long n_valid = 0, n_invalid = 0;
  double p_all = 0.0, p_hit = 0.0;                       // per (class, segment) worker
  long long n_hit = 0;
  __syncthreads();
  int parity = 0;
  for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x, parity ^= 1) {
    const long long b = t / tiles_per_frame;
    const long long s = (t % tiles_per_frame) * kThreads + tid;
    const bool in = s < S;
    // phase A
    int g = kIgnore;
    float cw = 0.f, cwt = 0.f, ow = 0.f, owt = 0.f;
    if (in) {
      const L lv = label[b * S + s];
      const float* x = logits + (size_t)b * C * S + s;
      float m = -INFINITY, xg = 0.f;
      for (int c0 = 0; c0 < C; c0 += kChunk) {           // kChunk loads in flight before the first use
        float v[kChunk];
#pragma unroll
        for (int k = 0; k < kChunk; ++k) v[k] = c0 + k < C ? __ldcs(x + (size_t)(c0 + k) * S) : 0.f;
        if (c0 == 0) g = label_class(lv, C);
#pragma unroll
        for (int k = 0; k < kChunk; ++k)
          if (c0 + k < C) {
            sp[(c0 + k) * kPitch + tid] = v[k];
            m = fmaxf(m, v[k]);
            if (c0 + k == g) xg = v[k];
          }
      }
      float sum = 0.f;
      for (int c = 0; c < C; ++c) {
        const float e = expf(sp[c * kPitch + tid] - m);
        sp[c * kPitch + tid] = e;
        sum += e;
      }
      const float inv = 1.f / sum;
      for (int c = 0; c < C; ++c) sp[c * kPitch + tid] *= inv;
      if (g >= 0) {                                      // nn.CrossEntropyLoss(weight, ignore_index=255)
        cw = weight[g];
        cwt = cw * (logf(sum) + m - xg);
      }
      if (occ != nullptr && g != kIgnore) {              // cascade target: every label but 0 and 255 becomes 1
        const int go = g == 0 ? 0 : 1;
        const float x0 = __ldcs(occ + (size_t)b * 2 * S + s), x1 = __ldcs(occ + ((size_t)b * 2 + 1) * S + s);
        const float mo = fmaxf(x0, x1);
        const float lse = mo + log1pf(expf(-fabsf(x0 - x1)));
        ow = occ_weight[go];
        owt = ow * (lse - (go ? x1 : x0));
      }
    } else {
      for (int c = 0; c < C; ++c) sp[c * kPitch + tid] = 0.f;
    }
    sg[tid] = g;
    for (int f0 = 0; f0 < F; f0 += kChunk) {
      uint8_t mv[kChunk];
#pragma unroll
      for (int k = 0; k < kChunk; ++k)
        mv[k] = (in && f0 + k < F) ? __ldcs(masks + ((size_t)b * F + f0 + k) * S + s) : (uint8_t)0;
#pragma unroll
      for (int k = 0; k < kChunk; ++k) {
        if (f0 + k >= F) break;
        sm[(f0 + k) * kThreads + tid] = mv[k];
        const unsigned any = __ballot_sync(0xffffffffu, mv[k] != 0);
        if (lane == 0 && any) atomicOr(&act[parity * 2 + ((f0 + k) >> 5)], 1u << ((f0 + k) & 31));
      }
    }
    const unsigned valid = __ballot_sync(0xffffffffu, g != kIgnore), bad = __ballot_sync(0xffffffffu, g == kInvalid);
    cwt = warp_sum(cwt);
    cw = warp_sum(cw);
    if (occ != nullptr) {
      owt = warp_sum(owt);
      ow = warp_sum(ow);
    }
    if (lane == 0) {
      ce += cwt;
      ce_w += cw;
      oce += owt;
      oce_w += ow;
      n_valid += __popc(valid);
      n_invalid += __popc(bad);
    }
    __syncthreads();
    unsigned long long present = act[parity * 2] | ((unsigned long long)act[parity * 2 + 1] << 32);
    if (tid < 2) act[(parity ^ 1) * 2 + tid] = 0u;       // the next tile's flags; nobody reads them before then
    // phase B
    if (worker) {
      float pa = 0.f, ph = 0.f;
      int nh = 0;
      for (int v = v0; v < v1; ++v) {
        const int gv = sg[v];
        if (gv == kIgnore) continue;
        const float p = sp[my_c * kPitch + v];
        pa += p;
        if (gv == my_c) {
          ph += p;
          ++nh;
        }
      }
      p_all += pa;
      p_hit += ph;
      n_hit += nh;
    }
    // phase C: every voxel counts, ignored labels included (the reference masks the whole probability tensor)
    while (present) {
      const int f = __ffsll((long long)present) - 1;
      present &= present - 1;
      if (worker) {
        float q = 0.f;
        for (int v = v0; v < v1; ++v) {
          const uint8_t mv = sm[f * kThreads + v];
          if (mv) q += (float)mv * sp[my_c * kPitch + v];
        }
        part[tid] = q;
      }
      __syncthreads();
      if (tid < C) {
        double q = 0.0;
        for (int k = 0; k < nseg; ++k) q += part[tid * nseg + k];
        facc[f * C + tid] += q;
      }
      __syncthreads();
    }
    __syncthreads();
  }
  // block partials, in a fixed order
  const int K = OCCD_SSC_LOSS_SUMS(C, F);
  double* out = work + (size_t)blockIdx.x * K;
  if (lane == 0) {
    red[wid * 6 + 0] = ce;
    red[wid * 6 + 1] = ce_w;
    red[wid * 6 + 2] = (double)n_valid;
    red[wid * 6 + 3] = (double)n_invalid;
    red[wid * 6 + 4] = oce;
    red[wid * 6 + 5] = oce_w;
  }
  __syncthreads();
  if (tid < 6) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += red[w * 6 + tid];
    out[tid] = s;
  }
  __syncthreads();
  red[tid] = worker ? p_all : 0.0;
  red[kThreads + tid] = worker ? p_hit : 0.0;
  red[2 * kThreads + tid] = worker ? (double)n_hit : 0.0;
  __syncthreads();
  if (tid < C) {
    double a = 0.0, h = 0.0, n = 0.0;
    for (int k = 0; k < nseg; ++k) {
      a += red[tid * nseg + k];
      h += red[kThreads + tid * nseg + k];
      n += red[2 * kThreads + tid * nseg + k];
    }
    out[6 + tid] = a;
    out[6 + C + tid] = h;
    out[6 + 2 * C + tid] = n;
  }
  for (int i = tid; i < F * C; i += kThreads) out[6 + 3 * C + i] = facc[i];
}

template <typename L>
int launch_ssc(const float* logits, const void* label, int B, int C, long long S, const float* weight,
               const float* occ, const float* occ_weight, const uint8_t* masks, int F, double* sums, double* work,
               cudaStream_t st) {
  OCCD_CHECK_ARG((uintptr_t)label % sizeof(L) == 0, "occd_ssc_loss_sums: label is not aligned to its element size");
  const long long tpf = (S + kThreads - 1) / kThreads, n_tiles = tpf * B;
  const int grid = (int)(n_tiles < kGrid ? n_tiles : kGrid);
  const SscSmem L_(C, F);
  auto* kern = ssc_loss_kernel<L>;
  if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L_.bytes) != cudaSuccess) {
    occd_set_last_error(cudaGetErrorString(cudaGetLastError()));
    return OCCD_ERR_CUDA;
  }
  kern<<<grid, kThreads, L_.bytes, st>>>(logits, (const L*)label, C, S, tpf, n_tiles, weight, occ, occ_weight, masks,
                                         F, work);
  OCCD_CHECK_LAUNCH();
  return add_partials(work, grid, OCCD_SSC_LOSS_SUMS(C, F), sums, st);
}

// ---- CRP relation logits against the mega-context matrices -----------------------------------------------------
// A tile is 32 x 32 entries (m, n) of one relation; the matrix tile (n, m) is staged transposed through shared
// memory so that both arrays are read along their contiguous axis.  Each warp keeps per-relation fp64 sums.
__global__ void __launch_bounds__(kThreads) crp_kernel(const float* __restrict__ P, const uint8_t* __restrict__ cp,
                                                       int R, int M, int N, long long n_tiles,
                                                       double* __restrict__ work) {
  __shared__ int tile[32][33];
  __shared__ double wacc[kWarps][OCCD_CRP_MAX_RELATIONS * 4];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int i = tid; i < kWarps * R * 4; i += kThreads) wacc[i / (R * 4)][i % (R * 4)] = 0.0;
  const int tm = (M + 31) / 32, tn = (N + 31) / 32;
  for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const int nt = (int)(t % tn), mt = (int)((t / tn) % tm);
    const long long br = t / ((long long)tn * tm);            // b * R + r
    const int r = (int)(br % R);
    const size_t base = (size_t)br * M * N;
    const int m0 = mt * 32, n0 = nt * 32;
    float xs[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {                      // both arrays' loads in flight before the barrier
      const int m = m0 + wid + 8 * k, n = n0 + lane;
      xs[k] = (m < M && n < N) ? __ldcs(P + base + (size_t)m * N + n) : 0.f;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int n = n0 + wid + 8 * k, m = m0 + lane;
      tile[wid + 8 * k][lane] = (n < N && m < M) ? (int)__ldcs(cp + base + (size_t)n * M + m) : 0;
    }
    __syncthreads();
    float a = 0.f, bn = 0.f, ys = 0.f, zs = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int m = m0 + wid + 8 * k, n = n0 + lane;
      if (m < M && n < N) {
        const float x = xs[k];
        const float y = (float)tile[lane][wid + 8 * k];
        const float l = log1pf(expf(-fabsf(x)));
        a += y * (fmaxf(-x, 0.f) + l);             // y * softplus(-x)
        bn += (1.f - y) * (fmaxf(x, 0.f) + l);     // (1 - y) * softplus(x)
        ys += y;
        zs += y == 0.f ? 1.f : 0.f;
      }
    }
    a = warp_sum(a);
    bn = warp_sum(bn);
    ys = warp_sum(ys);
    zs = warp_sum(zs);
    if (lane == 0) {
      wacc[wid][r * 4 + 0] += a;
      wacc[wid][r * 4 + 1] += bn;
      wacc[wid][r * 4 + 2] += ys;
      wacc[wid][r * 4 + 3] += zs;
    }
    __syncthreads();
  }
  __syncthreads();
  for (int k = tid; k < R * 4; k += kThreads) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += wacc[w][k];
    work[(size_t)blockIdx.x * R * 4 + k] = s;
  }
}

// ---- depth classification (DepthClsLoss.get_depth_loss, occdepth/loss/depth_loss.py:14-87) ----------------------
// One thread per low-resolution pixel: the nearest-resized gt's f x f patch, its smallest nonzero depth, the bin, and
// the binary cross-entropy of the pixel's D probabilities against the one-hot bin (bin 0 dropped).
__global__ void __launch_bounds__(kThreads) depth_kernel(const float* __restrict__ gt, int H, int W,
                                                         const float* __restrict__ prob, int D, int h, int w, int f,
                                                         float sh, float sw, float lo, float step, long long n_pix,
                                                         double* __restrict__ work) {
  __shared__ double red[kWarps][2];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  double acc = 0.0, fg = 0.0;
  const long long hw = (long long)h * w;
  for (long long i0 = (long long)blockIdx.x * kThreads; i0 < n_pix; i0 += (long long)gridDim.x * kThreads) {
    const long long i = i0 + tid;
    float s = 0.f;
    bool is_fg = false;
    if (i < n_pix) {
      const long long n = i / hw;
      const int y = (int)((i % hw) / w), x = (int)(i % w);
      float dmin = 1e5f;
      for (int dy = 0; dy < f; ++dy) {
        const int iy = min((int)floorf((float)(y * f + dy) * sh), H - 1);      // F.interpolate(mode="nearest")
        const float* row = gt + ((size_t)n * H + iy) * W;
#pragma unroll 8
        for (int dx = 0; dx < f; ++dx) {
          const int ix = min((int)floorf((float)(x * f + dx) * sw), W - 1);
          const float d = row[ix];
          const float v = d == 0.f ? 1e5f : d;
          if (v < dmin || isnan(v)) dmin = isnan(dmin) ? dmin : v;            // torch.min propagates NaN
        }
      }
      const float bin = (dmin - lo) / step;
      const int k = (bin < (float)(D + 1) && bin >= 0.f) ? (int)bin : 0;     // .long() truncates
      if (k >= 1) {
        is_fg = true;
        const float* p = prob + (size_t)n * D * hw + (i % hw);
#pragma unroll 8
        for (int d = 0; d < D; ++d) {
          const float pv = __ldcs(p + (size_t)d * hw);
          s -= d == k - 1 ? fmaxf(logf(pv), -100.f) : fmaxf(log1pf(-pv), -100.f);
        }
      }
    }
    s = warp_sum(s);
    const unsigned cnt = __popc(__ballot_sync(0xffffffffu, is_fg));
    if (lane == 0) {
      acc += s;
      fg += cnt;
    }
  }
  if (lane == 0) {
    red[wid][0] = acc;
    red[wid][1] = fg;
  }
  __syncthreads();
  if (tid < 2) {
    double v = 0.0;
    for (int w_ = 0; w_ < kWarps; ++w_) v += red[w_][tid];
    work[(size_t)blockIdx.x * 2 + tid] = v;
  }
}

}  // namespace

extern "C" int occd_ssc_loss_sums(const float* logits, const void* label, int label_dtype, int B, int n_classes,
                                  long long S, const float* weight, const float* occ_logits, const float* occ_weight,
                                  const uint8_t* frustum_masks, int n_frustums, double* sums, double* work,
                                  long long work_len, void* stream) {
  OCCD_CHECK_ARG(logits && label && weight && sums && work && B > 0 && S > 0, "occd_ssc_loss_sums: args");
  OCCD_CHECK_ARG(n_classes > 0 && n_classes <= OCCD_SSC_LOSS_MAX_CLASSES,
                 "occd_ssc_loss_sums: n_classes must be in [1, 64]");
  OCCD_CHECK_ARG(n_frustums >= 0 && n_frustums <= OCCD_SSC_LOSS_MAX_FRUSTUMS,
                 "occd_ssc_loss_sums: n_frustums must be in [0, 64]");
  OCCD_CHECK_ARG((n_frustums == 0) == (frustum_masks == nullptr),
                 "occd_ssc_loss_sums: frustum_masks is required exactly when n_frustums > 0");
  OCCD_CHECK_ARG((occ_logits == nullptr) == (occ_weight == nullptr),
                 "occd_ssc_loss_sums: occ_logits and occ_weight go together");
  OCCD_CHECK_ARG((uintptr_t)sums % 8 == 0 && (uintptr_t)work % 8 == 0 && (uintptr_t)logits % 4 == 0 &&
                     (uintptr_t)weight % 4 == 0 && (uintptr_t)occ_logits % 4 == 0 && (uintptr_t)occ_weight % 4 == 0,
                 "occd_ssc_loss_sums: misaligned pointer");
  OCCD_CHECK_ARG(work_len >= (long long)OCCD_LOSS_WORK_BLOCKS * OCCD_SSC_LOSS_SUMS(n_classes, n_frustums),
                 "occd_ssc_loss_sums: work must hold OCCD_LOSS_WORK_BLOCKS * OCCD_SSC_LOSS_SUMS(C, F) doubles");
  OCCD_CHECK_ARG((S + kThreads - 1) / kThreads * B < (1LL << 40), "occd_ssc_loss_sums: too many voxels");
  cudaStream_t st = (cudaStream_t)stream;
  switch (label_dtype) {
    case OCCD_DTYPE_F32:
      return launch_ssc<float>(logits, label, B, n_classes, S, weight, occ_logits, occ_weight, frustum_masks,
                               n_frustums, sums, work, st);
    case OCCD_DTYPE_U8:
      return launch_ssc<uint8_t>(logits, label, B, n_classes, S, weight, occ_logits, occ_weight, frustum_masks,
                                 n_frustums, sums, work, st);
    case OCCD_DTYPE_I64:
      return launch_ssc<long long>(logits, label, B, n_classes, S, weight, occ_logits, occ_weight, frustum_masks,
                                   n_frustums, sums, work, st);
    default: occd_set_last_error("occd_ssc_loss_sums: label dtype must be F32, U8 or I64"); return OCCD_ERR_ARG;
  }
}

extern "C" int occd_crp_relation_sums(const float* P_logits, const uint8_t* cp, int B, int R, int M, int N,
                                      double* sums, double* work, long long work_len, void* stream) {
  OCCD_CHECK_ARG(P_logits && cp && sums && work && B > 0 && M > 0 && N > 0, "occd_crp_relation_sums: args");
  OCCD_CHECK_ARG(R > 0 && R <= OCCD_CRP_MAX_RELATIONS, "occd_crp_relation_sums: n_relations must be in [1, 16]");
  OCCD_CHECK_ARG((uintptr_t)P_logits % 4 == 0 && (uintptr_t)sums % 8 == 0 && (uintptr_t)work % 8 == 0,
                 "occd_crp_relation_sums: misaligned pointer");
  OCCD_CHECK_ARG(work_len >= (long long)OCCD_LOSS_WORK_BLOCKS * 4 * R,
                 "occd_crp_relation_sums: work must hold OCCD_LOSS_WORK_BLOCKS * 4 * R doubles");
  cudaStream_t st = (cudaStream_t)stream;
  const long long n_tiles = (long long)B * R * ((M + 31) / 32) * ((N + 31) / 32);
  const int grid = (int)(n_tiles < kGrid ? n_tiles : kGrid);
  crp_kernel<<<grid, kThreads, 0, st>>>(P_logits, cp, R, M, N, n_tiles, work);
  OCCD_CHECK_LAUNCH();
  return add_partials(work, grid, 4 * R, sums, st);
}

extern "C" int occd_depth_cls_sums(const float* gt, int n_maps, int H, int W, const float* prob, int D, int h, int w,
                                   int factor, double d0, double step, double* sums, double* work, long long work_len,
                                   void* stream) {
  OCCD_CHECK_ARG(gt && prob && sums && work && n_maps > 0 && H > 0 && W > 0 && h > 0 && w > 0,
                 "occd_depth_cls_sums: args");
  OCCD_CHECK_ARG(D > 0 && D <= OCCD_DEPTH_MAX_BINS, "occd_depth_cls_sums: depth bins must be in [1, 1024]");
  OCCD_CHECK_ARG(factor > 0 && factor <= 64 && step > 0.0, "occd_depth_cls_sums: factor / step");
  OCCD_CHECK_ARG((uintptr_t)gt % 4 == 0 && (uintptr_t)prob % 4 == 0 && (uintptr_t)sums % 8 == 0 &&
                     (uintptr_t)work % 8 == 0,
                 "occd_depth_cls_sums: misaligned pointer");
  OCCD_CHECK_ARG(work_len >= (long long)OCCD_LOSS_WORK_BLOCKS * 2,
                 "occd_depth_cls_sums: work must hold OCCD_LOSS_WORK_BLOCKS * 2 doubles");
  cudaStream_t st = (cudaStream_t)stream;
  const long long n_pix = (long long)n_maps * h * w;
  const long long blocks = (n_pix + kThreads - 1) / kThreads;
  const int grid = (int)(blocks < kGrid ? blocks : kGrid);
  // the resize's float scale and the bin's float operands, as PyTorch forms them from the sizes and Python floats
  const float sh = (float)H / (float)((long long)h * factor), sw = (float)W / (float)((long long)w * factor);
  depth_kernel<<<grid, kThreads, 0, st>>>(gt, H, W, prob, D, h, w, factor, sh, sw, (float)(d0 - step), (float)step,
                                          n_pix, work);
  OCCD_CHECK_LAUNCH();
  return add_partials(work, grid, 2, sums, st);
}
