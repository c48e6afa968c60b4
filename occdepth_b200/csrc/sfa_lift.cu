// Stereo-SFA 2D->3D lift: fused multi-scale, multi-view gather + cosine soft-assignment.
//
// Replaces reference occdepth/models/SFA.py:12-106 (SFA.forward) as driven by
// occdepth/models/OccDepth.py:262-298 (_forward_2d_to_3d: one SFA call per 2D scale, summed).
//
// One launch does what the reference does in 4 x ~85 ATen kernels:
//   for every voxel n, every scale s, every view v:
//       f_v = sum_p feat_s[v][ (y_p // s) * w_s + (x_p // s) ] * fov_p / sum_p fov_p      (0/0 -> 0)
//       m_v = any_p fov_p
//   V == 2:  cos = <f_0,f_1> / (max(|f_0|,eps) max(|f_1|,eps)) * m_0 m_1
//            out_s = [(cos + [m_0>m_1]) f_0 + (cos + [m_1>m_0]) f_1] / (V (V-1))
//   V == 1:  out_s = f_0
//   out = sum_s out_s   (optionally * prior[n] * scale_const for the FlospDepth product, OccDepth.py:339)
//
// Memory-bound kernel: feature maps are channels-last so that one voxel's gather is one contiguous
// C*sizeof(T) line; G lanes cooperate on a voxel with 16-byte vector loads; the (x,y)/fov records of a
// block's voxels are staged through shared memory with coalesced loads; the cosine reductions are
// G-lane shuffle reductions; every output element is written exactly once.
#include "common.cuh"
#include "../../include/occdepth_b200.h"

namespace {

constexpr int kThreads = 256;
constexpr int kIters = 4;  // voxel batches per block

template <typename T> struct FeatTraits;
// predicated 16-byte read-only load: zeros when !ok, no branch (the gather loop is issue bound; a divergent branch
// per load costs a BSSY/BSYNC pair and splits the warp's loads)
__device__ __forceinline__ uint4 ldg16_pred(const void* p, bool ok) {
  uint4 v;
  asm("{\n"
      " .reg .pred q;\n"
      " setp.ne.s32 q, %5, 0;\n"
      " mov.b32 %0, 0;\n mov.b32 %1, 0;\n mov.b32 %2, 0;\n mov.b32 %3, 0;\n"
      " @q ld.global.nc.v4.b32 {%0, %1, %2, %3}, [%4];\n"
      "}"
      : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
      : "l"(p), "r"((int)ok));
  return v;
}
template <> struct FeatTraits<float> {
  static constexpr int VEC = 4;   // elements per 16-byte vector
  static __device__ __forceinline__ void load(const float* p, float* f) {
    float4 v = __ldg(reinterpret_cast<const float4*>(p));
    f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
  }
  static __device__ __forceinline__ void load_pred(const float* p, bool ok, float* f) {
    const uint4 v = ldg16_pred(p, ok);
    f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y); f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w);
  }
};
template <> struct FeatTraits<__nv_bfloat16> {
  static constexpr int VEC = 8;
  static __device__ __forceinline__ void load(const __nv_bfloat16* p, float* f) {
    uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
    unpack8(v, f);
  }
  static __device__ __forceinline__ void load_pred(const __nv_bfloat16* p, bool ok, float* f) {
    unpack8(ldg16_pred(p, ok), f);
  }
};

struct SfaKParams {
  const void* feat[OCCD_SFA_MAX_SCALES];
  int h[OCCD_SFA_MAX_SCALES], w[OCCD_SFA_MAX_SCALES];
  int div[OCCD_SFA_MAX_SCALES], shift[OCCD_SFA_MAX_SCALES];
  long long vstride[OCCD_SFA_MAX_SCALES];  // elements between views
  int vrow[OCCD_SFA_MAX_SCALES];           // the same in rows of C elements (P == 1 fast path: fits 32 bits)
  int n_scales, C, P;
  long long N;
  const long long* pix;
  const unsigned char* fov;
  void* out;
  int out_mode, out_cstride;
  long long out_n;  // voxels in the output (planar stride)
  int perm_nyu, S1, S2;
  const float* prior;
  float scale_const;
};

__device__ __forceinline__ long long floordiv64(long long a, int d, int shift) {
  if (shift >= 0) return a >> shift;  // arithmetic shift == floor division for d = 2^shift
  long long q = a / d;
  if ((a % d != 0) && ((a < 0) != (d < 0))) --q;
  return q;
}

template <typename T, int V, int NV, int G>
__global__ void __launch_bounds__(kThreads)
sfa_lift_kernel(const SfaKParams p) {
  constexpr int VEC = FeatTraits<T>::VEC;
  constexpr int VPB = kThreads / G;   // voxels per batch
  constexpr int CPL = NV * VEC;       // channels per lane
  extern __shared__ __align__(16) unsigned char smem_raw[];

  const int P = p.P;
  const long long block_n0 = (long long)blockIdx.x * (VPB * kIters);
  const int n_block = (int)min((long long)(VPB * kIters), p.N - block_n0);
  // smem: pix records [V][n_block][P] int64x2, then fov [V][n_block][P] bytes
  longlong2* s_pix = reinterpret_cast<longlong2*>(smem_raw);
  unsigned char* s_fov = smem_raw + (size_t)V * VPB * kIters * P * sizeof(longlong2);

  // ---- stage indices (coalesced) ----
  const int recs = n_block * P;
  for (int v = 0; v < V; ++v) {
    const longlong2* gp = reinterpret_cast<const longlong2*>(p.pix) + ((long long)v * p.N + block_n0) * P;
    const unsigned char* gf = p.fov + ((long long)v * p.N + block_n0) * P;
    for (int i = threadIdx.x; i < recs; i += kThreads) {
      s_pix[(size_t)v * VPB * kIters * P + i] = gp[i];
      s_fov[(size_t)v * VPB * kIters * P + i] = gf[i];
    }
  }
  __syncthreads();

  const int lane_g = threadIdx.x % G;
  const int grp = threadIdx.x / G;

#pragma unroll 1
  for (int it = 0; it < kIters; ++it) {
    const int ln = it * VPB + grp;  // voxel index local to the block
    const bool active = ln < n_block;
    float acc[CPL];
#pragma unroll
    for (int i = 0; i < CPL; ++i) acc[i] = 0.f;

#pragma unroll 1
    for (int s = 0; s < p.n_scales; ++s) {
      const T* feat = reinterpret_cast<const T*>(p.feat[s]);
      const int hs = p.h[s], ws = p.w[s];
      const long long hw = (long long)hs * ws;
      float f[V][CPL];
      float m[V];
#pragma unroll
      for (int v = 0; v < V; ++v) {
#pragma unroll
        for (int i = 0; i < CPL; ++i) f[v][i] = 0.f;
        int cnt = 0;
        if (active) {
          for (int pp = 0; pp < P; ++pp) {
            const size_t r = (size_t)v * VPB * kIters * P + (size_t)ln * P + pp;
            if (s_fov[r]) {
              ++cnt;
              const longlong2 xy = s_pix[r];
              const long long xs = floordiv64(xy.x, p.div[s], p.shift[s]);
              const long long ys = floordiv64(xy.y, p.div[s], p.shift[s]);
              const long long idx = ys * ws + xs;
              if (idx >= 0 && idx < hw) {
                const T* src = feat + (long long)v * p.vstride[s] + idx * p.C;
#pragma unroll
                for (int j = 0; j < NV; ++j) {
                  const int c0 = (j * G + lane_g) * VEC;
                  if (c0 < p.C) {
                    float t[VEC];
                    FeatTraits<T>::load(src + c0, t);
#pragma unroll
                    for (int e = 0; e < VEC; ++e) f[v][j * VEC + e] += t[e];
                  }
                }
              }
            }
          }
        }
        m[v] = cnt > 0 ? 1.f : 0.f;
        if (cnt > 1) {
          const float fc = (float)cnt;
#pragma unroll
          for (int i = 0; i < CPL; ++i) f[v][i] = __fdiv_rn(f[v][i], fc);
        }
      }

      if (V == 1) {
#pragma unroll
        for (int i = 0; i < CPL; ++i) acc[i] += f[0][i];
      } else {
        float pair_acc[CPL];
#pragma unroll
        for (int i = 0; i < CPL; ++i) pair_acc[i] = 0.f;
#pragma unroll
        for (int a = 0; a < V; ++a) {
#pragma unroll
          for (int b = a + 1; b < V; ++b) {
            float dot = 0.f, na = 0.f, nb = 0.f;
#pragma unroll
            for (int i = 0; i < CPL; ++i) {
              dot = fmaf(f[a][i], f[b][i], dot);
              na = fmaf(f[a][i], f[a][i], na);
              nb = fmaf(f[b][i], f[b][i], nb);
            }
#pragma unroll
            for (int o = G / 2; o > 0; o >>= 1) {
              dot += __shfl_xor_sync(0xffffffffu, dot, o);
              na += __shfl_xor_sync(0xffffffffu, na, o);
              nb += __shfl_xor_sync(0xffffffffu, nb, o);
            }
            const float eps = 1e-8f;
            const float cosv = dot / (fmaxf(sqrtf(na), eps) * fmaxf(sqrtf(nb), eps));
            const float c = cosv * (m[a] * m[b]);
            const float wa = c + ((m[a] > m[b]) ? 1.f : 0.f);
            const float wb = c + ((m[b] > m[a]) ? 1.f : 0.f);
#pragma unroll
            for (int i = 0; i < CPL; ++i) pair_acc[i] += wa * f[a][i] + wb * f[b][i];
          }
        }
        const float inv = 1.f / (float)(V * (V - 1));
#pragma unroll
        for (int i = 0; i < CPL; ++i) acc[i] += pair_acc[i] * inv;
      }
    }

    if (!active) continue;
    const long long n = block_n0 + ln;
    long long no = n;
    if (p.perm_nyu) {  // reference SFA.py:90-97: (C, S0, S2, S1) -> permute(0,1,3,2)
      const long long i0 = n / ((long long)p.S1 * p.S2);
      const int k = (int)((n / p.S1) % p.S2);
      const int j = (int)(n % p.S1);
      no = (i0 * p.S1 + j) * p.S2 + k;
    }
    if (p.prior) {
      const float pr = p.prior[no];
#pragma unroll
      for (int i = 0; i < CPL; ++i) acc[i] = acc[i] * pr * p.scale_const;
    }
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int c0 = (j * G + lane_g) * VEC;
      if (c0 >= p.C) continue;
      if (p.out_mode == OCCD_SFA_OUT_BF16_CL) {
        __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + no * p.out_cstride + c0;
        if (VEC == 8) {
          *reinterpret_cast<uint4*>(o) = pack8(&acc[j * VEC]);
        } else {
          __nv_bfloat162 lo = __floats2bfloat162_rn(acc[j * VEC], acc[j * VEC + 1]);
          __nv_bfloat162 hi = __floats2bfloat162_rn(acc[j * VEC + 2], acc[j * VEC + 3]);
          uint2 u;
          u.x = *reinterpret_cast<unsigned*>(&lo);
          u.y = *reinterpret_cast<unsigned*>(&hi);
          *reinterpret_cast<uint2*>(o) = u;
        }
      } else if (p.out_mode == OCCD_SFA_OUT_F32_CL || p.out_mode == OCCD_SFA_OUT_TF32_CL) {
        float* o = reinterpret_cast<float*>(p.out) + no * p.out_cstride + c0;
        if (p.out_mode == OCCD_SFA_OUT_TF32_CL) {   // operand of the 3-D net's kind::tf32 convolutions
#pragma unroll
          for (int e = 0; e < VEC; ++e) acc[j * VEC + e] = round_tf32(acc[j * VEC + e]);
        }
#pragma unroll
        for (int e = 0; e < VEC; e += 4)
          *reinterpret_cast<float4*>(o + e) =
              make_float4(acc[j * VEC + e], acc[j * VEC + e + 1], acc[j * VEC + e + 2], acc[j * VEC + e + 3]);
      } else {  // planar fp32 [C][out_n] == reference (C, X, Y, Z)
        float* o = reinterpret_cast<float*>(p.out);
#pragma unroll
        for (int e = 0; e < VEC; ++e) o[(long long)(c0 + e) * p.out_n + no] = acc[j * VEC + e];
      }
    }
  }
}

// one scale's contribution: acc += sum over view pairs of the cosine-weighted features (SFA.py:65-92 semantics)
template <int V, int CPL, int G>
__device__ __forceinline__ void sfa_reduce_views(const float (&f)[V][CPL], const float (&m)[V], float (&acc)[CPL]) {
  if (V == 1) {
#pragma unroll
    for (int i = 0; i < CPL; ++i) acc[i] += f[0][i];
  } else if (V == 2) {
    // one pair: accumulate straight into acc (no pair accumulator: 4 vectors per lane stay in registers)
    float dot = 0.f, na = 0.f, nb = 0.f;
#pragma unroll
    for (int i = 0; i < CPL; ++i) {
      dot = fmaf(f[0][i], f[V - 1][i], dot);
      na = fmaf(f[0][i], f[0][i], na);
      nb = fmaf(f[V - 1][i], f[V - 1][i], nb);
    }
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) {
      dot += __shfl_xor_sync(0xffffffffu, dot, o);
      na += __shfl_xor_sync(0xffffffffu, na, o);
      nb += __shfl_xor_sync(0xffffffffu, nb, o);
    }
    // dot / (max(|a|, eps) max(|b|, eps)) with eps = 1e-8: max(sqrt(x), eps) == sqrt(max(x, eps^2))
    const float cosv = dot * rsqrtf(fmaxf(na, 1e-16f)) * rsqrtf(fmaxf(nb, 1e-16f));
    const float c = cosv * (m[0] * m[V - 1]);
    const float wa = (c + ((m[0] > m[V - 1]) ? 1.f : 0.f)) * 0.5f;      // / (V (V-1)) with V == 2
    const float wb = (c + ((m[V - 1] > m[0]) ? 1.f : 0.f)) * 0.5f;
#pragma unroll
    for (int i = 0; i < CPL; ++i) acc[i] += wa * f[0][i] + wb * f[V - 1][i];
  } else {
    float pair_acc[CPL];
#pragma unroll
    for (int i = 0; i < CPL; ++i) pair_acc[i] = 0.f;
#pragma unroll
    for (int a = 0; a < V; ++a) {
#pragma unroll
      for (int b = a + 1; b < V; ++b) {
        float dot = 0.f, na = 0.f, nb = 0.f;
#pragma unroll
        for (int i = 0; i < CPL; ++i) {
          dot = fmaf(f[a][i], f[b][i], dot);
          na = fmaf(f[a][i], f[a][i], na);
          nb = fmaf(f[b][i], f[b][i], nb);
        }
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) {
          dot += __shfl_xor_sync(0xffffffffu, dot, o);
          na += __shfl_xor_sync(0xffffffffu, na, o);
          nb += __shfl_xor_sync(0xffffffffu, nb, o);
        }
        const float eps = 1e-8f;
        const float cosv = dot / (fmaxf(sqrtf(na), eps) * fmaxf(sqrtf(nb), eps));
        const float c = cosv * (m[a] * m[b]);
        const float wa = c + ((m[a] > m[b]) ? 1.f : 0.f);
        const float wb = c + ((m[b] > m[a]) ? 1.f : 0.f);
#pragma unroll
        for (int i = 0; i < CPL; ++i) pair_acc[i] += wa * f[a][i] + wb * f[b][i];
      }
    }
    const float inv = 1.f / (float)(V * (V - 1));
#pragma unroll
    for (int i = 0; i < CPL; ++i) acc[i] += pair_acc[i] * inv;
  }
}

// Fast path for P == 1 (pattern_id 0, every shipped config): one (x,y,fov) record per (view, voxel).
// Index math is 32-bit (h*w < 2^31) and done once per (view, voxel) by one thread (staged in shared memory); the gather
// loop issues a scale's V x NV predicated 16-byte loads per lane back to back, then reduces them.
template <typename T, int V, int NV, int G, int KI>
__global__ void __launch_bounds__(kThreads)   // (kThreads, 4) forces 64 registers + spills: measured slower (r02)
sfa_lift_p1_kernel(const SfaKParams p) {
  constexpr int VEC = FeatTraits<T>::VEC;
  constexpr int VPB = kThreads / G;
  constexpr int CPL = NV * VEC;
  constexpr int NS = OCCD_SFA_MAX_SCALES;
  // row index of the gathered pixel at every scale (or -1), worked out ONCE per (view, voxel) by one thread; the
  // gather loop below only reads them back (the kernel is issue bound: with every lane of a voxel's group redoing
  // this arithmetic it executed ~250 warp instructions per voxel, ncu r02)
  __shared__ int4 s_off[V][VPB * KI];
  __shared__ unsigned char s_in[V][VPB * KI];
  static_assert(OCCD_SFA_MAX_SCALES == 4, "offsets are staged as one int4 per (view, voxel)");
  pdl_wait();
  const long long block_n0 = (long long)blockIdx.x * (VPB * KI);
  const int n_block = (int)min((long long)(VPB * KI), p.N - block_n0);
  const int ns = p.n_scales;
  for (int i = threadIdx.x; i < V * n_block; i += kThreads) {
    const int v = i / n_block, ln = i - v * n_block;
    longlong2 xy = __ldg(reinterpret_cast<const longlong2*>(p.pix) + (long long)v * p.N + block_n0 + ln);
    const bool in = p.fov[(long long)v * p.N + block_n0 + ln] != 0;
    // 32-bit fast math is valid for |x|,|y| < 2^30; anything else cannot address a feature map anyway
    if (xy.x < -(1LL << 30) || xy.x > (1LL << 30) || xy.y < -(1LL << 30) || xy.y > (1LL << 30)) {
      xy.x = -1; xy.y = 0;  // flat index negative -> treated as the zero column, mask stays as given
    }
    const int x = (int)xy.x, y = (int)xy.y;
    int o4[NS];
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      int o = -1;
      if (in && s < ns) {
        int xs, ys;
        if (p.shift[s] >= 0) { xs = x >> p.shift[s]; ys = y >> p.shift[s]; }
        else { xs = (int)floordiv64(x, p.div[s], -1); ys = (int)floordiv64(y, p.div[s], -1); }
        const long long idx = (long long)ys * p.w[s] + xs;
        const int hw = p.h[s] * p.w[s];
        if (idx >= 0 && idx < hw) o = v * p.vrow[s] + (int)idx;
      }
      o4[s] = o;
    }
    s_off[v][ln] = make_int4(o4[0], o4[1], o4[2], o4[3]);
    s_in[v][ln] = in ? 1 : 0;
  }
  __syncthreads();
  const int lane_g = threadIdx.x % G;
  const int grp = threadIdx.x / G;

#pragma unroll 1
  for (int it = 0; it < KI; ++it) {
    const int ln = it * VPB + grp;
    const bool active = ln < n_block;
    float m[V];
    int off[V][NS];  // element offset of the gathered pixel's channel vector, or -1
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const int4 o = active ? s_off[v][ln] : make_int4(-1, -1, -1, -1);
      off[v][0] = o.x; off[v][1] = o.y; off[v][2] = o.z; off[v][3] = o.w;
      m[v] = (active && s_in[v][ln]) ? 1.f : 0.f;
    }
    // per scale: the V x NV gathers of a lane are issued back to back, then reduced (the floor is the scattered
    // 256-byte row fetches themselves)
    float acc[CPL];
#pragma unroll
    for (int i = 0; i < CPL; ++i) acc[i] = 0.f;
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      if (s >= ns) break;
      const T* feat = reinterpret_cast<const T*>(p.feat[s]);
      float f[V][CPL];
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const bool ok = off[v][s] >= 0;
        const T* row = feat + (long long)(ok ? off[v][s] : 0) * p.C + lane_g * VEC;
#pragma unroll
        for (int j = 0; j < NV; ++j)
          FeatTraits<T>::load_pred(row + j * G * VEC, ok && (j * G + lane_g) * VEC < p.C, &f[v][j * VEC]);
      }
      sfa_reduce_views<V, CPL, G>(f, m, acc);
    }
    if (!active) continue;
    const long long n = block_n0 + ln;
    long long no = n;
    if (p.perm_nyu) {
      const long long i0 = n / ((long long)p.S1 * p.S2);
      const int k = (int)((n / p.S1) % p.S2);
      const int j = (int)(n % p.S1);
      no = (i0 * p.S1 + j) * p.S2 + k;
    }
    if (p.prior) {
      const float pr = p.prior[no];
#pragma unroll
      for (int i = 0; i < CPL; ++i) acc[i] = acc[i] * pr * p.scale_const;
    }
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int c0 = (j * G + lane_g) * VEC;
      if (c0 >= p.C) continue;
      if (p.out_mode == OCCD_SFA_OUT_BF16_CL) {
        __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + no * p.out_cstride + c0;
        if (VEC == 8) {
          *reinterpret_cast<uint4*>(o) = pack8(&acc[j * VEC]);
        } else {
          __nv_bfloat162 lo = __floats2bfloat162_rn(acc[j * VEC], acc[j * VEC + 1]);
          __nv_bfloat162 hi = __floats2bfloat162_rn(acc[j * VEC + 2], acc[j * VEC + 3]);
          uint2 u;
          u.x = *reinterpret_cast<unsigned*>(&lo);
          u.y = *reinterpret_cast<unsigned*>(&hi);
          *reinterpret_cast<uint2*>(o) = u;
        }
      } else if (p.out_mode == OCCD_SFA_OUT_F32_CL || p.out_mode == OCCD_SFA_OUT_TF32_CL) {
        float* o = reinterpret_cast<float*>(p.out) + no * p.out_cstride + c0;
        if (p.out_mode == OCCD_SFA_OUT_TF32_CL) {   // operand of the 3-D net's kind::tf32 convolutions
#pragma unroll
          for (int e = 0; e < VEC; ++e) acc[j * VEC + e] = round_tf32(acc[j * VEC + e]);
        }
#pragma unroll
        for (int e = 0; e < VEC; e += 4)
          *reinterpret_cast<float4*>(o + e) =
              make_float4(acc[j * VEC + e], acc[j * VEC + e + 1], acc[j * VEC + e + 2], acc[j * VEC + e + 3]);
      } else {
        float* o = reinterpret_cast<float*>(p.out);
#pragma unroll
        for (int e = 0; e < VEC; ++e) o[(long long)(c0 + e) * p.out_n + no] = acc[j * VEC + e];
      }
    }
  }
}

static bool sfa_fits_int32(const SfaKParams& kp, int n_views) {
  for (int s = 0; s < kp.n_scales; ++s)
    if ((long long)n_views * kp.vstride[s] >= (1LL << 31) || kp.n_scales > OCCD_SFA_MAX_SCALES) return false;
  return true;
}

// G lanes cooperate on one voxel, each holding NV 16-byte vectors of the C channels.  Fewer lanes per voxel = less
// redundant index / cosine-scalar work per voxel, more vectors per lane = more independent 16-byte gathers in flight
// per lane.
template <typename T, int V, int NV, int G>
int launch_g(const SfaKParams& kp, cudaStream_t st) {
  constexpr int VPB = kThreads / G;
  const long long per_block = (long long)VPB * kIters;
  const long long blocks = (kp.N + per_block - 1) / per_block;
  if (kp.P == 1 && sfa_fits_int32(kp, V)) {
    // two voxel batches per block
    constexpr int KI = 2;
    const unsigned nb = (unsigned)((kp.N + VPB * KI - 1) / (VPB * KI));
    OCCD_LAUNCH_CHECKED((sfa_lift_p1_kernel<T, V, NV, G, KI>), dim3(nb), dim3(kThreads), 0, st, kp);
    return OCCD_OK;
  } else {
    const size_t smem = (size_t)V * VPB * kIters * kp.P * (sizeof(longlong2) + 1);
    if (smem > 200 * 1024) {
      occd_set_last_error("occd_sfa_lift_fwd: pattern count too large for the index staging buffer");
      return OCCD_ERR_UNSUPPORTED;
    }
    if (smem > 48 * 1024)
      cudaFuncSetAttribute(sfa_lift_kernel<T, V, NV, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    sfa_lift_kernel<T, V, NV, G><<<(unsigned)blocks, kThreads, smem, st>>>(kp);
  }
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

template <typename T, int V>
int launch_nv(const SfaKParams& kp, cudaStream_t st) {
  constexpr int VEC = FeatTraits<T>::VEC;
  const int vecs = (kp.C + VEC - 1) / VEC;           // 16-byte vectors per voxel
  // vectors per lane: 4 for fp32 (16 channels), 2 for bf16 (16 channels: four 8-element vectors cost 64 registers of
  // gathered values per scale).  OCCD_LIFT_NV=2 / 4 overrides (experiment hook, tools/lift_bench.py)
  static const int nv_env = [] { const char* e = getenv("OCCD_LIFT_NV"); return e ? atoi(e) : 0; }();
  const bool nv2 = nv_env == 2 || (nv_env != 4 && VEC == 8);
  if (vecs <= 4) return launch_g<T, V, 1, 4>(kp, st);
  if (nv2) {
    if (vecs <= 8) return launch_g<T, V, 2, 4>(kp, st);
    if (vecs <= 16) return launch_g<T, V, 2, 8>(kp, st);
    if (vecs <= 32) return launch_g<T, V, 2, 16>(kp, st);
    if (vecs <= 64) return launch_g<T, V, 2, 32>(kp, st);
  } else {
    if (vecs <= 8) return launch_g<T, V, 4, 2>(kp, st);
    if (vecs <= 16) return launch_g<T, V, 4, 4>(kp, st);
    if (vecs <= 32) return launch_g<T, V, 4, 8>(kp, st);
    if (vecs <= 64) return launch_g<T, V, 4, 16>(kp, st);
  }
  occd_set_last_error("occd_sfa_lift_fwd: C too large (max 256 fp32 / 512 bf16 channels)");
  return OCCD_ERR_UNSUPPORTED;
}

template <typename T>
int launch_v(const SfaKParams& kp, int V, cudaStream_t st) {
  switch (V) {
    case 1: return launch_nv<T, 1>(kp, st);
    case 2: return launch_nv<T, 2>(kp, st);
    case 3: return launch_nv<T, 3>(kp, st);
    case 4: return launch_nv<T, 4>(kp, st);
  }
  occd_set_last_error("occd_sfa_lift_fwd: n_views must be 1..4");
  return OCCD_ERR_UNSUPPORTED;
}

}  // namespace

extern "C" int occd_sfa_lift_fwd(const occd_sfa_params* a, void* stream) {
  OCCD_CHECK_ARG(a != nullptr, "occd_sfa_lift_fwd: null params");
  OCCD_CHECK_ARG(a->n_scales >= 1 && a->n_scales <= OCCD_SFA_MAX_SCALES, "occd_sfa_lift_fwd: n_scales must be 1..4");
  OCCD_CHECK_ARG(a->pix && a->fov && a->out, "occd_sfa_lift_fwd: null pointer");
  OCCD_CHECK_ARG(a->N >= 0 && a->P >= 1, "occd_sfa_lift_fwd: bad N/P");
  OCCD_CHECK_ARG(a->feat_dtype == OCCD_DTYPE_F32 || a->feat_dtype == OCCD_DTYPE_BF16, "occd_sfa_lift_fwd: feat dtype");
  const int vec = a->feat_dtype == OCCD_DTYPE_F32 ? 4 : 8;
  OCCD_CHECK_ARG(a->C > 0 && a->C % vec == 0, "occd_sfa_lift_fwd: C must be a multiple of the 16-byte vector width");
  OCCD_CHECK_ARG(a->out_mode >= 0 && a->out_mode <= 3, "occd_sfa_lift_fwd: out_mode");
  if (a->out_mode != OCCD_SFA_OUT_F32_PLANAR)
    OCCD_CHECK_ARG(a->out_cstride >= a->C && a->out_cstride % vec == 0, "occd_sfa_lift_fwd: out_cstride");
  if (a->N == 0) return OCCD_OK;
  SfaKParams kp;
  for (int s = 0; s < OCCD_SFA_MAX_SCALES; ++s) {
    kp.feat[s] = nullptr; kp.h[s] = kp.w[s] = 0; kp.div[s] = 1; kp.shift[s] = 0; kp.vstride[s] = 0; kp.vrow[s] = 0;
  }
  for (int s = 0; s < a->n_scales; ++s) {
    OCCD_CHECK_ARG(a->feat[s] != nullptr && a->h[s] > 0 && a->w[s] > 0 && a->div[s] != 0, "occd_sfa_lift_fwd: scale spec");
    kp.feat[s] = a->feat[s]; kp.h[s] = a->h[s]; kp.w[s] = a->w[s]; kp.div[s] = a->div[s];
    kp.vstride[s] = a->vstride[s] ? a->vstride[s] : (long long)a->h[s] * a->w[s] * a->C;
    OCCD_CHECK_ARG(kp.vstride[s] % a->C == 0, "occd_sfa_lift_fwd: view stride must be a multiple of C");
    kp.vrow[s] = (int)(kp.vstride[s] / a->C < (1LL << 31) ? kp.vstride[s] / a->C : 0);   // used only when sfa_fits_int32
    int sh = -1;
    for (int b = 0; b < 30; ++b) if (a->div[s] == (1 << b)) sh = b;
    kp.shift[s] = sh;
  }
  kp.n_scales = a->n_scales; kp.C = a->C; kp.P = a->P; kp.N = a->N;
  kp.pix = reinterpret_cast<const long long*>(a->pix); kp.fov = a->fov;
  kp.out = a->out; kp.out_mode = a->out_mode; kp.out_cstride = a->out_cstride; kp.out_n = a->N;
  kp.perm_nyu = a->perm_nyu; kp.S1 = a->S1; kp.S2 = a->S2;
  if (a->perm_nyu) OCCD_CHECK_ARG(a->S1 > 0 && a->S2 > 0 && a->N % ((long long)a->S1 * a->S2) == 0, "occd_sfa_lift_fwd: NYU dims");
  kp.prior = a->prior; kp.scale_const = a->scale_const;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (a->feat_dtype == OCCD_DTYPE_F32) return launch_v<float>(kp, a->n_views, st);
  return launch_v<__nv_bfloat16>(kp, a->n_views, st);
}
