// Shared-memory-tiled depthwise KxK conv + folded BN + activation + squeeze (channels-last, element type T =
// __nv_bfloat16 or TF32-valued float -- see Elem<T> in common.cuh).
// Same contract as dwconv_kernel (effnet_ops.cu); replaces geffnet conv_dw + bn + act (+ the SE squeeze) as
// iterated by Encoder.forward (unet2d.py:188-196).
//
// Why a second variant: the direct kernel keeps a (PX-1)*S+K wide input window per filter row in registers and
// ends up at 229-252 registers/thread for K = 5 (one 8-warp block per SM), so every layer runs latency-bound at
// 0.6-0.9 TB/s.  Here a CTA stages ONE zero-filled input halo tile (TH x 16 outputs x 8*CVB channels) in shared
// memory with cp.async -- every input byte crosses L2->SM once, coalesced in 16*CVB-byte runs -- and the FMA loop
// reads 16-byte vectors from shared memory, so the register budget is the 4x8 accumulators + one filter row.
//
// The three phases are written as __host__ __device__ functions of (block index, thread index): the CUDA kernel
// calls them with __syncthreads() in between, and tests/host_emul/ runs exactly the same index arithmetic
// thread by thread on the CPU (no GPU needed to check tiling, padding, stride and ragged-edge handling).
#pragma once
#include <string.h>
#include <math.h>
#include "common.cuh"

namespace dwt {

constexpr int kTW = 16;  // output tile width
// PXV = consecutive outputs (along W) per thread: 4 with 256-thread CTAs, or 8 with 128-thread CTAs -- one input
// vector then feeds up to K taps of 8 outputs, and the filter row is fetched once per 8 outputs: 28 % fewer
// shared-memory wavefronts per output (the kernel is shared-memory-pipe bound: ncu r02, MIO throttle the top stall)

#define DWT_HD __host__ __device__ __forceinline__

struct Args {
  const void* in;     // T [B][H][W][cs_in]
  const float* w;     // [K*K][C] BN-folded filter taps
  const float* bias;  // [C]
  void* out;          // T [B][OH][OW][cs_out]
  long long* pool;    // [B][C] fixed-point (2^-24) squeeze sums, or null
  int H, W, OH, OW, C, cs_in, cs_out, pad_top, pad_left, act, tiles_x;
};

template <typename T, int K, int S, int CVB, int TH, int PXV = 4>
struct Cfg {
  static constexpr int PX = PXV;
  static constexpr int NT = 1024 / PXV;           // threads per CTA (256 / 128): the slots of one pass cover 16 x 16
  static constexpr int PIECES = (int)sizeof(T) / 2;  // 16-byte pieces per 8-channel vector
  static constexpr int CT = CVB * 8;              // channels per CTA
  static constexpr int GX = kTW / PX;             // thread groups along W
  static constexpr int GROUPS = NT / CVB;         // (row, x-group) slots per pass
  static constexpr int RPP = GROUPS / GX;         // output rows per pass
  static constexpr int PASSES = TH / RPP;
  static_assert(TH % RPP == 0 && PASSES >= 1, "tile height must be a multiple of the rows per pass");
  static constexpr int ITH = (TH - 1) * S + K, ITW = (kTW - 1) * S + K;  // input halo tile
  static constexpr int NIN = (PX - 1) * S + K;    // input vectors one thread reads per filter row
  static constexpr int TILE_ELEMS = ITH * ITW * CT;  // T
  static constexpr int W_ELEMS = K * K * CT;         // fp32, layout [tap][half][CVB][4]
  static constexpr int RED_ELEMS = GROUPS * CT;      // fp32
  static constexpr size_t kTileBytes = (size_t)TILE_ELEMS * sizeof(T);
  static constexpr size_t kSmemBytes = kTileBytes + (size_t)W_ELEMS * 4 + (size_t)RED_ELEMS * 4;
  static_assert(kTileBytes % 16 == 0, "weights must start 16-byte aligned");
};

DWT_HD void copy16_async(void* smem_dst, const void* gsrc) {
#ifdef __CUDA_ARCH__
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)),
               "l"(gsrc)
               : "memory");
#else
  memcpy(smem_dst, gsrc, 16);
#endif
}

DWT_HD void zero16(void* smem_dst) {
#ifdef __CUDA_ARCH__
  *reinterpret_cast<uint4*>(smem_dst) = make_uint4(0u, 0u, 0u, 0u);
#else
  memset(smem_dst, 0, 16);
#endif
}

DWT_HD float bits2f(uint32_t u) {
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  memcpy(&f, &u, 4);
  return f;
#endif
}

// 8 bf16 (one 16-byte vector) -> 4 float2; element 2i sits in the low half of word i
DWT_HD void unpack8f2(const uint4& u, float2* f) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) f[i] = make_float2(bits2f(w[i] << 16), bits2f(w[i] & 0xffff0000u));
}

DWT_HD uint32_t f2bits(float f) {
#ifdef __CUDA_ARCH__
  return __float_as_uint(f);
#else
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
#endif
}

// fp32 -> nearest TF32 value (10-bit mantissa), ties away from zero: what cvt.rna.tf32.f32 computes
DWT_HD float tf32_rna(float v) {
#ifdef __CUDA_ARCH__
  return round_tf32(v);
#else
  return bits2f((f2bits(v) + 0x1000u) & 0xffffe000u);
#endif
}

// one 8-channel vector of the staged tile -> 4 float2
// (sw: the fp32 tile's halves are stored swapped at this column, see phase_load)
DWT_HD void load8f2(const __nv_bfloat16* p, float2* f, int) { unpack8f2(*reinterpret_cast<const uint4*>(p), f); }
DWT_HD void load8f2(const float* p, float2* f, int sw) {
  const float4 a = *reinterpret_cast<const float4*>(p + 4 * sw), b = *reinterpret_cast<const float4*>(p + 4 - 4 * sw);
  f[0] = make_float2(a.x, a.y); f[1] = make_float2(a.z, a.w);
  f[2] = make_float2(b.x, b.y); f[3] = make_float2(b.z, b.w);
}

// round + store one output vector; v[] is left holding the stored values (what the next layer reads)
DWT_HD void store8(__nv_bfloat16* p, float* v) {
  uint4 packed;
  uint32_t* pw = reinterpret_cast<uint32_t*>(&packed);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __nv_bfloat162 h2 = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
    uint32_t bits;
    memcpy(&bits, &h2, 4);
    pw[i] = bits;
  }
  *reinterpret_cast<uint4*>(p) = packed;
  float2 r[4];
  unpack8f2(packed, r);
#pragma unroll
  for (int i = 0; i < 4; ++i) { v[2 * i] = r[i].x; v[2 * i + 1] = r[i].y; }
}
DWT_HD void store8(float* p, float* v) {
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = tf32_rna(v[i]);
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}

// two IEEE fp32 FMAs (sm_90 has no packed FFMA2; the host emulation and the device compute the same values)
DWT_HD float2 fma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

// activation over one 8-channel vector (device: the same uniform-branch fast-math epilogue as the direct kernel)
template <bool FAST_SILU>
DWT_HD void act8(float* v, int act) {
#ifdef __CUDA_ARCH__
  apply_act8<FAST_SILU>(v, act);
#else
  for (int i = 0; i < 8; ++i) {
    switch (act) {
      case ACT_RELU: v[i] = v[i] > 0.f ? v[i] : 0.f; break;
      case ACT_LEAKY: v[i] = v[i] > 0.f ? v[i] : 0.01f * v[i]; break;
      case ACT_SILU: v[i] = v[i] / (1.f + expf(-v[i])); break;
      case ACT_SIGMOID: v[i] = 1.f / (1.f + expf(-v[i])); break;
      default: break;
    }
  }
#endif
}

struct BlockIdx {
  int x, y, z;
};

// ---- phase 1: stage the zero-filled input halo tile and this CTA's filter taps in shared memory ----------------
template <typename T, int K, int S, int CVB, int TH, int PXV = 4>
DWT_HD void phase_load(const Args& a, BlockIdx blk, int tid, T* tile, float* wsm) {
  using C_ = Cfg<T, K, S, CVB, TH, PXV>;
  const int b = blk.z, c0 = blk.y * C_::CT;
  const int gy0 = (blk.x / a.tiles_x) * TH * S - a.pad_top;
  const int gx0 = (blk.x % a.tiles_x) * kTW * S - a.pad_left;
  constexpr int PC = C_::PIECES, EPP = 8 / PC;   // 16-byte pieces per vector, elements per piece
  const T* inb = reinterpret_cast<const T*>(a.in) + (long long)b * a.H * a.W * a.cs_in;
  for (int i = tid; i < C_::ITH * C_::ITW * CVB * PC; i += C_::NT) {
    const int piece = i % (CVB * PC), pix = i / (CVB * PC);   // piece = (cv, half): consecutive 16-byte runs
    const int iy = pix / C_::ITW, ix = pix - iy * C_::ITW;
    const int gy = gy0 + iy, gx = gx0 + ix, c = c0 + piece * EPP;
    // fp32 tiles: the two 16-byte halves of an 8-channel vector swap places in every other group of C_::PX*S columns, so
    // the 8 lanes of a quarter warp (4 channel vectors x 2 column groups, 512 bytes apart) hit 32 distinct banks when
    // they read the same half (ncu r02: a third of the kernel's shared-memory wavefronts were bank conflicts)
    const int sw = PC == 2 ? ((ix / (C_::PX * S)) & 1) : 0;
    T* dst = tile + (long long)pix * C_::CT + (piece ^ sw) * EPP;
    if (gy >= 0 && gy < a.H && gx >= 0 && gx < a.W && c < a.C)
      copy16_async(dst, inb + ((long long)gy * a.W + gx) * a.cs_in + c);
    else
      zero16(dst);
  }
  // filter taps: wsm[tap][half][cv][4] so that the 8 lanes of a quarter warp read 128 contiguous bytes
  for (int i = tid; i < K * K * 2 * CVB; i += C_::NT) {
    const int cv = i % CVB, h = (i / CVB) % 2, tap = i / (2 * CVB);
    const int c = c0 + cv * 8 + h * 4;
    float* dst = wsm + ((tap * 2 + h) * CVB + cv) * 4;
    if (c < a.C)
      copy16_async(dst, a.w + (long long)tap * a.C + c);
    else
      zero16(dst);
  }
}

// ---- phase 2: FMA loop out of shared memory, activation, bf16 store, per-thread squeeze partials -> red[] -----
template <typename T, int K, int S, int CVB, int TH, int PXV = 4>
DWT_HD void phase_compute(const Args& a, BlockIdx blk, int tid, const T* tile, const float* wsm,
                          float* red) {
  using C_ = Cfg<T, K, S, CVB, TH, PXV>;
  const int cv = tid % CVB, g = tid / CVB;
  const int gxi = g % C_::GX, r0 = g / C_::GX;
  const int b = blk.z, c = blk.y * C_::CT + cv * 8;
  const int ty0 = (blk.x / a.tiles_x) * TH, ox0 = (blk.x % a.tiles_x) * kTW + gxi * C_::PX;
  const bool cvalid = c < a.C;
  float2 psum[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) psum[i] = make_float2(0.f, 0.f);
#pragma unroll 1
  for (int pass = 0; pass < C_::PASSES; ++pass) {
    const int orow = r0 + pass * C_::RPP, oy = ty0 + orow;
    if (!cvalid || oy >= a.OH || ox0 >= a.OW) continue;
    float2 acc[C_::PX][4];
    {
      const float4 b0 = *reinterpret_cast<const float4*>(a.bias + c);
      const float4 b1 = *reinterpret_cast<const float4*>(a.bias + c + 4);
#pragma unroll
      for (int p = 0; p < C_::PX; ++p) {
        acc[p][0] = make_float2(b0.x, b0.y);
        acc[p][1] = make_float2(b0.z, b0.w);
        acc[p][2] = make_float2(b1.x, b1.y);
        acc[p][3] = make_float2(b1.z, b1.w);
      }
    }
#pragma unroll
    for (int ky = 0; ky < K; ++ky) {
      float2 wv[K][4];
#pragma unroll
      for (int kx = 0; kx < K; ++kx) {
        const float* wp = wsm + (((ky * K + kx) * 2) * CVB + cv) * 4;
        const float4 w0 = *reinterpret_cast<const float4*>(wp);
        const float4 w1 = *reinterpret_cast<const float4*>(wp + CVB * 4);
        wv[kx][0] = make_float2(w0.x, w0.y);
        wv[kx][1] = make_float2(w0.z, w0.w);
        wv[kx][2] = make_float2(w1.x, w1.y);
        wv[kx][3] = make_float2(w1.z, w1.w);
      }
      const T* rowp = tile + ((long long)(orow * S + ky) * C_::ITW + gxi * C_::PX * S) * C_::CT + cv * 8;
#pragma unroll
      for (int j = 0; j < C_::NIN; ++j) {
        float2 x[4];
        load8f2(rowp + j * C_::CT, x, C_::PIECES == 2 ? ((gxi + j / (C_::PX * S)) & 1) : 0);
#pragma unroll
        for (int kx = 0; kx < K; ++kx) {
          const int d = j - kx;  // input column j feeds output p = d / S through tap kx (compile-time resolved)
          if (d >= 0 && d % S == 0 && d / S < C_::PX) {
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[d / S][i] = fma2(x[i], wv[kx][i], acc[d / S][i]);
          }
        }
      }
    }
    T* orow_p = reinterpret_cast<T*>(a.out) + (((long long)b * a.OH + oy) * a.OW + ox0) * a.cs_out + c;
#pragma unroll
    for (int p = 0; p < C_::PX; ++p) {
      if (ox0 + p >= a.OW) break;
      float v[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        v[2 * i] = acc[p][i].x;
        v[2 * i + 1] = acc[p][i].y;
      }
      act8<sizeof(T) == 2>(v, a.act);
      store8(orow_p + (long long)p * a.cs_out, v);
      if (a.pool) {
        // squeeze what the next layer will actually read (the rounded activation)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          psum[i].x += v[2 * i];
          psum[i].y += v[2 * i + 1];
        }
      }
    }
  }
  if (a.pool) {
    float* rp = red + g * C_::CT + cv * 8;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      rp[2 * i] = psum[i].x;
      rp[2 * i + 1] = psum[i].y;
    }
  }
}

// ---- phase 3: one thread per channel folds the CTA's partials and adds them to pool[b][c] (integer atomics:
//      order-independent, so the SE gates are bit-reproducible run to run) ---------------------------------------
template <typename T, int K, int S, int CVB, int TH, int PXV = 4>
DWT_HD void phase_pool(const Args& a, BlockIdx blk, int tid, const float* red) {
  using C_ = Cfg<T, K, S, CVB, TH, PXV>;
  const int c = blk.y * C_::CT + tid;
  if (tid >= C_::CT || c >= a.C) return;
  float s = 0.f;
  for (int g = 0; g < C_::GROUPS; ++g) s += red[g * C_::CT + tid];
  long long* dst = a.pool + (long long)blk.z * a.C + c;
#ifdef __CUDA_ARCH__
  atomicAdd(reinterpret_cast<unsigned long long*>(dst), (unsigned long long)__float2ll_rn(s * 16777216.f));
#else
  *dst += llrintf(s * 16777216.f);
#endif
}

#ifdef __CUDACC__
template <typename T, int K, int S, int CVB, int TH, int PXV = 4>
__global__ void __launch_bounds__(1024 / PXV, PXV == 4 ? 2 : 3) dwconv_tiled_kernel(const Args a) {
  using C_ = Cfg<T, K, S, CVB, TH, PXV>;
  pdl_wait();
  extern __shared__ __align__(16) unsigned char dwt_smem[];
  T* tile = reinterpret_cast<T*>(dwt_smem);
  float* wsm = reinterpret_cast<float*>(dwt_smem + C_::kTileBytes);
  float* red = wsm + C_::W_ELEMS;
  const BlockIdx blk{(int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z};
  const int tid = threadIdx.x;
  phase_load<T, K, S, CVB, TH, PXV>(a, blk, tid, tile, wsm);
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  phase_compute<T, K, S, CVB, TH, PXV>(a, blk, tid, tile, wsm, red);
  if (a.pool) {
    __syncthreads();
    phase_pool<T, K, S, CVB, TH, PXV>(a, blk, tid, red);
  }
}
#endif

// tile-shape choice shared by the launcher and the host emulation: CVB = 4 for layers narrower than 64 channels
// (and always for fp32: 32 channels x 4 bytes = the same 128-byte runs and tile bytes as 64 bf16 channels),
// tall tiles (TH = 16) when the layer still fills the GPU twice over, TH = 8 otherwise and for stride 2
struct Choice {
  int cvb, th;
};
static inline Choice choose(int B, int OH, int OW, int C, int S, int n_sms, int elem_size = 2) {
  Choice ch;
  ch.cvb = (C < 64 || elem_size == 4) ? 4 : 8;
  if (ch.cvb == 4) {
    ch.th = 16;   // 64 (row, x-group) slots per pass / 4 x-groups = 16 rows per pass
  } else if (S == 2) {
    ch.th = 8;
  } else {
    const long long tiles16 = (long long)B * ((OH + 15) / 16) * ((OW + kTW - 1) / kTW) * ((C + 63) / 64);
    ch.th = tiles16 >= 4LL * n_sms ? 16 : 8;
  }
  return ch;
}

}  // namespace dwt
