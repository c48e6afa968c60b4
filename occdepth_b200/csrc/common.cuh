// Shared device/host helpers for the occdepth_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#define OCCD_OK 0
#define OCCD_ERR_ARG 1      // bad argument (null pointer, unsupported shape)
#define OCCD_ERR_CUDA 2     // CUDA runtime/driver error (see occd_last_error)
#define OCCD_ERR_UNSUPPORTED 3

extern "C" void occd_set_last_error(const char* msg);

#define OCCD_CHECK_ARG(cond, msg)                 \
  do {                                            \
    if (!(cond)) {                                \
      occd_set_last_error(msg);                   \
      return OCCD_ERR_ARG;                        \
    }                                             \
  } while (0)

#define OCCD_CHECK_LAUNCH()                                  \
  do {                                                       \
    cudaError_t e__ = cudaGetLastError();                    \
    if (e__ != cudaSuccess) {                                \
      occd_set_last_error(cudaGetErrorString(e__));          \
      return OCCD_ERR_CUDA;                                  \
    }                                                        \
  } while (0)

// activation codes shared by every epilogue (host enum mirrors include/occdepth_b200.h)
enum : int { ACT_NONE = 0, ACT_RELU = 1, ACT_LEAKY = 2, ACT_SILU = 3, ACT_SIGMOID = 4 };

__device__ __forceinline__ float apply_act(float v, int act) {
  switch (act) {
    case ACT_RELU: return fmaxf(v, 0.f);
    case ACT_LEAKY: return v > 0.f ? v : 0.01f * v;
    case ACT_SILU: return v / (1.f + __expf(-v));
    case ACT_SIGMOID: return 1.f / (1.f + __expf(-v));
    default: return v;
  }
}

// activation over 8 values with ONE uniform branch (keeps the epilogues free of per-element switches)
// SiLU with ONE MUFU op per element: x sigmoid(x) = h + h tanh(h), h = x / 2 (tanh.approx.f32: max relative error
// 2^-11).  Used by the bf16 mode only, whose stores round to 2^-9; the tf32 mode keeps ex2 + rcp (two MUFU ops)
__device__ __forceinline__ float silu_tanh(float x) {
  const float h = 0.5f * x;
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
  return fmaf(h, t, h);
}

template <bool FAST_SILU = false>
__device__ __forceinline__ void apply_act8(float* v, int act) {
  if (act == ACT_NONE) return;
  if (act == ACT_RELU) {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = fmaxf(v[i], 0.f);
  } else if (act == ACT_LEAKY) {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = v[i] > 0.f ? v[i] : 0.01f * v[i];
  } else if (act == ACT_SILU) {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = FAST_SILU ? silu_tanh(v[i]) : __fdividef(v[i], 1.f + __expf(-v[i]));
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = __fdividef(1.f, 1.f + __expf(-v[i]));
  }
}

__device__ __forceinline__ float bf2f(__nv_bfloat16 v) { return __bfloat162float(v); }

// 8 x bf16 <-> 8 x float through one 16-byte vector
struct alignas(16) bf16x8 {
  __nv_bfloat162 v[4];
};

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(p[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 u;
  __nv_bfloat162* p = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) p[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return u;
}

__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}


// ---------------------------------------------------------------------------------------------------------------
// Activation element types.  Two precision modes share every kernel (template parameter T):
//   __nv_bfloat16 : bf16 storage, wgmma .bf16 operands ("bf16" throughput mode)
//   float         : fp32 storage holding TF32-representable values (10-bit mantissa, round-to-nearest-away at every
//                   store), wgmma .tf32 operands -- the reference-precision mode: the reference's convolutions
//                   are fp32 nn.Conv*d (modules.py:158-175, DDR.py:111-139) which PyTorch itself runs as TF32 on CUDA
// One "vector" is always 8 consecutive channels: 16 bytes of bf16 or 32 bytes of fp32.
__device__ __forceinline__ float round_tf32(float v) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
  return __uint_as_float(u);
}

// 8 fp32 values as two 16-byte accesses (sm_90 has no 256-bit global loads / stores)
__device__ __forceinline__ void ld256_f(const float* p, float* f) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
__device__ __forceinline__ void ld256_nc_f(const float* p, float* f) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p + 4));
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
__device__ __forceinline__ void st256_f(float* p, const float* f) {
  *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(f[4], f[5], f[6], f[7]);
}

template <typename T> struct Elem;
template <> struct Elem<__nv_bfloat16> {
  static constexpr int kDtype = 1;  // OCCD_DTYPE_BF16
  // what the consumer of a stored value reads back
  static __device__ __forceinline__ float rnd(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
  static __device__ __forceinline__ __nv_bfloat16 cvt(float v) { return __float2bfloat16_rn(v); }
  static __device__ __forceinline__ float up(__nv_bfloat16 v) { return __bfloat162float(v); }
  static __device__ __forceinline__ void ld8(const __nv_bfloat16* p, float* f) {
    unpack8(*reinterpret_cast<const uint4*>(p), f);
  }
  static __device__ __forceinline__ void ld8_nc(const __nv_bfloat16* p, float* f) {
    unpack8(__ldg(reinterpret_cast<const uint4*>(p)), f);
  }
  static __device__ __forceinline__ void st8(__nv_bfloat16* p, const float* f) {
    *reinterpret_cast<uint4*>(p) = pack8(f);
  }
  static __device__ __forceinline__ void st8_exact(__nv_bfloat16* p, const float* f) { st8(p, f); }
  // st8 that also returns the stored (rounded) values
  static __device__ __forceinline__ void st8_rb(__nv_bfloat16* p, float* f) {
    const uint4 u = pack8(f);
    *reinterpret_cast<uint4*>(p) = u;
    unpack8(u, f);
  }
};
template <> struct Elem<float> {
  static constexpr int kDtype = 0;  // OCCD_DTYPE_F32 (TF32-valued)
  static __device__ __forceinline__ float rnd(float v) { return round_tf32(v); }
  static __device__ __forceinline__ float cvt(float v) { return round_tf32(v); }
  static __device__ __forceinline__ float up(float v) { return v; }
  static __device__ __forceinline__ void ld8(const float* p, float* f) { ld256_f(p, f); }
  static __device__ __forceinline__ void ld8_nc(const float* p, float* f) { ld256_nc_f(p, f); }
  static __device__ __forceinline__ void st8(float* p, const float* f) {
    float r[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) r[i] = round_tf32(f[i]);
    st256_f(p, r);
  }
  static __device__ __forceinline__ void st8_exact(float* p, const float* f) { st256_f(p, f); }
  static __device__ __forceinline__ void st8_rb(float* p, float* f) {
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = round_tf32(f[i]);
    st256_f(p, f);
  }
};

// host-side dispatch over the activation dtype of a C-ABI call (OCCD_DTYPE_F32 | OCCD_DTYPE_BF16)
#define OCCD_DISPATCH_DTYPE(dtype, T, ...)                                   \
  do {                                                                       \
    if ((dtype) == 1) { using T = __nv_bfloat16; __VA_ARGS__; }              \
    else if ((dtype) == 0) { using T = float; __VA_ARGS__; }                 \
    else { occd_set_last_error("unsupported activation dtype"); return OCCD_ERR_ARG; } \
  } while (0)

static inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// ---------------------------------------------------------------------------------------------------------------
// Programmatic dependent launch for every kernel of the plan: a kernel launched through occd_launch carries
// cudaLaunchAttributeProgrammaticStreamSerialization, so its blocks may be scheduled while the previous grid drains;
// pdl_wait() -- the kernel's FIRST statement, before any global read or write -- blocks until that grid has
// completed and flushed.  OCCD_PDL=0 falls back to plain launches (pdl_wait is then a no-op).
#include <stdlib.h>
#include <utility>
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

static inline int occd_pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("OCCD_PDL");
    v = (e && atoi(e) == 0) ? 0 : 1;
  }
  return v;
}

template <typename... KArgs, typename... Args>
static inline cudaError_t occd_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                      Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = occd_pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

#define OCCD_LAUNCH_CHECKED(...)                              \
  do {                                                        \
    cudaError_t e__ = occd_launch(__VA_ARGS__);               \
    if (e__ != cudaSuccess) {                                 \
      occd_set_last_error(cudaGetErrorString(e__));           \
      return OCCD_ERR_CUDA;                                   \
    }                                                         \
  } while (0)
