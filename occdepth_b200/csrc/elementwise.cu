// Small bandwidth-bound helpers around the implicit-GEMM convolutions (channels-last activations, bf16 or
// TF32-valued fp32: see Elem<T> in common.cuh).
#include "conv_common.cuh"

namespace {

// softmax over C (<= 32) planar fp32 channels -> bf16 channels-last window
// replaces nn.Softmax(dim=1) + torch.cat of modules.py:168-171
template <typename T>
__global__ void softmax_planar_to_cl_kernel(const float* __restrict__ in, T* __restrict__ out, int C,
                                            long long S, long long total, int cstride, int coff) {
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long b = i / S, s = i % S;
  const float* p = in + b * C * S + s;
  float m = -INFINITY;
  for (int c = 0; c < C; ++c) m = fmaxf(m, p[(long long)c * S]);
  float e[32];
  float sum = 0.f;
  for (int c = 0; c < C; ++c) { e[c] = expf(p[(long long)c * S] - m); sum += e[c]; }
  T* o = out + i * cstride + coff;
  for (int c = 0; c < C; ++c) o[c] = Elem<T>::cvt(e[c] / sum);
}

// out[b][r][c] (row-major [R][ldo]) = in[b][c][r] where in is channels-last [positions P][cstride] window:
// i.e. weight[f][m] = ctx[m][f]   (CRP3D.py:62-63,81: the mega-context becomes the B operand of the bmm)
template <typename T>
__global__ void cl_transpose_kernel(const T* __restrict__ in, T* __restrict__ out, int P,
                                    int C, int cstride, int coff, int ldo, long long in_bstride,
                                    long long out_bstride) {
  __shared__ T tile[32][33];
  const int b = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const T* inb = in + b * in_bstride;
  T* outb = out + b * out_bstride;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int pp = p0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (pp < P && c < C) ? inb[(long long)pp * cstride + coff + c] : Elem<T>::cvt(0.f);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, pp = p0 + threadIdx.x;
    if (c < C && pp < P) outb[(long long)c * ldo + pp] = tile[threadIdx.x][i];
  }
}

// copy a channel window between channels-last buffers (C multiple of 8)
// (16-byte pieces: 8 bf16 or 4 fp32 channels)
template <typename T>
__global__ void copy_channels_kernel(const T* __restrict__ in, T* __restrict__ out,
                                     long long positions, int C, int in_cs, int in_off, int out_cs, int out_off) {
  constexpr int E = 16 / sizeof(T);
  const int vec = C / E;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= positions * vec) return;
  const long long pos = i / vec;
  const int v = (int)(i % vec);
  *reinterpret_cast<uint4*>(out + pos * out_cs + out_off + v * E) =
      *reinterpret_cast<const uint4*>(in + pos * in_cs + in_off + v * E);
}

// class map of the caller-side post-processing (scripts/generate_output.py:94-95: softmax -> argmax -> uint16):
// softmax is monotonic, so the class is the FIRST index of the largest logit (np.argmax tie rule).  Optional
// label remap inv_map[class] of the submission writer (scripts/generate_kitti_submission.py:79).
constexpr int kMaxLut = 64;
struct ClassLut {
  int use;
  unsigned short v[kMaxLut];
};

__global__ void argmax_classes_kernel(const float* __restrict__ in, unsigned short* __restrict__ out, int C,
                                      long long S, long long total, const ClassLut lut) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long b = i / S, s = i - b * S;
  const float* p = in + b * C * S + s;
  float best = p[0];
  int arg = 0;
  for (int c = 1; c < C; ++c) {
    const float v = p[(long long)c * S];
    if (v > best) { best = v; arg = c; }
  }
  out[i] = lut.use ? lut.v[arg] : (unsigned short)arg;
}

// argmax_classes_kernel plus the top class's softmax probability (OCCD_OUT1_CLASS_U16_CONF's confidence): the same
// running arg-max and softmax as the class-map epilogues (conv_common.cuh), over the channels in ascending order
__global__ void argmax_classes_conf_kernel(const float* __restrict__ in, unsigned short* __restrict__ out,
                                           unsigned short* __restrict__ conf, int C, long long S, long long total,
                                           const ClassLut lut) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long b = i / S, s = i - b * S;
  const float* p = in + b * C * S + s;
  ClassArg a = class_arg_init();
  for (int c = 0; c < C; ++c) class_arg_take(a, p[(long long)c * S], c, true);
  out[i] = lut.use ? lut.v[a.c] : (unsigned short)a.c;
  const __half_raw h = __float2half_rn(class_arg_conf(a));
  conf[i] = h.x;
}

// argmax_classes_conf_kernel's pass, then a second one over the same logits that writes every class's probability
// (OCCD_OUT1_CLASS_U16_PROBS's second part, probs[b][c][s])
__global__ void class_probs_kernel(const float* __restrict__ in, unsigned short* __restrict__ out,
                                   unsigned short* __restrict__ probs, int C, long long S, long long total,
                                   const ClassLut lut) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long b = i / S, s = i - b * S;
  const float* p = in + b * C * S + s;
  ClassArg a = class_arg_init();
  for (int c = 0; c < C; ++c) class_arg_take(a, p[(long long)c * S], c, true);
  out[i] = lut.use ? lut.v[a.c] : (unsigned short)a.c;
  unsigned short* q = probs + b * C * S + s;
  for (int c = 0; c < C; ++c) {
    const __half_raw h = __float2half_rn(class_arg_prob(a, p[(long long)c * S]));
    q[(long long)c * S] = h.x;
  }
}

int class_lut_of(const int* lut, int C, ClassLut* l) {
  l->use = lut ? 1 : 0;
  for (int c = 0; c < kMaxLut; ++c) l->v[c] = (lut && c < C) ? (unsigned short)lut[c] : 0;  // .astype(np.uint16)
  return OCCD_OK;
}

}  // namespace

extern "C" int occd_argmax_classes(const float* in, void* out, long long B, int C, long long S, const int* lut,
                                   void* stream) {
  OCCD_CHECK_ARG(in && out && B > 0 && C > 0 && C <= 65535 && S > 0, "occd_argmax_classes: args");
  OCCD_CHECK_ARG(!lut || C <= kMaxLut, "occd_argmax_classes: a label remap supports at most 64 classes");
  const long long total = B * S;
  OCCD_CHECK_ARG((total + 255) / 256 <= 2147483647LL, "occd_argmax_classes: too many positions");
  ClassLut l;
  class_lut_of(lut, C, &l);
  argmax_classes_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      in, (unsigned short*)out, C, S, total, l);
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

extern "C" int occd_argmax_classes_conf(const float* in, void* out, void* conf, long long B, int C, long long S,
                                        const int* lut, void* stream) {
  OCCD_CHECK_ARG(in && out && conf && B > 0 && C > 0 && C <= 65535 && S > 0, "occd_argmax_classes_conf: args");
  OCCD_CHECK_ARG(reinterpret_cast<uintptr_t>(out) % 2 == 0 && reinterpret_cast<uintptr_t>(conf) % 2 == 0,
                 "occd_argmax_classes_conf: out and conf must be 2-byte aligned");
  OCCD_CHECK_ARG(!lut || C <= kMaxLut, "occd_argmax_classes_conf: a label remap supports at most 64 classes");
  const long long total = B * S;
  OCCD_CHECK_ARG((total + 255) / 256 <= 2147483647LL, "occd_argmax_classes_conf: too many positions");
  ClassLut l;
  class_lut_of(lut, C, &l);
  argmax_classes_conf_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      in, (unsigned short*)out, (unsigned short*)conf, C, S, total, l);
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

extern "C" int occd_class_probs(const float* logits, void* map, void* probs, long long B, int C, long long S,
                                const int* lut, void* stream) {
  OCCD_CHECK_ARG(logits && map && probs && B > 0 && C > 0 && C <= 65535 && S > 0, "occd_class_probs: args");
  OCCD_CHECK_ARG(reinterpret_cast<uintptr_t>(map) % 2 == 0 && reinterpret_cast<uintptr_t>(probs) % 2 == 0,
                 "occd_class_probs: map and probs must be 2-byte aligned");
  OCCD_CHECK_ARG(!lut || C <= kMaxLut, "occd_class_probs: a label remap supports at most 64 classes");
  const long long total = B * S;
  OCCD_CHECK_ARG((total + 255) / 256 <= 2147483647LL, "occd_class_probs: too many positions");
  ClassLut l;
  class_lut_of(lut, C, &l);
  class_probs_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      logits, (unsigned short*)map, (unsigned short*)probs, C, S, total, l);
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

extern "C" int occd_softmax_planar_to_cl(const float* in, void* out, int dtype, long long B, int C, long long S,
                                         int cstride, int coff, void* stream) {
  OCCD_CHECK_ARG(in && out && B > 0 && C > 0 && C <= 32 && S > 0 && coff + C <= cstride, "occd_softmax_planar_to_cl: args");
  const long long total = B * S;
  OCCD_DISPATCH_DTYPE(dtype, T, OCCD_LAUNCH_CHECKED(softmax_planar_to_cl_kernel<T>, dim3((unsigned)((total + 255) / 256)),
                                                    dim3(256), 0, (cudaStream_t)stream, in, (T*)out, C, S, total,
                                                    cstride, coff));
  return OCCD_OK;
}

extern "C" int occd_cl_transpose(const void* in, void* out, int dtype, int B, int P, int C, int cstride, int coff,
                                 int ldo, long long out_bstride, void* stream) {
  OCCD_CHECK_ARG(in && out && B > 0 && P > 0 && C > 0 && coff + C <= cstride && ldo >= P, "occd_cl_transpose: args");
  dim3 grid((P + 31) / 32, (C + 31) / 32, B), block(32, 8);
  OCCD_DISPATCH_DTYPE(dtype, T, (cl_transpose_kernel<T><<<grid, block, 0, (cudaStream_t)stream>>>(
                                     (const T*)in, (T*)out, P, C, cstride, coff, ldo, (long long)P * cstride,
                                     out_bstride)));
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

extern "C" int occd_copy_channels(const void* in, void* out, int dtype, long long positions, int C, int in_cstride,
                                  int in_coff, int out_cstride, int out_coff, void* stream) {
  OCCD_CHECK_ARG(in && out && positions > 0 && C > 0 && C % 8 == 0 && in_coff % 8 == 0 && out_coff % 8 == 0 &&
                 in_cstride % 8 == 0 && out_cstride % 8 == 0, "occd_copy_channels: args");
  const long long total = positions * (C / (dtype == OCCD_DTYPE_F32 ? 4 : 8));
  OCCD_DISPATCH_DTYPE(dtype, T, (copy_channels_kernel<T><<<(unsigned)((total + 255) / 256), 256, 0,
                                                            (cudaStream_t)stream>>>(
                                     (const T*)in, (T*)out, positions, C, in_cstride, in_coff, out_cstride,
                                     out_coff)));
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}
