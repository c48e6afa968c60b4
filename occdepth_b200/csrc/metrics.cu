// Semantic scene completion metrics on the device: the confusion matrix of a class map against its labels, from which
// every count of the reference's SSCMetrics.add_batch follows (loss/sscMetrics.py:70-91, called by OccDepth.step
// :526-529 with nonempty=None).  The reference copies the logits to the host and runs np.argmax plus three np.where
// passes per class; here one pass reads the class map and the labels once.
#include <string.h>

#include "common.cuh"
#include "ssc_labels.cuh"
#include "../../include/occdepth_b200.h"

namespace {

using namespace ssc_labels;

constexpr int kMaxClasses = 64;          // the class-map remap's cap: (64*64 + 1) uint32 bins = 16 KB of shared memory
constexpr int kGroup = 8;                // elements per thread and iteration: one 16-byte load of a uint16 map
constexpr int kThreads = 256;

__device__ __forceinline__ int pred_class(unsigned short v, int C) { return v < C ? (int)v : kInvalid; }
__device__ __forceinline__ int pred_class(long long v, int C) {
  return (unsigned long long)v < (unsigned long long)C ? (int)v : kInvalid;
}

// kGroup consecutive elements: vector loads when the group is aligned (16 bytes, or 8 for a uint8 group), else one
// load per element
template <bool VEC, typename T>
__device__ __forceinline__ void load_group(const T* __restrict__ p, T (&v)[kGroup]) {
  constexpr int NB = kGroup * (int)sizeof(T);
  if constexpr (!VEC) {
#pragma unroll
    for (int k = 0; k < kGroup; ++k) v[k] = p[k];
  } else if constexpr (NB >= 16) {
    uint4 r[NB / 16];
#pragma unroll
    for (int k = 0; k < NB / 16; ++k) r[k] = __ldcs(reinterpret_cast<const uint4*>(p) + k);
    memcpy(v, r, NB);
  } else {
    const uint2 r = __ldcs(reinterpret_cast<const uint2*>(p));
    memcpy(v, &r, NB);
  }
}

// counts[g*C + p] += voxels with label g and prediction p; counts[C*C] += invalid voxels; label 255 is skipped.
// Elements [0, head) and [head + kGroup*ngroups, n) are read one by one (the vector groups start at `head`, where both
// pointers are aligned).  Bins are block-private uint32 in shared memory (the host sizes the grid so that no block
// counts 2^31 voxels); bin (0,0), which holds most voxels of a scene, is a register per thread, so the common case
// never contends on one shared address.  One global atomic per nonzero bin and block at the end.
template <bool VEC, typename P, typename L>
__global__ void __launch_bounds__(kThreads) ssc_confusion_kernel(const P* __restrict__ pred,
                                                                 const L* __restrict__ label, long long n,
                                                                 long long head, long long ngroups, int C,
                                                                 unsigned long long* __restrict__ counts) {
  extern __shared__ unsigned int bins[];
  const int nbins = C * C + 1;
  for (int i = threadIdx.x; i < nbins; i += kThreads) bins[i] = 0u;
  __syncthreads();
  unsigned int zero_zero = 0;
  auto count = [&](P pv, L lv) {
    const int g = label_class(lv, C);
    if (g == kIgnore) return;
    const int p = pred_class(pv, C);
    const int bin = (g < 0 || p < 0) ? C * C : g * C + p;
    if (bin == 0) ++zero_zero;
    else atomicAdd(&bins[bin], 1u);
  };
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long gi = (long long)blockIdx.x * kThreads + threadIdx.x; gi < ngroups; gi += stride) {
    const long long e = head + gi * kGroup;
    P pv[kGroup];
    L lv[kGroup];
    load_group<VEC>(pred + e, pv);
    load_group<VEC>(label + e, lv);
#pragma unroll
    for (int k = 0; k < kGroup; ++k) count(pv[k], lv[k]);
  }
  if (blockIdx.x == 0) {                                   // head and tail: fewer than 2 * kGroup elements
    const long long tail = head + ngroups * kGroup;
    const long long i = threadIdx.x < head ? threadIdx.x : tail + (threadIdx.x - head);
    if (threadIdx.x < 2 * kGroup && i < n && (i < head || i >= tail)) count(pred[i], label[i]);
  }
  if (zero_zero) atomicAdd(&bins[0], zero_zero);
  __syncthreads();
  for (int i = threadIdx.x; i < nbins; i += kThreads)
    if (bins[i]) atomicAdd(&counts[i], (unsigned long long)bins[i]);
}

template <typename P, typename L>
int launch_confusion(const void* pred, const void* label, long long n, int C, long long* counts, cudaStream_t st) {
  if ((uintptr_t)pred % sizeof(P) || (uintptr_t)label % sizeof(L)) {
    occd_set_last_error("occd_ssc_confusion: pred / label are not aligned to their element size");
    return OCCD_ERR_ARG;
  }
  // first offset (< kGroup) from which both arrays' groups are aligned for the vector loads, if there is one
  const uintptr_t ap = kGroup * sizeof(P) < 16 ? kGroup * sizeof(P) : 16;
  const uintptr_t al = kGroup * sizeof(L) < 16 ? kGroup * sizeof(L) : 16;
  long long head = -1;
  for (int h = 0; h < kGroup && h < n; ++h)
    if (((uintptr_t)pred + h * sizeof(P)) % ap == 0 && ((uintptr_t)label + h * sizeof(L)) % al == 0) {
      head = h;
      break;
    }
  const bool vec = head >= 0;
  if (!vec) head = 0;
  const long long ngroups = (n - head) / kGroup;
  static int n_sms = 0;
  if (n_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n_sms <= 0) n_sms = 132;
  }
  // 4 blocks per SM keep enough loads in flight to stream both arrays; more blocks only add flush atomics.  A block
  // counts at most ceil(ngroups / blocks) * kGroup + 2 * kGroup voxels, which must stay below 2^31 (uint32 bins)
  long long blocks = (ngroups + kThreads - 1) / kThreads;
  if (blocks > 4LL * n_sms) blocks = 4LL * n_sms;
  const long long per_block = 1LL << 30;
  const long long need = (ngroups * kGroup + per_block - 1) / per_block;
  if (blocks < need) blocks = need;
  if (blocks < 1) blocks = 1;
  OCCD_CHECK_ARG(blocks <= 2147483647LL, "occd_ssc_confusion: too many voxels");
  const size_t smem = (size_t)(C * C + 1) * sizeof(unsigned int);
  auto* out = reinterpret_cast<unsigned long long*>(counts);
  if (vec)
    ssc_confusion_kernel<true, P, L><<<(unsigned)blocks, kThreads, smem, st>>>((const P*)pred, (const L*)label, n,
                                                                              head, ngroups, C, out);
  else
    ssc_confusion_kernel<false, P, L><<<(unsigned)blocks, kThreads, smem, st>>>((const P*)pred, (const L*)label, n,
                                                                               head, ngroups, C, out);
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

template <typename P>
int dispatch_label(const void* pred, const void* label, int label_dtype, long long n, int C, long long* counts,
                   cudaStream_t st) {
  switch (label_dtype) {
    case OCCD_DTYPE_F32: return launch_confusion<P, float>(pred, label, n, C, counts, st);
    case OCCD_DTYPE_U8: return launch_confusion<P, uint8_t>(pred, label, n, C, counts, st);
    case OCCD_DTYPE_I64: return launch_confusion<P, long long>(pred, label, n, C, counts, st);
    default: occd_set_last_error("occd_ssc_confusion: label dtype must be F32, U8 or I64"); return OCCD_ERR_ARG;
  }
}

}  // namespace

extern "C" int occd_ssc_confusion(const void* pred, int pred_dtype, const void* label, int label_dtype, long long n,
                                  int n_classes, long long* counts, void* stream) {
  OCCD_CHECK_ARG(pred && label && counts && n > 0, "occd_ssc_confusion: args");
  OCCD_CHECK_ARG(n_classes > 0 && n_classes <= kMaxClasses, "occd_ssc_confusion: n_classes must be in [1, 64]");
  OCCD_CHECK_ARG((uintptr_t)counts % sizeof(long long) == 0, "occd_ssc_confusion: counts must be 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  switch (pred_dtype) {
    case OCCD_DTYPE_U16: return dispatch_label<unsigned short>(pred, label, label_dtype, n, n_classes, counts, st);
    case OCCD_DTYPE_I64: return dispatch_label<long long>(pred, label, label_dtype, n, n_classes, counts, st);
    default: occd_set_last_error("occd_ssc_confusion: pred dtype must be U16 or I64"); return OCCD_ERR_ARG;
  }
}
