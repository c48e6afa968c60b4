// CPU emulation harness for the staging bodies of csrc/normalize_rgb.cuh (occd_stage_rgb_u8_cl, occd_depth_u16_to_f32):
// IEEE float32 / float64 arithmetic with explicit rounding, so the host run is the device result.
#include "normalize_rgb.cuh"

extern "C" void occd_set_last_error(const char*) {}

// out_dtype 0: float (TF32 values), 1: bf16
extern "C" int stage_rgb_emulate(const void* in, long long img_stride, long long row_stride, int n, int H, int W,
                                 const float* mean, const float* stdv, void* out, int out_dtype, int cstride) {
  nrm::StageArgs a;
  a.in = (const unsigned char*)in; a.img_stride = img_stride; a.row_stride = row_stride;
  a.out = out; a.H = H; a.W = W; a.cstride = cstride;
  for (int c = 0; c < 3; ++c) { a.mean[c] = mean[c]; a.stdv[c] = stdv[c]; }
  const long long total = (long long)n * H * W;
  for (long long i = 0; i < total; ++i) {
    if (out_dtype == 1) nrm::stage_body<__nv_bfloat16>(a, i);
    else nrm::stage_body<float>(a, i);
  }
  return 0;
}

extern "C" int depth_emulate(const unsigned short* in, float* out, long long n, double divisor, float max_depth) {
  for (long long i = 0; i < n; ++i) out[i] = nrm::depth_u16(in[i], divisor, max_depth);
  return 0;
}
