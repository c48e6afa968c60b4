// CPU emulation harness for the camera-format staging bodies of csrc/normalize_rgb.cuh (occd_stage_camera_u8_cl):
// the device's integer colour conversion and fixed-point remap, then the float32 normalisation with explicit rounding,
// so the host run is the device result.
#include "normalize_rgb.cuh"

extern "C" void occd_set_last_error(const char*) {}

template <int FMT, bool MAPS>
static void run(const nrm::StageArgs& a, long long total, int out_dtype) {
  for (long long i = 0; i < total; ++i) {
    if (out_dtype == 1) nrm::stage_body<__nv_bfloat16, FMT, MAPS>(a, i);
    else nrm::stage_body<float, FMT, MAPS>(a, i);
  }
}

// format: 0 RGB, 1 BGR, 2 NV12 (OCCD_PIX_*); out_dtype 0: float (TF32 values), 1: bf16; maps may be NULL
extern "C" int stage_camera_emulate(const void* in, int format, long long img_stride, long long row_stride,
                                    long long uv_offset, int n, int H0, int W0, int H, int W, const float* maps,
                                    long long map_stride, const float* mean, const float* stdv, void* out,
                                    int out_dtype, int cstride) {
  nrm::StageArgs a;
  a.in = (const unsigned char*)in; a.img_stride = img_stride; a.row_stride = row_stride;
  a.out = out; a.H = H; a.W = W; a.cstride = cstride;
  for (int c = 0; c < 3; ++c) { a.mean[c] = mean[c]; a.stdv[c] = stdv[c]; }
  a.uv_offset = uv_offset; a.H0 = H0; a.W0 = W0; a.maps = maps; a.map_stride = map_stride;
  const long long total = (long long)n * H * W;
  switch (format * 2 + (maps != nullptr)) {
    case 0: run<nrm::PIX_RGB, false>(a, total, out_dtype); break;
    case 1: run<nrm::PIX_RGB, true>(a, total, out_dtype); break;
    case 2: run<nrm::PIX_BGR, false>(a, total, out_dtype); break;
    case 3: run<nrm::PIX_BGR, true>(a, total, out_dtype); break;
    case 4: run<nrm::PIX_NV12, false>(a, total, out_dtype); break;
    case 5: run<nrm::PIX_NV12, true>(a, total, out_dtype); break;
    default: return 1;
  }
  return 0;
}

// the remap weight table the device's __constant__ copy is built from: 1024 cells x 4 taps
extern "C" void remap_table(unsigned short* out) {
  for (int k = 0; k < 1024; ++k)
    for (int t = 0; t < 4; ++t) out[k * 4 + t] = nrm::kRemapTabHost.w[k][t];
}
