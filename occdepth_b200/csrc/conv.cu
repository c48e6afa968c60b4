// Generalised N-d convolution as implicit GEMM.
//   TC path  : TMA (5-D tiled tensor maps, zero-filled halos, traversal strides) -> swizzled smem ->
//              wgmma (M=128 positions, N<=256 channels, fp32 accumulators in registers; two MMA warpgroups on a
//              ping-pong or cooperative schedule, see conv_kernels.cuh) ->
//              epilogue (bias + residuals + activation, channels-last / fp32 planar stores)
//   SIMT path: CUDA-core direct convolution with identical semantics (cross-check and odd shapes)
// The tensor-core kernels live in conv_kernels.cuh; this file plans them (tile shapes, N tile, pipeline depth, tensor
// maps), runs the SIMT path and dispatches a plan to the kernel compiled for its N tile.
// Two operand types share every kernel (template parameter T, see Elem<T> / tc::Mma<T, N>):
//   float (TF32 values, wgmma .tf32, K chunk = 32 / 16 / 8 channels)  -- reference-precision mode
//   __nv_bfloat16 (wgmma .bf16, K chunk = 64 / 32 / 16 channels)      -- throughput mode
// A K chunk is always one swizzled smem row of RB = 128 / 64 / 32 bytes; one wgmma step consumes 32 bytes of it.
// See include/occdepth_b200.h for the reference call sequences this replaces.
#include "conv_kernels.cuh"
#include <new>
#include <utility>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>

namespace {

using namespace occd_conv;

// the 8 accumulator sums of channel group g at one output position (conv_simt_kernel)
template <typename T>
__device__ __forceinline__ void simt_acc8(const SimtParams& p, int b, int od, int oh, int ow, int g, float* acc) {
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  for (int tp = 0; tp < p.n_taps; ++tp) {
    const int s = p.tap_src[tp];
    const int id = od * p.stride[0] + p.tap_dz[tp] + p.src_d0;
    const int ih = oh * p.stride[1] + p.tap_dy[tp];
    const int iw = ow * p.stride[2] + p.tap_dx[tp];
    if (id < 0 || id >= p.ID || ih < 0 || ih >= p.IH || iw < 0 || iw >= p.IW) continue;
    const T* in = reinterpret_cast<const T*>(p.src[s]) +
                  ((((long long)b * p.ID + id) * p.IH + ih) * p.IW + iw) * p.src_cstride[s] + p.src_coff[s];
    const T* w = reinterpret_cast<const T*>(p.weight) +
                 ((long long)b * p.w_batch_rows + (long long)tp * p.Cout_pad + g * 8) * p.Kpad;
    const int C = p.src_C[s];
    for (int c = 0; c < C; c += 8) {
      float x[8];
      Elem<T>::ld8(in + c, x);
      if (c + 8 > C) {
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (c + i >= C) x[i] = 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float wv[8];
        Elem<T>::ld8_nc(w + (long long)j * p.Kpad + c, wv);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[j] = fmaf(x[i], wv[i], acc[j]);
      }
    }
  }
}

// one thread per (output position, group of 8 channels); with a class-map output one thread per position walks every
// channel group, so that one thread holds the position's arg-max; with the probabilities it then walks them again,
// recomputing each group's sums, and stores every channel's probability
template <typename T>
__global__ void __launch_bounds__(128) conv_simt_kernel(const __grid_constant__ SimtParams p) {
  const bool cls = class_mode(p.epi.out1_mode), conf = class_softmax(p.epi.out1_mode);
  const int ngroups = cls ? 1 : p.epi.Cout_store / 8;
  const long long total = (long long)p.epi.B * p.epi.OD * p.epi.OH * p.epi.OW * ngroups;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g0 = (int)(idx % ngroups), g1 = cls ? p.epi.Cout_store / 8 : g0 + 1;
  long long pos = idx / ngroups;
  const int ow = (int)(pos % p.epi.OW); pos /= p.epi.OW;
  const int oh = (int)(pos % p.epi.OH); pos /= p.epi.OH;
  const int od = (int)(pos % p.epi.OD); pos /= p.epi.OD;
  const int b = (int)pos;
  ClassArg ca = class_arg_init();
  for (int g = g0; g < g1; ++g) {
    float acc[8];
    simt_acc8<T>(p, b, od, oh, ow, g, acc);
    if (!cls) {
      conv_epilogue_row<T, 8>(p.epi, b, od, oh, ow, g * 8, acc);
      continue;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (g * 8 + i < p.epi.Cout)
        class_arg_take(ca, class_value<T>(p.epi, epi_pos(p.epi, b, od, oh, ow), g * 8 + i, acc[i]), g * 8 + i, conf);
  }
  if (!cls) return;
  const long long ps = epi_pos(p.epi, b, od, oh, ow);
  class_store(p.epi, ps, ca);
  if (p.epi.out1_mode != OCCD_OUT1_CLASS_U16_PROBS) return;
  for (int g = g0; g < g1; ++g) {
    float acc[8];
    simt_acc8<T>(p, b, od, oh, ow, g, acc);
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (g * 8 + i < p.epi.Cout)
        class_prob_store(p.epi, b, ps, g * 8 + i, class_value<T>(p.epi, ps, g * 8 + i, acc[i]), ca);
  }
}

// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !ptr) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

int round_up(int a, int b) { return (a + b - 1) / b * b; }

// Estimated cycles of one 32-byte K step of a 128 x N tile: one m64nN wgmma in each MMA warpgroup.  Estimates from
// data-sheet figures, not measurements: at 495 TF32 (989 BF16) TFLOP/s and 1.83 GHz an SM does 1024 TF32 (2048
// BF16) FMA per clock, so the step takes N tensor cycles in either precision; the two instructions read
// 2 x (64 rows x 32 B of A + N x 32 B of B) from shared memory at a nominal 128 B per clock, which bounds narrow tiles.
double mma_step_cycles(int n) {
  const double smem = 2.0 * (64 * 32 + n * 32) / 128.0;
  return n > smem ? (double)n : smem;
}

// K chunk (channels) for a source of C channels: the smallest swizzled row (32 / 64 / 128 bytes) that holds it,
// else the 128-byte row
int chunk_channels(int C, int esize) {
  for (int rb = 32; rb <= 128; rb *= 2)
    if (C <= rb / esize) return rb / esize;
  return 128 / esize;
}

}  // namespace

// per-role clock64 tracing of the conv kernels: part of the ABI, not built into the sm_90a kernels.  NULL (tracing
// off) is accepted; a buffer is refused.
extern "C" int occd_conv_debug_trace(long long* device_buf) {
  if (device_buf) {
    occd_set_last_error("occd_conv_debug_trace: per-role tracing is not available in this build");
    return OCCD_ERR_UNSUPPORTED;
  }
  return OCCD_OK;
}

static void fill_epi(const occd_conv_desc* d, ConvEpi* e) {
  e->B = d->B; e->OD = d->OD; e->OH = d->OH; e->OW = d->OW;
  for (int i = 0; i < 3; ++i) { e->omul[i] = d->omul[i]; e->oadd[i] = d->oadd[i]; }
  e->ODf = d->ODf; e->OHf = d->OHf; e->OWf = d->OWf;
  e->Cout = d->Cout;
  e->Cout_store = round_up(d->Cout, 8);
  e->bias = d->bias;
  e->out0 = d->out0;
  e->out0_cstride = d->out0_cstride; e->out0_coff = d->out0_coff;
  e->act = d->act;
  e->out0_exact = d->out0_exact;
  e->res1 = d->res1;
  e->res1_cstride = d->res1_cstride; e->res1_coff = d->res1_coff;
  e->res2 = d->res2;
  e->res2_cstride = d->res2_cstride; e->res2_coff = d->res2_coff; e->res2_post = d->res2_post;
  e->out1_mode = d->out1_mode; e->out1 = d->out1;
  e->out1_cstride = d->out1_cstride; e->out1_coff = d->out1_coff; e->out1_C = d->out1_C;
}

static ConvEpi* plan_epi(occd_conv_plan* pl) {
  switch (pl->impl) {
    case OCCD_CONV_IMPL_SIMT: return &pl->simt.epi;
    case OCCD_CONV_IMPL_HALO: return &pl->halo.epi;
    case OCCD_CONV_IMPL_HALOX: return &pl->halox.epi;
    default: return &pl->tc.epi;
  }
}

static const char* impl_tag(int impl) {
  switch (impl) {
    case OCCD_CONV_IMPL_SIMT: return "simt";
    case OCCD_CONV_IMPL_HALO: return "halo";
    case OCCD_CONV_IMPL_HALOX: return "halox";
    case OCCD_CONV_IMPL_TCX: return "tcx";
    default: return "tc";
  }
}

// plan creation refuses the descriptor: the message names the impl
static int refuse(const occd_conv_plan* pl, int rc, const char* msg) {
  char buf[256];
  snprintf(buf, sizeof(buf), "occd_conv_plan_create(%s): %s", impl_tag(pl->impl), msg);
  occd_set_last_error(buf);
  return rc;
}
// a shape the impl's kernel cannot run
#define PLAN_REQUIRE(cond, msg) do { if (!(cond)) return refuse(pl, OCCD_ERR_UNSUPPORTED, msg); } while (0)

static int n_sms_current() {
  static int n_sms[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (n_sms[dev] == 0) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0) n_sms[dev] = v;
    else n_sms[dev] = 132;
  }
  return n_sms[dev];
}

// Persistent kernels: one CTA per SM, or one per tile when there are fewer tiles
static int persistent_grid(occd_conv_plan* pl, long long num_tiles) {
  PLAN_REQUIRE(num_tiles <= 2147483647LL, "too many tiles");
  const int n_sms = n_sms_current();
  pl->grid = dim3((unsigned)(num_tiles < n_sms ? num_tiles : n_sms));
  return OCCD_OK;
}

// The K chunk (pl->kc channels, pl->rb bytes per swizzled smem row) for sources of at most C channels
static int set_k_chunk(occd_conv_plan* pl, int C) {
  pl->kc = chunk_channels(C, pl->esize);
  pl->rb = pl->kc * pl->esize;
  return pl->kc;
}

// The halo kernels' grid: a stride-1 "same" convolution, output grid = input grid less the source's halo margins
static int same_grid(const occd_conv_desc* d, const occd_conv_plan* pl) {
  PLAN_REQUIRE(d->stride[0] == 1 && d->stride[1] == 1 && d->stride[2] == 1, "stride must be 1");
  PLAN_REQUIRE(d->omul[0] == 1 && d->omul[1] == 1 && d->omul[2] == 1 && d->oadd[0] == 0 && d->oadd[1] == 0 &&
               d->oadd[2] == 0, "identity output mapping only");
  PLAN_REQUIRE(d->OD + 2 * d->src_d0 == d->ID && d->OH == d->IH && d->OW == d->IW,
               "output grid must equal the input grid (plus symmetric halo margins)");
  return OCCD_OK;
}

// Each tensor-core geometry below is pure host arithmetic.  Besides its parameter block it returns the activation
// TMA box and traversal strides in (W, H, D) order and the weight box's rows (the N tile); occd_conv_plan_create
// encodes the tensor maps from them once the geometry has accepted the descriptor.

// The halo kernel's shapes: stride-1 "same" convolution of one source whose taps are {-d,0,d} offsets (*dil = d), one
// k-chunk, one compiled N tile
static int halo_shape(const occd_conv_desc* d, const occd_conv_plan* pl, int* dil) {
  PLAN_REQUIRE(d->n_src == 1, "one source only");
  if (const int rc = same_grid(d, pl)) return rc;
  PLAN_REQUIRE(d->n_taps <= 27, "at most 27 taps");
  PLAN_REQUIRE(d->src_C[0] <= 128 / pl->esize && d->Cout_pad <= 128,
               "channel counts too large for the resident-weight scheme (one K chunk)");
  PLAN_REQUIRE(HaloTiles::has(d->Cout_pad), "no kernel compiled for this Cout_pad (16, 32, 48 or 64)");
  *dil = 0;
  for (int i = 0; i < d->n_taps; ++i) {
    const int o[3] = {abs(d->taps[i].dz), abs(d->taps[i].dy), abs(d->taps[i].dx)};
    for (int k = 0; k < 3; ++k)
      if (o[k]) { if (!*dil) *dil = o[k]; PLAN_REQUIRE(o[k] == *dil, "taps must be {-d,0,d} offsets"); }
  }
  PLAN_REQUIRE(*dil >= 1 && *dil <= 8, "dilation must be 1..8");
  return OCCD_OK;
}

// OCCD_CONV_IMPL_AUTO plans a conv of three or more taps of the halo kernel's shapes on it, and on TC where the tile
// search below refuses it
static bool halo_eligible(const occd_conv_desc* d, const occd_conv_plan* pl) {
  int dil;
  return d->n_taps >= 3 && halo_shape(d, pl, &dil) == OCCD_OK;
}

// Halo-tile plan: a conv of halo_shape, resident weights, a box of at least 50 % useful MMA rows
static int halo_geometry(const occd_conv_desc* d, occd_conv_plan* pl, int box[3], int traversal[3], int* n_tile) {
  int dil;
  if (const int rc = halo_shape(d, pl, &dil)) return rc;
  int hal[3] = {0, 0, 0};
  for (int i = 0; i < d->n_taps; ++i) {
    if (d->taps[i].dz) hal[0] = 1;
    if (d->taps[i].dy) hal[1] = 1;
    if (d->taps[i].dx) hal[2] = 1;
  }
  HaloParams& h = pl->halo;
  PLAN_REQUIRE(d->Kpad == set_k_chunk(pl, d->src_C[0]), "Kpad must equal the k-chunk");
  const int row_bytes = pl->rb;
  h.d = dil; h.D = d->OD; h.H = d->IH; h.W = d->IW;
  h.src_d0 = d->src_d0;
  h.hd = hal[0]; h.hh = hal[1]; h.hw = hal[2];
  h.n_taps = d->n_taps;
  h.N_tile = d->Cout_pad;
  h.b_stride = round_up(h.N_tile * row_bytes, 1024);
  h.w_bytes = h.n_taps * h.b_stride;
  PLAN_REQUIRE(h.w_bytes <= 112 * 1024, "weights do not fit in shared memory");
  const int sD = (d->OD + dil - 1) / dil, sH = (d->IH + dil - 1) / dil, sW = (d->IW + dil - 1) / dil;
  const int smem_total = 227 * 1024 - staging_bytes(kStageHalo) - h.w_bytes - 2048;   // staging, barriers, slack
  // W extent of the box: the whole sub-sampled line when it fits, else equal splits of at most 62
  const int nW = (sW + 61) / 62;
  const int BW = (sW + nW - 1) / nW;
  long long best_cost = -1;
  for (int BD = 1; BD <= (hal[0] ? 4 : 1); ++BD)
    for (int BH = 1; BH <= sH && BH <= 96; ++BH) {
      const int PD = BD + 2 * hal[0], PH = BH + 2 * hal[1], PW = BW + 2 * hal[2];
      if ((PW - 1) * dil + 1 > 256 || (PH - 1) * dil + 1 > 256 || (PD - 1) * dil + 1 > 256) continue;
      const int R0 = (hal[0] * PH + hal[1]) * PW + hal[2];
      const int Rend = ((BD - 1 + hal[0]) * PH + (BH - 1 + hal[1])) * PW + BW - 1 + hal[2];
      const int nM = (Rend - R0 + 1 + 127) / 128;
      if (nM * h.N_tile > 256) continue;
      int rows_alloc = PD * PH * PW;
      if (R0 + nM * 128 + R0 > rows_alloc) rows_alloc = R0 + nM * 128 + R0;
      const int stage = round_up(rows_alloc * row_bytes, 1024);
      if (2 * stage > smem_total) continue;
      if (2 * BD * BH * BW < nM * 128) continue;  // < 50 % useful MMA rows: the per-tap kernel is the better choice
      const long long tiles = (long long)((sD + BD - 1) / BD) * ((sH + BH - 1) / BH) * nW;
      const long long cost = tiles * nM * 1000 + tiles;  // MMA work first, then tile count
      if (best_cost < 0 || cost < best_cost) {
        best_cost = cost;
        h.BD = BD; h.BH = BH; h.BW = BW; h.PD = PD; h.PH = PH; h.PW = PW;
        h.R0 = R0; h.nM = nM; h.a_stage_bytes = stage;
      }
    }
  PLAN_REQUIRE(best_cost >= 0, "no tile shape fits");
  h.tilesD = (sD + h.BD - 1) / h.BD; h.tilesH = (sH + h.BH - 1) / h.BH; h.tilesW = nW;
  h.box_bytes = h.PD * h.PH * h.PW * row_bytes;
  h.stages = smem_total / h.a_stage_bytes;
  if (h.stages > 4) h.stages = 4;
  h.rb = row_bytes;
  for (int i = 0; i < d->n_taps; ++i)
    h.tap_off16[i] = (h.R0 + ((d->taps[i].dz / dil) * h.PH + d->taps[i].dy / dil) * h.PW + d->taps[i].dx / dil) *
                     row_bytes / 16;
  h.pdl = occd_pdl_enabled();
  pl->smem = (size_t)h.w_bytes + (size_t)h.stages * h.a_stage_bytes + staging_bytes(kStageHalo) + 128 + 1024;
  box[0] = (h.PW - 1) * dil + 1; box[1] = (h.PH - 1) * dil + 1; box[2] = (h.PD - 1) * dil + 1;
  traversal[0] = traversal[1] = traversal[2] = dil;
  *n_tile = h.N_tile;
  return persistent_grid(pl, (long long)d->B * dil * dil * dil * h.tilesD * h.tilesH * h.tilesW);
}

// x-packed halo plan (conv_halox_kernel)
static int halox_geometry(const occd_conv_desc* d, occd_conv_plan* pl, int box[3], int traversal[3], int* n_tile) {
  PLAN_REQUIRE(d->n_src == 1 && !d->weight_per_image, "one source, shared weights");
  if (const int rc = same_grid(d, pl)) return rc;
  PLAN_REQUIRE(d->IW == 8 || d->IW == 16 || d->IW == 32, "innermost extent W must be 8, 16 or 32 (one warp row)");
  PLAN_REQUIRE(d->n_taps % 3 == 0 && d->n_taps <= 27, "taps must come as W triples");
  PLAN_REQUIRE(d->src_C[0] <= 128 / pl->esize && 3 * d->Cout_pad <= 256, "one K chunk, 3 * Cout_pad <= 256");
  const int dil = d->taps[2].dx;
  PLAN_REQUIRE(dil >= 1 && dil <= 8 && dil < d->IW, "W dilation");
  int hal[2] = {0, 0};
  for (int i = 0; i < d->n_taps; i += 3) {
    const occd_conv_tap &a = d->taps[i], &b = d->taps[i + 1], &c = d->taps[i + 2];
    PLAN_REQUIRE(a.dx == -dil && b.dx == 0 && c.dx == dil && a.dz == b.dz && a.dz == c.dz && a.dy == b.dy &&
                 a.dy == c.dy, "taps must be ordered (dz, dy) groups of dx = -d, 0, +d");
    PLAN_REQUIRE((a.dz == 0 || abs(a.dz) == dil) && (a.dy == 0 || abs(a.dy) == dil), "D / H taps must be {-d, 0, d}");
    if (a.dz) hal[0] = 1;
    if (a.dy) hal[1] = 1;
  }
  HaloxParams& h = pl->halox;
  PLAN_REQUIRE(d->Kpad == set_k_chunk(pl, d->src_C[0]), "Kpad must equal the k-chunk");
  const int RB = pl->rb, NMMA = RB / 32;
  h.d = dil; h.D = d->OD; h.H = d->IH;
  h.src_d0 = d->src_d0;
  h.hd = hal[0]; h.hh = hal[1];
  h.n_groups = d->n_taps / 3;
  h.CP = d->Cout_pad;
  h.N_tile = 3 * d->Cout_pad;
  PLAN_REQUIRE(HaloxTiles::has(h.N_tile), "no kernel compiled for this Cout_pad (16, 32, 48, 64 or 80)");
  h.rb = RB;
  h.PW = d->IW;
  h.b_stride = round_up(h.N_tile * RB, 1024);
  h.w_bytes = h.n_groups * h.b_stride;
  const int smem_total = 227 * 1024 - xp_xchg_bytes(dil) - h.w_bytes - 2048;   // neighbour exchange, barriers, slack
  PLAN_REQUIRE(smem_total > 0, "weights do not fit in shared memory");
  const int HR = 128 / h.PW;                               // h-rows of one plane per M tile
  const int sD = (d->OD + dil - 1) / dil, sH = (d->IH + dil - 1) / dil;
  // CTA tile = BD planes x nB blocks of HR h-rows (<= 2 M tiles: two accumulator sets of nM x N_tile columns)
  double best = -1.0;
  const int cand[3][2] = {{1, 1}, {1, 2}, {2, 1}};
  for (int ci = 0; ci < 3; ++ci) {
    const int BD = cand[ci][0], nB = cand[ci][1];
    const int BH = nB * HR, PD = BD + 2 * hal[0], PH = BH + 2 * hal[1];
    if ((PH - 1) * dil + 1 > 256 || (PD - 1) * dil + 1 > 256) continue;
    const int rows = PD * PH * h.PW;
    const int stage = round_up(rows * RB, 1024);
    if (stage > smem_total) continue;
    const int stages = smem_total / stage;
    const int nM = BD * nB;
    // cycles per useful output: the MMA steps (mma_step_cycles) plus, single-buffered, the un-overlapped
    // L2 -> smem fill at the chip's ~42 B/cycle/SM (an estimate)
    const double eff_d = (double)(sD < BD ? sD : BD) / BD, eff_h = (double)(sH < BH ? sH : BH) / BH;
    const double mma = (double)nM * h.n_groups * NMMA * mma_step_cycles(h.N_tile);
    const double fill = stages >= 2 ? 0.0 : (double)rows * RB / 42.0;
    // (tie-break: the tile that reloads the fewest halo rows per output)
    const double cost = (mma + fill + 1e-3 * rows * RB) / (BD * BH * h.PW * eff_d * eff_h);
    if (best < 0 || cost < best) {
      best = cost;
      h.BD = BD; h.BH = BH; h.PD = PD; h.PH = PH; h.nM = nM;
      h.a_stage_bytes = stage; h.stages = stages > 4 ? 4 : stages;
    }
  }
  PLAN_REQUIRE(best >= 0, "no tile shape fits");
  h.ring = 0;
  {
    // plane ring instead of a single-stage box (see HaloxParams): needs D taps and four single-plane stages
    const int PHr = HR + 2 * hal[1];
    const int plane = round_up(PHr * h.PW * RB, 1024);
    if (h.stages < 2 && hal[0] == 1 && 4 * plane <= smem_total && (PHr - 1) * dil + 1 <= 256) {
      h.ring = 1;
      h.BD = 1; h.BH = HR; h.PD = 3; h.PH = PHr; h.nM = 1;
      h.a_stage_bytes = plane; h.stages = 4;
    }
  }
  {
    const int nB = h.BH / HR;
    int m = 0;
    for (int pd = 0; pd < h.BD; ++pd)
      for (int blk = 0; blk < nB; ++blk, ++m) {
        h.mt_pd[m] = pd + h.hd;
        h.mt_ph0[m] = h.hh + blk * HR;
        h.mt_row[m] = (h.mt_pd[m] * h.PH + h.mt_ph0[m]) * h.PW;
      }
  }
  h.tilesD = (sD + h.BD - 1) / h.BD; h.tilesH = (sH + h.BH - 1) / h.BH;
  h.box_bytes = (h.ring ? 1 : h.PD) * h.PH * h.PW * RB;
  for (int g = 0; g < h.n_groups; ++g) {
    h.grp_off[g] = ((d->taps[3 * g].dz / dil) * h.PH + d->taps[3 * g].dy / dil) * h.PW;
    h.grp_dz[g] = (signed char)(d->taps[3 * g].dz / dil);
    h.grp_row[g] = (short)((h.hh + d->taps[3 * g].dy / dil) * h.PW);
  }
  h.sD = sD;
  h.n_cols = d->B * dil * dil * h.tilesH;
  h.pdl = occd_pdl_enabled();
  pl->smem = (size_t)h.w_bytes + (size_t)h.stages * h.a_stage_bytes + xp_xchg_bytes(dil) + 128 + 1024;
  box[0] = h.PW; box[1] = (h.PH - 1) * dil + 1; box[2] = h.ring ? 1 : (h.PD - 1) * dil + 1;   // ring: one plane per load
  traversal[0] = 1; traversal[1] = traversal[2] = dil;
  *n_tile = h.N_tile;
  const long long num_tiles = h.ring ? (long long)h.n_cols * sD      // ring mode: M tiles; each CTA takes a contiguous share
                                     : (long long)d->B * dil * dil * h.tilesD * h.tilesH;
  if (const int rc = persistent_grid(pl, num_tiles)) return rc;
  h.pp = ping_pong(h.N_tile, h.ring ? num_tiles : num_tiles * h.nM, pl->grid.x);   // M tiles per CTA
  return OCCD_OK;
}

// Per-tap (TC) plan.  xp: x-packed variant (TCX)
static int tc_geometry(const occd_conv_desc* d, occd_conv_plan* pl, bool xp, int box[3], int traversal[3],
                       int* n_tile) {
  int maxC = 0;
  for (int s = 0; s < d->n_src; ++s) maxC = d->src_C[s] > maxC ? d->src_C[s] : maxC;
  TcParams& t = pl->tc;
  const int KC = set_k_chunk(pl, maxC), RB = pl->rb;
  if (d->Kpad % KC != 0) return refuse(pl, OCCD_ERR_ARG, "Kpad must be a multiple of the K chunk");
  t.n_taps = xp ? d->n_taps / 3 : d->n_taps;  // x-packed: one pipeline item per (source, dz, dy) group
  const int n_groups = d->n_groups > 1 ? d->n_groups : 1;
  if (n_groups > 1) {
    bool ok = !xp && n_groups <= OCCD_CONV_MAX_GROUPS && d->group_tap0[0] == 0 && d->group_tap0[n_groups] == d->n_taps &&
              d->out1_mode == OCCD_OUT1_NONE && d->out0 != nullptr &&
              (d->res2 == nullptr || (d->res2_post && d->res1 == nullptr));
    for (int g = 0; ok && g < n_groups; ++g) {
      ok = d->group_tap0[g + 1] > d->group_tap0[g];
      for (int i = 0; i < 3; ++i) ok = ok && d->group_oadd[g][i] >= 0 && d->group_oadd[g][i] < d->omul[i];
    }
    PLAN_REQUIRE(ok, "tap groups need the per-tap TC kernel, ascending non-empty tap ranges covering all taps, "
                     "0 <= group_oadd < omul, no second output and at most one residual");
  }
  t.n_groups = n_groups;
  t.src_d0 = d->src_d0;
  t.w_batch_rows = d->weight_per_image ? d->n_taps * d->Cout_pad : 0;
  for (int s = 0; s < OCCD_CONV_MAX_SRC; ++s) t.n_kchunks[s] = s < d->n_src ? (d->src_C[s] + KC - 1) / KC : 0;
  for (int i = 0; i < 3; ++i) t.stride[i] = d->stride[i];
  for (int g = 0; g < n_groups; ++g) {
    t.grp_tap0[g] = (short)(n_groups > 1 ? d->group_tap0[g] : 0);
    t.grp_tap0[g + 1] = (short)(n_groups > 1 ? d->group_tap0[g + 1] : t.n_taps);
    for (int i = 0; i < 3; ++i) t.grp_oadd[g][i] = (signed char)(n_groups > 1 ? d->group_oadd[g][i] : 0);
  }
  if (xp) {
    // groups of three W taps -1, 0, +1 share one MMA with N = 3 * Cout_pad; the tile is 32 positions wide (30
    // outputs + one halo column each side) so that lane == column in the epilogue
    PLAN_REQUIRE(d->n_taps % 3 == 0 && d->stride[2] == 1 && 3 * d->Cout_pad <= 256,
                 "needs W-tap triples, W stride 1 and 3 * Cout_pad <= 256");
    for (int i = 0; i < d->n_taps; i += 3) {
      const occd_conv_tap &a = d->taps[i], &b = d->taps[i + 1], &c = d->taps[i + 2];
      PLAN_REQUIRE(a.dx == -1 && b.dx == 0 && c.dx == 1 && a.src == b.src && a.src == c.src && a.dz == b.dz &&
                   a.dz == c.dz && a.dy == b.dy && a.dy == c.dy,
                   "taps must be ordered (src, dz, dy) groups of dx = -1, 0, +1");
      t.tap_src[i / 3] = (signed char)b.src;
      t.tap_dz[i / 3] = (short)b.dz; t.tap_dy[i / 3] = (short)b.dy; t.tap_dx[i / 3] = 0;
    }
    t.TW = 32;
    long long best = -1;
    for (int th = 4; th >= 1; th >>= 1) {
      const int tdd = 4 / th;
      const long long vol = (long long)round_up(d->OH, th) * round_up(d->OD, tdd);
      if (best < 0 || vol < best) { best = vol; t.TH = th; t.TD = tdd; }
    }
  } else {
    for (int i = 0; i < d->n_taps; ++i) {
      t.tap_src[i] = (signed char)d->taps[i].src;
      t.tap_dz[i] = (short)d->taps[i].dz; t.tap_dy[i] = (short)d->taps[i].dy; t.tap_dx[i] = (short)d->taps[i].dx;
    }
    // tile box (TD,TH,TW), product 128: minimal padded volume, but a wide innermost extent (long contiguous TMA
    // runs, coalesced stores) wins whenever it costs < 4% extra positions
    long long best = -1;
    for (int pass = 0; pass < 2; ++pass)
      for (int tw = 128; tw >= 1; tw >>= 1)
        for (int th = 128 / tw; th >= 1; th >>= 1) {
          const int tdd = 128 / (tw * th);
          if (tw * d->stride[2] > 256 || th * d->stride[1] > 256 || tdd * d->stride[0] > 256) continue;
          const long long vol = (long long)round_up(d->OW, tw) * round_up(d->OH, th) * round_up(d->OD, tdd);
          if (pass == 0) {
            if (best < 0 || vol < best) best = vol;
          } else if (vol * 100 <= best * 104) {
            t.TW = tw; t.TH = th; t.TD = tdd;
            pass = 2; tw = 0; break;  // first hit in (widest TW, tallest TH) order
          }
        }
  }
  t.TWv = xp ? 30 : t.TW;
  t.tiles_w = (d->OW + t.TWv - 1) / t.TWv; t.tiles_h = (d->OH + t.TH - 1) / t.TH; t.tiles_d = (d->OD + t.TD - 1) / t.TD;
  // N tile: the divisor of Cout_pad (multiple of 16, <= 256) with the smallest estimated makespan.  The model's
  // constants are estimates, not measurements: an M = 128 MMA step costs mma_step_cycles(N), an SM pulls ~44
  // bytes/cycle from L2 when the whole chip does, the epilogue drains ~12 bytes/cycle/SM, and a CTA's time is
  // waves * max(mainloop, epilogue) + min(mainloop, epilogue): the ping-pong schedule's overlap (N <= 128, see
  // kTcThreads).  For the cooperative widths above 128 that overlap does not happen and the estimate is optimistic;
  // it is kept because the wide tiles it picks for the large decoder convs measure near the tensor-core rate.
  // Small-M layers (late encoder stages: 9 M tiles) get narrow N tiles that spread the write-bound epilogue over
  // every SM; large-M layers get the widest tile (fewest re-reads of the A operand).
  t.Cout_pad = d->Cout_pad;
  double est_mainloop = 0.0, est_epi = 0.0;   // the final N tile's estimates, for the schedule choice below
  if (xp) t.N_tile = 3 * d->Cout_pad;  // one N tile: the three taps' weights stacked
  {
    int iters = 0;
    for (int i = 0; i < t.n_taps; ++i) iters += t.n_kchunks[t.tap_src[i]];
    iters = (iters + n_groups - 1) / n_groups;   // tap groups: the mean group; every CTA gets its share of each
    const long long m_tiles0 = (long long)d->B * t.tiles_d * t.tiles_h * t.tiles_w * n_groups;
    const int n_sms = n_sms_current();
    // (a class map, with or without its confidence or probabilities, is costed as the planar logits it stands in
    // for: every plan of one descriptor gets the same tiles, so the map equals the arg-max of the logits bit for bit)
    const double out_bytes_per_col = 128.0 * ((d->out0 ? pl->esize : 0) + (d->out1_mode == OCCD_OUT1_CL ? pl->esize : 0) +
                                              (d->out1_mode == OCCD_OUT1_F32_PLANAR || class_mode(d->out1_mode) ? 4 : 0));
    // per-tile mainloop and epilogue of an n-column tile that stores out_cols channels
    auto estimate = [&](int n, int out_cols, double& mainloop, double& epi) {
      const double mma = (RB / 32) * mma_step_cycles(n);
      const double load = (128.0 + n) * RB / 44.0;
      mainloop = iters * (mma > load ? mma : load);
      epi = out_bytes_per_col * out_cols / 12.0;
    };
    double best = -1.0;
    for (int n = 16; !xp && n <= 256 && n <= d->Cout_pad; n += 16) {
      if (d->Cout_pad % n) continue;
      double mainloop, epi;
      estimate(n, n, mainloop, epi);
      const long long tiles = m_tiles0 * (d->Cout_pad / n);
      const double waves = (double)((tiles + n_sms - 1) / n_sms);
      const double span = waves * (mainloop > epi ? mainloop : epi) + (mainloop > epi ? epi : mainloop);
      if (best < 0 || span <= best * 1.02) {   // within 2 %: the wider tile (fewer tiles, fewer A re-reads) wins
        if (best < 0 || span < best) best = span;
        t.N_tile = n;
      }
    }
    estimate(t.N_tile, xp ? d->Cout_pad : t.N_tile, est_mainloop, est_epi);
  }
  PLAN_REQUIRE(!class_mode(d->out1_mode) || xp || t.N_tile >= d->Cout_pad,
               "a class map needs every output channel in one N tile");
  PLAN_REQUIRE(d->out1_mode != OCCD_OUT1_CLASS_U16_PROBS || xp || t.N_tile <= kProbsMaxN,
               "class probabilities need an N tile of at most 96 channels");
  PLAN_REQUIRE(xp ? TcxTiles::has(t.N_tile) : TcTiles::has(t.N_tile),
               xp ? "no kernel compiled for this Cout_pad (16, 32, 48, 64 or 80)" : "no kernel compiled for this N tile");
  t.rb = RB;
  // programmatic dependent launch (common.cuh): the conv kernels wait on griddepcontrol after their prologue (barrier
  // init, tensor-map prefetch overlap the tail of the previous grid); results are bit-identical either way
  t.pdl = occd_pdl_enabled();
  t.a_bytes = 128 * RB;
  t.b_bytes = t.N_tile * RB;
  t.b_stride = round_up(t.b_bytes, 1024);
  const int stage_bytes = t.a_bytes + t.b_stride;
  int total_iters = 0;   // (tap, k-chunk) items of one tile; with tap groups: of the largest group
  for (int g = 0; g < n_groups; ++g) {
    int it = 0;
    for (int i = t.grp_tap0[g]; i < t.grp_tap0[g + 1]; ++i) it += t.n_kchunks[t.tap_src[i]];
    t.grp_iters[g] = (short)it;
    if (it > total_iters) total_iters = it;
  }
  // persistent kernel: one CTA per SM owns the shared memory (227 KB less the epilogue staging and barriers)
  const int st_bytes = xp ? xp_xchg_bytes(1) : staging_bytes(kStageWide);
  const int budget = 227 * 1024 - st_bytes - 16 * kMaxStages - 64 - 1024;
  // (tap, k-chunk) items per pipeline stage: the single-thread producer/MMA hand-off costs ~0.25 us, so a stage
  // must carry >= ~512 tensor-pipe cycles of work (or up to 9 items) while leaving >= 3 stages in flight
  const int mma_cycles_per_item = (int)((RB / 32) * mma_step_cycles(t.N_tile));
  int group = (512 + mma_cycles_per_item - 1) / mma_cycles_per_item;
  if (group > 9) group = 9;
  if (group > total_iters) group = total_iters;
  while (group > 1 && 3 * group * stage_bytes > budget) --group;
  t.group = group;
  int stages = budget / (group * stage_bytes);
  if (stages > kMaxStages) stages = kMaxStages;
  const int groups_per_tile = (total_iters + group - 1) / group;
  {
    // ring depth: two tiles' worth of stage groups, but never fewer than 8 stages when they fit (a conv with one
    // item per tile otherwise keeps only two TMA loads in flight)
    int cap = 2 * groups_per_tile;
    if (cap < 8) cap = 8;
    if (stages > cap) stages = cap;
  }
  if (stages < 1) stages = 1;
  t.stages = stages;
  pl->smem = (size_t)stages * group * stage_bytes + st_bytes + 16 * kMaxStages + 64 + 1024;  // + staging, barriers, alignment slack
  const long long m_tiles = (long long)d->B * t.tiles_d * t.tiles_h * t.tiles_w;
  const long long all_tiles = m_tiles * (xp ? 1 : d->Cout_pad / t.N_tile) * n_groups;
  if (const int rc = persistent_grid(pl, all_tiles)) return rc;
  t.num_m_tiles = (int)m_tiles;
  // ping-pong hides a tile's epilogue under the next tile's mainloop, but one warpgroup then stores a whole tile
  // alone: a launch whose epilogue outweighs its mainloop (1x1 convs over few channels, store-bound) keeps both
  // warpgroups storing at once
  t.pp = ping_pong(t.N_tile, all_tiles, pl->grid.x) && est_mainloop >= est_epi;
  box[0] = t.TW * d->stride[2]; box[1] = t.TH * d->stride[1]; box[2] = t.TD * d->stride[0];
  traversal[0] = d->stride[2]; traversal[1] = d->stride[1]; traversal[2] = d->stride[0];
  *n_tile = t.N_tile;
  return OCCD_OK;
}

// SIMT plan: one thread per output position and group of 8 channels (per position with a class map)
static int simt_geometry(const occd_conv_desc* d, occd_conv_plan* pl) {
  SimtParams& s = pl->simt;
  s.n_src = d->n_src; s.n_taps = d->n_taps;
  for (int i = 0; i < d->n_src; ++i) {
    s.src[i] = d->src[i];
    s.src_C[i] = d->src_C[i]; s.src_cstride[i] = d->src_cstride[i]; s.src_coff[i] = d->src_coff[i];
  }
  s.ID = d->ID; s.IH = d->IH; s.IW = d->IW; s.src_d0 = d->src_d0;
  for (int i = 0; i < 3; ++i) s.stride[i] = d->stride[i];
  s.weight = d->weight;
  s.Cout_pad = d->Cout_pad; s.Kpad = d->Kpad;
  s.w_batch_rows = d->weight_per_image ? d->n_taps * d->Cout_pad : 0;
  for (int i = 0; i < d->n_taps; ++i) {
    s.tap_src[i] = (signed char)d->taps[i].src;
    s.tap_dz[i] = (short)d->taps[i].dz; s.tap_dy[i] = (short)d->taps[i].dy; s.tap_dx[i] = (short)d->taps[i].dx;
  }
  const long long total = (long long)d->B * d->OD * d->OH * d->OW *
                          (class_mode(d->out1_mode) ? 1 : s.epi.Cout_store / 8);
  pl->grid = dim3((unsigned)((total + 127) / 128));
  return OCCD_OK;
}

// A fresh plan on kernel `impl`, laid out by that kernel's geometry
static int plan_geometry(const occd_conv_desc* d, occd_conv_plan* pl, int impl, int box[3], int traversal[3],
                         int* n_tile) {
  const int dtype = pl->dtype, esize = pl->esize;
  memset(pl, 0, sizeof(*pl));
  pl->impl = impl;
  pl->dtype = dtype;
  pl->esize = esize;
  fill_epi(d, plan_epi(pl));
  return impl == OCCD_CONV_IMPL_SIMT    ? simt_geometry(d, pl)
         : impl == OCCD_CONV_IMPL_HALO  ? halo_geometry(d, pl, box, traversal, n_tile)
         : impl == OCCD_CONV_IMPL_HALOX ? halox_geometry(d, pl, box, traversal, n_tile)
                                        : tc_geometry(d, pl, impl == OCCD_CONV_IMPL_TCX, box, traversal, n_tile);
}

// OCCD_CONV_IMPL_AUTO: the kernels to try, in order; the plan runs on the first whose geometry accepts the descriptor.
// HALOX first: its geometry's checks are its whole rule.  Then HALO where halo_eligible holds, else TCX for 48 or more
// output channels (narrower ones run best on the halo kernels; the TCX geometry checks the rest).  TC last.  Tap groups
// and per-image weights run on TC only.
static int auto_candidates(const occd_conv_desc* d, occd_conv_plan* pl, int impls[3]) {
  int n = 0;
  if (d->n_groups <= 1 && !d->weight_per_image) {
    impls[n++] = OCCD_CONV_IMPL_HALOX;
    pl->impl = OCCD_CONV_IMPL_HALO;   // (names the kernel in halo_eligible's refusals)
    if (halo_eligible(d, pl)) impls[n++] = OCCD_CONV_IMPL_HALO;
    else if (d->Cout_pad >= 48) impls[n++] = OCCD_CONV_IMPL_TCX;
  }
  impls[n++] = OCCD_CONV_IMPL_TC;
  return n;
}

// One tensor map of the plan's element type, swizzled to its K-chunk row; src: the source it maps, -1 for the weights
static int encode_map(occd_conv_plan* pl, CUtensorMap* tm, int rank, const void* base, const cuuint64_t* gdim,
                      const cuuint64_t* gstr, const cuuint32_t* box, const cuuint32_t* estr, int src) {
  const EncodeTiledFn enc = get_encode_fn();
  if (!enc) return refuse(pl, OCCD_ERR_CUDA, "cuTensorMapEncodeTiled unavailable (no CUDA driver / GPU?)");
  const CUresult r = enc(tm, pl->dtype == OCCD_DTYPE_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16,
                         rank, const_cast<void*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         pl->rb == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                       : (pl->rb == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B),
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_SUCCESS) return OCCD_OK;
  char msg[160];
  if (src < 0) snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled(weights) failed with %d", (int)r);
  else snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled(source %d) failed with %d", src, (int)r);
  return refuse(pl, OCCD_ERR_CUDA, msg);
}

// Source s, channels-last [B][ID][IH][IW] rows of src_cstride elements, channel window [src_coff, +src_C): one K
// chunk by the box (W, H, D), taken at the traversal strides
static int encode_activation(occd_conv_plan* pl, const occd_conv_desc* d, int s, const int box[3],
                             const int traversal[3]) {
  const cuuint64_t cs = (cuuint64_t)d->src_cstride[s] * pl->esize;
  const cuuint64_t gdim[5] = {(cuuint64_t)d->src_C[s], (cuuint64_t)d->IW, (cuuint64_t)d->IH, (cuuint64_t)d->ID,
                              (cuuint64_t)d->B};
  const cuuint64_t gstr[4] = {cs, cs * d->IW, cs * d->IW * d->IH, cs * d->IW * d->IH * d->ID};
  const cuuint32_t bx[5] = {(cuuint32_t)pl->kc, (cuuint32_t)box[0], (cuuint32_t)box[1], (cuuint32_t)box[2], 1};
  const cuuint32_t estr[5] = {1, (cuuint32_t)traversal[0], (cuuint32_t)traversal[1], (cuuint32_t)traversal[2], 1};
  return encode_map(pl, &pl->tmA[s], 5, (const char*)d->src[s] + (size_t)d->src_coff[s] * pl->esize, gdim, gstr, bx,
                    estr, s);
}

// The weights, [rows][Kpad]: one K chunk by box_rows (the N tile)
static int encode_weights(occd_conv_plan* pl, const occd_conv_desc* d, long long rows, int box_rows) {
  const cuuint64_t gdim[2] = {(cuuint64_t)d->Kpad, (cuuint64_t)rows};
  const cuuint64_t gstr[1] = {(cuuint64_t)d->Kpad * pl->esize};
  const cuuint32_t box[2] = {(cuuint32_t)pl->kc, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return encode_map(pl, &pl->tmW, 2, d->weight, gdim, gstr, box, estr, -1);
}

extern "C" int occd_conv_plan_create(const occd_conv_desc* d, occd_conv_plan** out) {
  OCCD_CHECK_ARG(d && out, "occd_conv_plan_create: null argument");
  OCCD_CHECK_ARG(d->dtype == OCCD_DTYPE_F32 || d->dtype == OCCD_DTYPE_BF16, "occd_conv_plan_create: dtype");
  OCCD_CHECK_ARG(d->n_src >= 1 && d->n_src <= OCCD_CONV_MAX_SRC, "occd_conv_plan_create: n_src");
  OCCD_CHECK_ARG(d->n_taps >= 1 && d->n_taps <= OCCD_CONV_MAX_TAPS, "occd_conv_plan_create: n_taps");
  OCCD_CHECK_ARG(d->src_d0 >= 0 && d->src_d0 < d->ID, "occd_conv_plan_create: src_d0");
  OCCD_CHECK_ARG(d->B > 0 && d->ID > 0 && d->IH > 0 && d->IW > 0 && d->OD > 0 && d->OH > 0 && d->OW > 0,
                 "occd_conv_plan_create: dims");
  OCCD_CHECK_ARG(d->Cout > 0 && d->Cout_pad >= d->Cout && d->Cout_pad % 16 == 0, "occd_conv_plan_create: Cout_pad");
  OCCD_CHECK_ARG(d->Kpad > 0 && d->Kpad % 8 == 0, "occd_conv_plan_create: Kpad must be a multiple of 8");
  OCCD_CHECK_ARG(d->weight && d->bias, "occd_conv_plan_create: weight/bias");
  OCCD_CHECK_ARG(d->out0 || d->out1_mode != OCCD_OUT1_NONE, "occd_conv_plan_create: no output");
  const int es = d->dtype == OCCD_DTYPE_F32 ? 4 : 2;
  auto aligned = [es](const void* p) { return (reinterpret_cast<uintptr_t>(p) % (8 * es)) == 0; };
  const int cst = round_up(d->Cout, 8);
  if (d->out0) OCCD_CHECK_ARG(d->out0_coff % 8 == 0 && d->out0_cstride % 8 == 0 && d->out0_coff + cst <= d->out0_cstride &&
                              aligned(d->out0), "occd_conv_plan_create: out0 channel window");
  if (d->res1) OCCD_CHECK_ARG(d->res1_coff % 8 == 0 && d->res1_cstride % 8 == 0 && d->res1_coff + cst <= d->res1_cstride &&
                              aligned(d->res1), "occd_conv_plan_create: res1 channel window");
  if (d->res2) OCCD_CHECK_ARG(d->res2_coff % 8 == 0 && d->res2_cstride % 8 == 0 && d->res2_coff + cst <= d->res2_cstride &&
                              aligned(d->res2), "occd_conv_plan_create: res2 channel window");
  if (d->out1_mode == OCCD_OUT1_CL)
    OCCD_CHECK_ARG(d->out1 && d->out1_coff % 8 == 0 && d->out1_cstride % 8 == 0 && d->out1_coff + cst <= d->out1_cstride &&
                   aligned(d->out1), "occd_conv_plan_create: out1 channel window");
  if (d->out1_mode == OCCD_OUT1_F32_PLANAR)
    OCCD_CHECK_ARG(d->out1 && d->out1_coff + d->Cout <= d->out1_C, "occd_conv_plan_create: out1 planar window");
  if (class_mode(d->out1_mode)) {
    OCCD_CHECK_ARG(d->out1 && reinterpret_cast<uintptr_t>(d->out1) % 2 == 0 && d->Cout <= 65535,
                   "occd_conv_plan_create: a class map needs an aligned uint16 out1 and at most 65535 classes");
    if (d->out0) {
      occd_set_last_error("occd_conv_plan_create: a class map is the launch's only output (out0 must be NULL)");
      return OCCD_ERR_UNSUPPORTED;
    }
  }
  for (int i = 0; i < 3; ++i) {
    OCCD_CHECK_ARG(d->stride[i] >= 1 && d->stride[i] <= 8 && d->omul[i] >= 1, "occd_conv_plan_create: stride/omul");
  }
  OCCD_CHECK_ARG((long long)(d->OD - 1) * d->omul[0] + d->oadd[0] < d->ODf &&
                 (long long)(d->OH - 1) * d->omul[1] + d->oadd[1] < d->OHf &&
                 (long long)(d->OW - 1) * d->omul[2] + d->oadd[2] < d->OWf, "occd_conv_plan_create: output mapping");
  for (int s = 0; s < d->n_src; ++s) {
    OCCD_CHECK_ARG(d->src[s] && d->src_C[s] > 0 && d->src_cstride[s] % 8 == 0 && d->src_coff[s] % 8 == 0 &&
                   d->src_coff[s] + d->src_C[s] <= d->src_cstride[s] && aligned(d->src[s]),
                   "occd_conv_plan_create: source channel window");
    OCCD_CHECK_ARG(d->src_C[s] <= d->Kpad, "occd_conv_plan_create: Kpad smaller than a source");
  }
  for (int i = 0; i < d->n_taps; ++i) {
    OCCD_CHECK_ARG(d->taps[i].src >= 0 && d->taps[i].src < d->n_src, "occd_conv_plan_create: tap source");
    OCCD_CHECK_ARG(abs(d->taps[i].dz) < 30000 && abs(d->taps[i].dy) < 30000 && abs(d->taps[i].dx) < 30000,
                   "occd_conv_plan_create: tap offset");
  }
  OCCD_CHECK_ARG(d->impl == OCCD_CONV_IMPL_TC || d->impl == OCCD_CONV_IMPL_SIMT || d->impl == OCCD_CONV_IMPL_HALO ||
                 d->impl == OCCD_CONV_IMPL_TCX || d->impl == OCCD_CONV_IMPL_HALOX || d->impl == OCCD_CONV_IMPL_AUTO,
                 "occd_conv_plan_create: impl");
  OCCD_CHECK_ARG(d->n_groups <= 1 || d->impl == OCCD_CONV_IMPL_TC || d->impl == OCCD_CONV_IMPL_AUTO,
                 "occd_conv_plan_create: tap groups: TC impl only");
  OCCD_CHECK_ARG(!d->weight_per_image || (d->impl != OCCD_CONV_IMPL_HALO && d->impl != OCCD_CONV_IMPL_HALOX),
                 "occd_conv_plan_create: per-image weights: TC or SIMT impl");

  occd_conv_plan* pl = new (std::nothrow) occd_conv_plan;
  OCCD_CHECK_ARG(pl != nullptr, "occd_conv_plan_create: out of memory");
  memset(pl, 0, sizeof(*pl));
  pl->dtype = d->dtype;
  pl->esize = es;

  int impls[3] = {d->impl};
  const int n_impls = d->impl == OCCD_CONV_IMPL_AUTO ? auto_candidates(d, pl, impls) : 1;
  int box[3], traversal[3], n_tile;   // the tensor-core geometries' TMA boxes
  int rc = OCCD_OK;
  for (int i = 0; i < n_impls; ++i)   // when every candidate refuses, the last (TC) refusal is returned
    if ((rc = plan_geometry(d, pl, impls[i], box, traversal, &n_tile)) == OCCD_OK) break;
  if (rc == OCCD_OK && pl->impl != OCCD_CONV_IMPL_SIMT) {
    for (int s = 0; rc == OCCD_OK && s < d->n_src; ++s) rc = encode_activation(pl, d, s, box, traversal);
    for (int s = d->n_src; s < OCCD_CONV_MAX_SRC; ++s) pl->tmA[s] = pl->tmA[0];
    const long long w_rows = (long long)d->n_taps * d->Cout_pad * (d->weight_per_image ? d->B : 1);
    if (rc == OCCD_OK) rc = encode_weights(pl, d, w_rows, n_tile);
  }
  if (rc != OCCD_OK) { delete pl; return rc; }
  *out = pl;
  return OCCD_OK;
}

extern "C" int occd_conv_plan_destroy(occd_conv_plan* plan) {
  delete plan;
  return OCCD_OK;
}

extern "C" int occd_conv_plan_set_class_lut(occd_conv_plan* pl, const int* lut, int n) {
  OCCD_CHECK_ARG(pl != nullptr, "occd_conv_plan_set_class_lut: null plan");
  ConvEpi* e = plan_epi(pl);
  OCCD_CHECK_ARG(class_mode(e->out1_mode), "occd_conv_plan_set_class_lut: the plan writes no class map");
  if (!lut) {
    e->class_lut_use = 0;
    return OCCD_OK;
  }
  OCCD_CHECK_ARG(n == e->Cout && n <= OCCD_CLASS_LUT_MAX,
                 "occd_conv_plan_set_class_lut: one label per class, at most 64 classes");
  for (int c = 0; c < OCCD_CLASS_LUT_MAX; ++c) e->class_lut[c] = c < n ? (unsigned short)lut[c] : 0;  // .astype(uint16)
  e->class_lut_use = 1;
  return OCCD_OK;
}

extern "C" int occd_conv_plan_info(const occd_conv_plan* pl, int* info) {
  OCCD_CHECK_ARG(pl && info, "occd_conv_plan_info: null");
  if (pl->impl == OCCD_CONV_IMPL_SIMT) {
    for (int i = 0; i < 8; ++i) info[i] = 0;
    info[6] = (int)pl->grid.x;
    return OCCD_OK;
  }
  if (pl->impl == OCCD_CONV_IMPL_HALO) {
    const HaloParams& h = pl->halo;
    info[0] = h.BD; info[1] = h.BH; info[2] = h.BW; info[3] = h.N_tile; info[4] = pl->kc;
    info[5] = h.stages * 100 + h.nM; info[6] = (int)pl->grid.x;
    info[7] = h.epi.B * h.d * h.d * h.d * h.tilesD * h.tilesH * h.tilesW;
    return OCCD_OK;
  }
  if (pl->impl == OCCD_CONV_IMPL_HALOX) {
    const HaloxParams& h = pl->halox;
    info[0] = h.BD; info[1] = h.BH; info[2] = h.PW; info[3] = h.N_tile; info[4] = pl->kc;
    info[5] = h.stages * 100 + h.nM; info[6] = (int)pl->grid.x;
    info[7] = h.epi.B * h.d * h.d * h.tilesD * h.tilesH;
    return OCCD_OK;
  }
  info[0] = pl->tc.TD; info[1] = pl->tc.TH; info[2] = pl->tc.TW; info[3] = pl->tc.N_tile;
  info[4] = pl->kc; info[5] = pl->tc.stages * 100 + pl->tc.group; info[6] = (int)pl->grid.x;
  info[7] = pl->tc.num_m_tiles * (pl->impl == OCCD_CONV_IMPL_TCX ? 1 : pl->tc.Cout_pad / pl->tc.N_tile);
  return OCCD_OK;
}

extern "C" int occd_conv_plan_impl(const occd_conv_plan* pl, int* impl) {
  OCCD_CHECK_ARG(pl && impl, "occd_conv_plan_impl: null");
  *impl = pl->impl;
  return OCCD_OK;
}

extern "C" int occd_conv_plan_schedule(const occd_conv_plan* pl, int* schedule) {
  OCCD_CHECK_ARG(pl && schedule, "occd_conv_plan_schedule: null");
  // conv_halo_kernel is always cooperative
  const int pp = pl->impl == OCCD_CONV_IMPL_HALOX ? pl->halox.pp
                 : (pl->impl == OCCD_CONV_IMPL_TC || pl->impl == OCCD_CONV_IMPL_TCX) ? pl->tc.pp : 0;
  *schedule = pl->impl == OCCD_CONV_IMPL_SIMT ? OCCD_CONV_SCHED_NONE
                                              : (pp ? OCCD_CONV_SCHED_PINGPONG : OCCD_CONV_SCHED_COOPERATIVE);
  return OCCD_OK;
}

template <typename T>
static int run_typed(const occd_conv_plan* pl, cudaStream_t st) {
  if (pl->impl == OCCD_CONV_IMPL_SIMT) {
    conv_simt_kernel<T><<<pl->grid, 128, 0, st>>>(pl->simt);
    OCCD_CHECK_LAUNCH();
    return OCCD_OK;
  }
  if (pl->impl == OCCD_CONV_IMPL_HALO || pl->impl == OCCD_CONV_IMPL_HALOX) return run_halo_family<T>(pl, st);
  if (pl->impl == OCCD_CONV_IMPL_TC || pl->impl == OCCD_CONV_IMPL_TCX) return run_tc_family<T>(pl, st);
  occd_set_last_error("occd_conv_run: bad plan");
  return OCCD_ERR_ARG;
}

extern "C" int occd_conv_run(const occd_conv_plan* pl, void* stream) {
  OCCD_CHECK_ARG(pl != nullptr, "occd_conv_run: null plan");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (pl->dtype == OCCD_DTYPE_F32) return run_typed<float>(pl, st);
  return run_typed<__nv_bfloat16>(pl, st);
}
