// The tensor-core convolution kernels (per-tap, halo-tile and x-packed halo-tile), their parameter blocks and
// launchers.  Each kernel is compiled once per N tile it can run with (NTiles below); the instantiations are spread
// over conv_tc_f32.cu, conv_tc_bf16.cu and conv_halo.cu so that they compile in parallel.  conv.cu plans.
#pragma once
#include "conv_common.cuh"
#include "conv_tc.cuh"
#include <type_traits>
#include <utility>

namespace occd_conv {

// 384 threads: warpgroup 0 is the TMA producer (one lane issues, the rest give their registers away), warpgroups 1
// and 2 issue wgmma and run the epilogue (fp32 accumulators in registers) on one of two schedules, chosen by the
// plan (ping_pong below) and compiled as a template parameter:
//   ping-pong: each MMA warpgroup owns whole 128-row tiles, alternately (warpgroup 1 the CTA's
//     tiles 0, 2, 4, ..., warpgroup 2 tiles 1, 3, ...).  A pair of named barriers passes the right to issue wgmma
//     from one to the other once a tile's last wgmma is issued, so one tile's epilogue runs under the next tile's
//     MMAs.  The accumulator is N registers per thread (two m64nN halves).
//   cooperative: both warpgroups work on every tile, each on 64 of its 128 rows (N / 2 registers), and
//     run their epilogues at the same time.
constexpr int kTcThreads = 384;
constexpr int kMaxStages = 24;
// Ping-pong needs the N-register accumulator to fit (N <= kPingPongMaxN) and pays off only when every warpgroup
// has tiles to alternate: a CTA with a single tile would leave one warpgroup idle and the other with the whole
// tile's epilogue, so plans with fewer than kPingPongMinTiles tiles per CTA stay cooperative.
constexpr int kPingPongMaxN = 128;
constexpr int kPingPongMinTiles = 4;
__host__ __device__ constexpr bool ping_pong(int n) { return n <= kPingPongMaxN; }
__host__ __device__ constexpr bool ping_pong(int n, long long tiles, long long ctas) {
  return ping_pong(n) && tiles >= kPingPongMinTiles * ctas;
}
// arrivals that free a stage: one per MMA warp that reads it (4 per warpgroup)
__host__ __device__ constexpr int empty_arrivals(bool pp) { return pp ? 4 : 8; }
constexpr int kEmptyArrivals = 8;   // the halo kernels: both warpgroups read every stage
// named barriers: 1 + wg: a warpgroup's epilogue staging / neighbour exchange; kTurnBar + wg: warpgroup wg may issue
// wgmma (ping-pong)
constexpr int kTurnBar = 3;
// accumulator staging for the epilogue: [2 warpgroups][64 rows][LD floats].  The per-tap kernel stages rounds of
// 32 columns (LD = kStageWide); the halo kernel, whose resident weights leave less shared memory, rounds of 8 columns
// (LD = kStageHalo)
constexpr int kStageWide = 36;
constexpr int kStageHalo = 10;
__host__ __device__ constexpr int staging_bytes(int ld) { return 2 * 64 * ld * 4; }
// The x-packed kernels keep the accumulator in registers and exchange only the W neighbours that cross a warp's 16
// rows: per 16-channel chunk, every warp leaves the Q_0 of its last d rows and the Q_2 of its first d rows
// ([4 warps][2][d][16] floats per warpgroup; d <= 8, the W dilation)
__host__ __device__ constexpr int xp_xchg_floats(int d) { return 4 * 2 * d * 16; }
__host__ __device__ constexpr int xp_xchg_bytes(int d) { return 2 * xp_xchg_floats(d) * 4; }

struct TcParams {
  ConvEpi epi;
  int n_taps;
  int n_kchunks[OCCD_CONV_MAX_SRC];
  int tiles_w, tiles_h, tiles_d, num_m_tiles;
  int src_d0;
  int w_batch_rows;  // weight rows per image (0: shared weights)
  int TD, TH, TW;
  int TWv;           // output columns per tile row: TW, or 30 for the x-packed variant (one halo column each side)
  int stride[3];
  int Cout_pad, N_tile;
  int stages, group;
  int a_bytes, b_stride, b_bytes;
  int rb;            // bytes per K chunk row: 128 / 64 / 32 == the swizzle mode
  int pdl;           // launched with programmatic stream serialization: wait for the producer grid after the prologue
  int pp;            // ping-pong schedule (else cooperative), see kTcThreads
  signed char tap_src[OCCD_CONV_MAX_TAPS];
  short tap_dz[OCCD_CONV_MAX_TAPS], tap_dy[OCCD_CONV_MAX_TAPS], tap_dx[OCCD_CONV_MAX_TAPS];
  // tap groups: n_groups convolutions over the same sources and iteration space in one launch (the sub-pixel phases
  // of a stride-2 transposed conv).  Tiles are ordered group-major, so every CTA of the persistent grid takes the
  // same share of each group (the groups differ in tap count).  n_groups == 1: the whole tap list, epi.oadd.
  int n_groups;
  short grp_tap0[OCCD_CONV_MAX_GROUPS + 1];
  short grp_iters[OCCD_CONV_MAX_GROUPS];
  signed char grp_oadd[OCCD_CONV_MAX_GROUPS][3];
};

// One pipeline item (one K chunk of RB bytes per row) of a warpgroup's NH x 64 x N accumulator tile: RB / 32 wgmma
// steps of NH m64nN instructions each (ping-pong: NH = 2, rows 0-63 and 64-127 with the same B operand, A advanced
// by a_half), issued as one wgmma group.  first: the item's first step overwrites the accumulators.  The steps are
// straight-line code for each of the three chunk widths: a wgmma inside a loop or behind a branch makes ptxas fence
// and close every instruction on its own.
template <typename T, int NMMA, int N, int NH>
__device__ __forceinline__ void mma_steps(float (&acc)[NH][N / 2], uint64_t da, uint64_t db, uint64_t a_half,
                                          bool first) {
  tc::wg_fence();
#pragma unroll
  for (int k = 0; k < NMMA; ++k)
#pragma unroll
    for (int h = 0; h < NH; ++h)
      tc::Mma<T, N>::issue(acc[h], da + h * a_half + 2 * k, db + 2 * k, (first && k == 0) ? 0u : 1u);
  tc::wg_commit();
}
template <typename T, int N, int NH>
__device__ __forceinline__ void mma_item(float (&acc)[NH][N / 2], uint64_t da, uint64_t db, uint64_t a_half,
                                         int nmma, bool first) {
  if (nmma == 4) mma_steps<T, 4, N, NH>(acc, da, db, a_half, first);
  else if (nmma == 2) mma_steps<T, 2, N, NH>(acc, da, db, a_half, first);
  else mma_steps<T, 1, N, NH>(acc, da, db, a_half, first);
}
template <int NH, int NA> __device__ __forceinline__ void acc_fence(float (&acc)[NH][NA]) {
#pragma unroll
  for (int h = 0; h < NH; ++h) tc::acc_fence(acc[h]);
}

// Ping-pong turn of the tile with CTA-local index q (owned by warpgroup q & 1): wait for the previous tile's owner to
// have issued its last wgmma; after the tile's own last wgmma, hand the turn on if the CTA has a next tile.  Every
// wait is matched by exactly one signal.
__device__ __forceinline__ void turn_take(int wg, int q) {
  if (q > 0) tc::pair_wait(kTurnBar + wg);
}
__device__ __forceinline__ void turn_pass(int wg, bool has_next) {
  if (has_next) tc::pair_signal(kTurnBar + (wg ^ 1));
}

// This thread's part of the 8-column block `blk` (a compile-time index after unrolling) of the accumulator tile ->
// st[row][col0, col0 + 8).  wgmma m64nN fragment: warp w of the warpgroup holds rows 16w + lane/4 and
// 16w + lane/4 + 8, columns 2 (lane % 4) + {0, 1} of every 8-column block, in acc[4 blk .. 4 blk + 3].
template <int LD, int N>
__device__ __forceinline__ void stage8(float* st, const float (&acc)[N / 2], int blk, int col0, int warp4,
                                       int lane) {
  const int r0 = 16 * warp4 + (lane >> 2), cc = col0 + 2 * (lane & 3);
  *reinterpret_cast<float2*>(st + r0 * LD + cc) = make_float2(acc[4 * blk], acc[4 * blk + 1]);
  *reinterpret_cast<float2*>(st + (r0 + 8) * LD + cc) = make_float2(acc[4 * blk + 2], acc[4 * blk + 3]);
}

// Epilogue of one warpgroup's 64-row tile, columns [0, N) of output channels n0 + [0, N): rounds of 32
// (LD = kStageWide) or 8 (kStageHalo) columns go through shared memory so that thread t owns row t / 2 and 16
// consecutive channels -- with 8-column rounds threads 0..63 own row t -- the vector width of the channels-last
// stores.  The caller gives the position of the thread's row; oa:
// per-launch output offset (tap groups) or nullptr for e.oadd.  A class map needs the whole channel range in this
// tile (n0 == 0, Cout <= N: plan creation refuses anything else); the two threads of a row merge their arg-max by
// shuffle and the first one stores.  With the probabilities both threads of the row then stage their channels again
// and store each channel's probability.
template <typename T, int N, int LD>
__device__ __forceinline__ void epilogue_rows(const ConvEpi& e, const float (&acc)[N / 2], float* st, int bar_id,
                                              int warp4, int lane, int t, bool valid, int b, int od, int oh, int ow,
                                              int n0, const signed char* oa) {
  constexpr int ROUND = LD == kStageWide ? 32 : 8;
  constexpr int TPR = ROUND == 8 ? 1 : 2, VW = ROUND / TPR;   // threads per row, channels per thread
  const int row = t / TPR, h = t % TPR;
  if (class_mode(e.out1_mode)) {
    // class map: every value joins the row's running arg-max (and softmax) as it leaves the staging buffer
    const bool conf = class_softmax(e.out1_mode);
    ClassArg ca = class_arg_init();
    const long long pos = valid ? epi_pos(e, b, od, oh, ow) : 0;
#pragma unroll
    for (int c0 = 0; c0 < N; c0 += ROUND) {
      tc::wg_sync(bar_id);
#pragma unroll
      for (int j = 0; j < ROUND / 8; ++j)
        if (c0 + 8 * j < N) stage8<LD, N>(st, acc, (c0 >> 3) + j, 8 * j, warp4, lane);
      tc::wg_sync(bar_id);
      const int cc = c0 + VW * h;
      if (valid && row < 64 && cc < N) {
#pragma unroll 1
        for (int i = 0; i < VW && n0 + cc + i < e.Cout; ++i)
          class_arg_take(ca, class_value<T>(e, pos, n0 + cc + i, st[row * LD + VW * h + i]), n0 + cc + i, conf);
      }
    }
    if constexpr (TPR == 2) class_arg_merge_xor(ca, 1, conf);
    if (valid && row < 64 && h == 0) class_store(e, pos, ca);
    // the probabilities: the same rounds again, now that the row's softmax is complete (wider tiles hold too many
    // accumulator registers for a second pass: plan creation refuses them the mode)
    if constexpr (N <= kProbsMaxN) {
      if (e.out1_mode == OCCD_OUT1_CLASS_U16_PROBS) {
#pragma unroll
        for (int c0 = 0; c0 < N; c0 += ROUND) {
          tc::wg_sync(bar_id);
#pragma unroll
          for (int j = 0; j < ROUND / 8; ++j)
            if (c0 + 8 * j < N) stage8<LD, N>(st, acc, (c0 >> 3) + j, 8 * j, warp4, lane);
          tc::wg_sync(bar_id);
          const int cc = c0 + VW * h;
          if (valid && row < 64 && cc < N) {
#pragma unroll 1
            for (int i = 0; i < VW && n0 + cc + i < e.Cout; ++i)
              class_prob_store(e, b, pos, n0 + cc + i, class_value<T>(e, pos, n0 + cc + i, st[row * LD + VW * h + i]),
                               ca);
          }
        }
      }
    }
    return;
  }
  const bool fast = VW == 16 && epi_fast_ok(e);
  EpiRow<T> er;
  if (fast)
    er = oa ? epi_row<T>(e, valid, b, od, oh, ow, n0, oa[0], oa[1], oa[2]) : epi_row<T>(e, valid, b, od, oh, ow, n0);
#pragma unroll
  for (int c0 = 0; c0 < N; c0 += ROUND) {
    tc::wg_sync(bar_id);   // the previous round's reads are done
#pragma unroll
    for (int j = 0; j < ROUND / 8; ++j)
      if (c0 + 8 * j < N) stage8<LD, N>(st, acc, (c0 >> 3) + j, 8 * j, warp4, lane);
    tc::wg_sync(bar_id);
    const int cc = c0 + VW * h;
    if (row < 64 && cc < N) {
      float v[VW];
      // staged rows are 8-byte aligned (LD is even)
      const float2* sp = reinterpret_cast<const float2*>(st + row * LD + VW * h);
#pragma unroll
      for (int i = 0; i < VW / 2; ++i) {
        const float2 x = sp[i];
        v[2 * i] = x.x; v[2 * i + 1] = x.y;
      }
      if constexpr (VW == 16) {
        if (fast) {
          EpiPre q;
          epi_prefetch<T>(er, cc, q);
          epi_finish_v<T>(er, cc, v, q.b, q.r);
          continue;
        }
      }
      if (valid) conv_epilogue_row<T, VW>(e, b, od, oh, ow, n0 + cc, v);
    }
  }
}

// __shfl_sync of an accumulator value on an f32 register: with the intrinsic the compiler keeps the accumulator in
// integer registers (shfl is a .b32 operation) and copies it into f32 registers around every wgmma, which breaks the
// wgmma pipeline (ptxas injects warpgroup.arrive / wait and serialises)
__device__ __forceinline__ float shfl_acc(float x, int src) {
  float r;
  asm volatile("shfl.sync.idx.b32 %0, %1, %2, 0x1f, 0xffffffff;" : "=f"(r) : "f"(x), "r"(src));
  return r;
}

// The x-packed epilogue's view of a thread's two rows 16 w + l / 4 + {0, 8} (lane l of warp w): lo_ok / hi_ok
// false where the W neighbour r - d / r + d falls outside the line, i.e. onto the conv's zero padding; and the
// output position of the row whose channels the thread stores, 16 w + l / 4 + 8 ((l % 4) >> 1)
struct XpRows {
  bool lo_ok[2], hi_ok[2];
  bool valid;
  int od, oh, ow;
};

// Epilogue of the x-packed kernels, straight from the accumulator registers: the accumulator holds three column
// groups Q_c (c = 0, 1, 2: the W taps -d, 0, +d) of CP = N / 3 columns each and out[r] = (Q_1[r] + Q_0[r - d]) +
// Q_2[r + d], where r -+ d stays inside the line of rows.  In the m64nN fragment lane l of warp w holds rows
// 16 w + l / 4 and + 8, columns 2 (l % 4) + {0, 1} of every 8-column block, so every thread
// holds the same channels of Q_0, Q_1 and Q_2: a neighbour inside the warp's 16 rows is a shuffle from lane l -+ 4 d,
// one in the next or previous warp comes through the exchange buffer xb (xp_xchg_floats(d) floats, this
// warpgroup's).  Chunks of 16 channels: two barriers each.  The sums of a row's 8-channel block are then gathered
// into one lane of the quad (a 4 x 4 transpose of channel pairs by shuffle), which runs the row epilogue on them;
// a class map instead takes them into the row's running arg-max (and softmax), and the two lanes of a row merge theirs;
// with the probabilities the chunk loop then runs again and both lanes store their channels' probabilities.
template <typename T, int N>
__device__ __forceinline__ void epilogue_xp(const ConvEpi& e, const float (&acc)[N / 2], float* xb, int bar_id,
                                            int warp4, int lane, int d, const XpRows& rows, int b) {
  constexpr int CP = N / 3;
  constexpr unsigned FULL = 0xffffffffu;
  const int g = lane >> 2, q = lane & 3;
  const int lo_src = (lane - 4 * d) & 31, hi_src = (lane + 4 * d) & 31;
  const int wfl = 2 * d * 16;   // exchange floats per warp: [Q_0 of the last d rows, Q_2 of the first d rows][16]
  float* const mine = xb + warp4 * wfl;
  const bool my_valid = rows.valid;   // after the transpose this lane holds 8 channels of row 16 w + g + 8 (q >> 1)
  // one copy of the chunk loop per output kind (CLS: class map), so that neither carries the other's registers;
  // a class map's values go to take(n, value)
  auto chunks = [&](auto cls, auto&& take) {
    constexpr bool CLS = decltype(cls)::value;
    const long long pos = CLS && my_valid ? epi_pos(e, b, rows.od, rows.oh, rows.ow) : 0;
#pragma unroll
    for (int c0 = 0; c0 < CP; c0 += 16) {
      tc::wg_sync(bar_id);   // the previous chunk's exchange reads are done
#pragma unroll
      for (int jb = 0; jb < 2; ++jb)
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int c = 8 * jb + 2 * q + k;
          const int j0 = 4 * ((c0 >> 3) + jb) + k, j2 = 4 * ((2 * CP + c0) >> 3) + 4 * jb + k;
          if (g >= 8 - d) mine[(g - (8 - d)) * 16 + c] = acc[j0 + 2];
          if (g < d) mine[(d + g) * 16 + c] = acc[j2];
        }
      tc::wg_sync(bar_id);
      float v[2][2][2];   // [row][8-channel block][channel of the pair]
#pragma unroll
      for (int jb = 0; jb < 2; ++jb)
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int c = 8 * jb + 2 * q + k;
          const int j0 = 4 * ((c0 >> 3) + jb) + k, j1 = 4 * ((CP + c0) >> 3) + 4 * jb + k,
                    j2 = 4 * ((2 * CP + c0) >> 3) + 4 * jb + k;
          const float q0a = shfl_acc(acc[j0], lo_src), q0b = shfl_acc(acc[j0 + 2], lo_src);
          const float q2a = shfl_acc(acc[j2], hi_src), q2b = shfl_acc(acc[j2 + 2], hi_src);
          // row 16 w + g: Q_0 of row g - d (the previous warp's when g < d), Q_2 of row g + d
          const float lo0 = g >= d ? q0a : (warp4 > 0 ? mine[g * 16 + c - wfl] : 0.f);
          const float hi0 = g + d < 8 ? q2a : q2b;
          // row 16 w + g + 8: Q_0 of row g + 8 - d, Q_2 of row g + 8 + d (the next warp's when g + d >= 8)
          const float lo1 = g >= d ? q0b : q0a;
          const float hi1 = g + d < 8 ? q2b : (warp4 < 3 ? mine[wfl + (2 * d + g - 8) * 16 + c] : 0.f);
          v[0][jb][k] = acc[j1] + (rows.lo_ok[0] ? lo0 : 0.f);
          v[0][jb][k] += rows.hi_ok[0] ? hi0 : 0.f;
          v[1][jb][k] = acc[j1 + 2] + (rows.lo_ok[1] ? lo1 : 0.f);
          v[1][jb][k] += rows.hi_ok[1] ? hi1 : 0.f;
        }
      // unit u = 2 * row + block: this lane holds its channel pair q; after the transpose o[p] is pair p of unit q
      float2 u[4], o[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) o[i] = u[i] = make_float2(v[i >> 1][i & 1][0], v[i >> 1][i & 1][1]);
#pragma unroll
      for (int k = 1; k < 4; ++k) {
        // lane q ^ k sends its pair of unit q while this lane sends its pair of unit q ^ k
        const int pk = q ^ k;
        float2 snd = u[0];
#pragma unroll
        for (int i = 1; i < 4; ++i) snd = pk == i ? u[i] : snd;
        const float2 r = make_float2(__shfl_xor_sync(FULL, snd.x, k), __shfl_xor_sync(FULL, snd.y, k));
#pragma unroll
        for (int i = 0; i < 4; ++i) o[i] = pk == i ? r : o[i];
      }
      float w8[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) { w8[2 * i] = o[i].x; w8[2 * i + 1] = o[i].y; }
      const int n0 = c0 + 8 * (q & 1);
      if constexpr (CLS) {
        if (my_valid && n0 < e.Cout) class_each8<T>(e, pos, n0, w8, take);
      } else {
        if (my_valid) conv_epilogue_row<T, 8>(e, b, rows.od, rows.oh, rows.ow, n0, w8);
      }
    }
  };
  if (class_mode(e.out1_mode)) {
    const bool conf = class_softmax(e.out1_mode);
    ClassArg ca = class_arg_init();
    chunks(std::true_type{}, [&](int n, float v) { class_arg_take(ca, v, n, conf); });
    // lanes q and q ^ 1 hold the two blocks of each chunk of one row
    class_arg_merge_xor(ca, 1, conf);
    if ((q & 1) == 0 && my_valid) class_store(e, epi_pos(e, b, rows.od, rows.oh, rows.ow), ca);
    if (e.out1_mode == OCCD_OUT1_CLASS_U16_PROBS) {
      const long long pos = my_valid ? epi_pos(e, b, rows.od, rows.oh, rows.ow) : 0;
      chunks(std::true_type{}, [&](int n, float v) { class_prob_store(e, b, pos, n, v, ca); });
    }
  } else {
    chunks(std::false_type{}, [](int, float) {});
  }
}

__device__ __forceinline__ void pdl_prologue_done(int pdl) {
  if (pdl) {
    // programmatic dependent launch: everything above (barrier init, tensor-map prefetch) overlapped the tail of the
    // producer grid; its results are only touched below this point
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  }
}

// XP: x-packed variant: the pipeline items are (source, dz, dy) groups whose B operand stacks the three W taps
// (N_tile = 3 * Cout_pad: with taps in lexicographic order that is 3 consecutive tap slices of the ordinary weight
// tensor), tiles are 32 wide with one halo column on each side, and the epilogue forms
// out[r] = Q_0[r-1] + Q_1[r] + Q_2[r+1] from the three column groups.  One A fetch then feeds 3x the output columns.
// N: the N tile (== p.N_tile), one m64nN wgmma per warpgroup and K step.
template <typename T, int N, bool XP, bool PP>
__global__ void __launch_bounds__(kTcThreads, 1)
conv_tc_kernel(const __grid_constant__ TcParams p, const __grid_constant__ CUtensorMap tmA0,
               const __grid_constant__ CUtensorMap tmA1, const __grid_constant__ CUtensorMap tmA2,
               const __grid_constant__ CUtensorMap tmW) {
  // Persistent, warp-specialised implicit GEMM.  Each CTA walks tiles blockIdx.x, +gridDim.x, ...:
  //   warp 0 (one lane): TMA producer -- runs ahead across tile boundaries, the smem ring never drains
  //   warpgroups 1, 2  : wgmma, then the epilogue from registers (ping-pong or cooperative, see kTcThreads)
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // dynamic smem is only guaranteed 16-byte aligned: round the base up to 1024 (swizzle atom alignment)
  const uint32_t smem_base = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_a = smem_base;
  const uint32_t smem_b = smem_a + (uint32_t)(p.stages * p.group) * p.a_bytes;
  constexpr int LD = kStageWide;
  static_assert(!PP || ping_pong(N), "ping-pong holds N accumulator registers per thread");
  constexpr int NH = PP ? 2 : 1;   // 64-row halves of the M tile in one warpgroup's accumulator
  const uint32_t smem_st = smem_b + (uint32_t)(p.stages * p.group) * p.b_stride;
  const uint32_t bar_base = smem_st + (uint32_t)(XP ? xp_xchg_bytes(1) : staging_bytes(LD));
  const uint32_t full_bar = bar_base;
  const uint32_t empty_bar = bar_base + 8u * kMaxStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n_tiles_n = XP ? 1 : p.Cout_pad / N;
  const int tiles_per_group = p.num_m_tiles * n_tiles_n;
  const int num_tiles = tiles_per_group * p.n_groups;
  const int RB = p.rb;
  const int KCH = RB / (int)sizeof(T);  // channels per K chunk

  if (threadIdx.x == 0) {
    tc::prefetch_tmap(&tmA0);
    tc::prefetch_tmap(&tmW);
    for (int s = 0; s < p.stages; ++s) {
      tc::mbar_init(full_bar + 8u * s, 1);
      tc::mbar_init(empty_bar + 8u * s, empty_arrivals(PP));
    }
    tc::fence_barrier_init();
  }
  __syncthreads();
  pdl_prologue_done(p.pdl);

  if (warp < 4) {
    tc::reg_dealloc<40>();
    if (warp == 0 && lane == 0) {
      // ===== TMA producer =====
      const CUtensorMap* maps[3] = {&tmA0, &tmA1, &tmA2};
      int s = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int grp = tile / tiles_per_group;
        const int tg = tile - grp * tiles_per_group;
        const int nt = tg % n_tiles_n;
        int t = tg / n_tiles_n;
        const int tw = t % p.tiles_w; t /= p.tiles_w;
        const int th = t % p.tiles_h; t /= p.tiles_h;
        const int td = t % p.tiles_d; t /= p.tiles_d;
        const int b = t;
        const int iw0 = XP ? tw * 30 - 1 : tw * p.TW * p.stride[2], ih0 = th * p.TH * p.stride[1],
                  id0 = td * p.TD * p.stride[0] + p.src_d0;
        const int n0 = nt * N;
        // items (tap, k-chunk) are loaded in groups of p.group per pipeline stage: one barrier hand-off per group
        int g = 0;
        int remaining = p.grp_iters[grp];
        for (int tp = p.grp_tap0[grp]; tp < p.grp_tap0[grp + 1]; ++tp) {
          const int src = p.tap_src[tp];
          const int cw = iw0 + p.tap_dx[tp], ch = ih0 + p.tap_dy[tp], cd = id0 + p.tap_dz[tp];
          const int wrow = b * p.w_batch_rows + (XP ? tp * N : tp * p.Cout_pad + n0);
          const int nk = p.n_kchunks[src];
          for (int kc = 0; kc < nk; ++kc) {
            if (g == 0) {
              const int cnt = remaining < p.group ? remaining : p.group;
              tc::mbar_wait(empty_bar + 8u * s, ph ^ 1u);
              tc::mbar_expect_tx(full_bar + 8u * s, (uint32_t)(cnt * (p.a_bytes + p.b_bytes)));
            }
            const uint32_t sa = smem_a + (uint32_t)(s * p.group + g) * p.a_bytes;
            const uint32_t sb = smem_b + (uint32_t)(s * p.group + g) * p.b_stride;
            tc::tma_load_5d(sa, maps[src], full_bar + 8u * s, kc * KCH, cw, ch, cd, b);
            tc::tma_load_2d(sb, &tmW, full_bar + 8u * s, kc * KCH, wrow);
            --remaining;
            if (++g == p.group || remaining == 0) {
              g = 0;
              if (++s == p.stages) { s = 0; ph ^= 1u; }
            }
          }
        }
      }
    }
    return;
  }

  // ===== MMA + epilogue warpgroups =====
  tc::reg_alloc<232>();
  const int wg = (warp >> 2) - 1;
  const int warp4 = warp & 3;
  const int t = threadIdx.x & 127;
  float* st = reinterpret_cast<float*>(smem_raw + (smem_st - tc::smem_u32(smem_raw))) +
              wg * (XP ? xp_xchg_floats(1) : 64 * LD);
  const int nmma = RB / 32;
  const uint64_t a_half = (uint64_t)(64 * RB / 16);
  const uint64_t da0 = tc::make_sdesc(smem_a, RB) + (PP ? 0 : wg * a_half);
  const uint64_t db0 = tc::make_sdesc(smem_b, RB);
  float acc[NH][N / 2];
  int s = 0;
  uint32_t ph = 0;
  int q = 0;   // CTA-local tile index
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++q) {
    const int tgrp = tile / tiles_per_group;       // tap group (sub-pixel phase) of this tile
    const int iters = p.grp_iters[tgrp];
    if (PP && (q & 1) != wg) {
      // the other warpgroup's tile: step over the stages the producer fills for it
      for (int n = (iters + p.group - 1) / p.group; n > 0; --n)
        if (++s == p.stages) { s = 0; ph ^= 1u; }
      continue;
    }
    if (PP) turn_take(wg, q);
    int prev = -1;
    for (int it = 0; it < iters;) {
      tc::mbar_wait(full_bar + 8u * s, ph);
      const int cnt = (iters - it) < p.group ? (iters - it) : p.group;
      for (int g = 0; g < cnt; ++g, ++it) {
        const uint64_t da = da0 + (uint64_t)((s * p.group + g) * (p.a_bytes >> 4));
        const uint64_t db = db0 + (uint64_t)((s * p.group + g) * (p.b_stride >> 4));
        mma_item<T, N, NH>(acc, da, db, a_half, nmma, it == 0);
      }
      if (PP && it == iters) turn_pass(wg, tile + (int)gridDim.x < num_tiles);   // the tile's last wgmma is issued
      tc::wg_wait_le(cnt);  // only this stage's groups are pending: hand the previous stage back to the producer
      if (prev >= 0 && lane == 0) tc::mbar_arrive(empty_bar + 8u * prev);
      prev = s;
      if (++s == p.stages) { s = 0; ph ^= 1u; }
    }
    tc::wg_wait<0>();
    if (lane == 0) tc::mbar_arrive(empty_bar + 8u * prev);
    acc_fence(acc);

    const int tg = tile - tgrp * tiles_per_group;
    const int nt = tg % n_tiles_n;
    int tt = tg / n_tiles_n;
    const int tw = tt % p.tiles_w; tt /= p.tiles_w;
    const int th = tt % p.tiles_h; tt /= p.tiles_h;
    const int td = tt % p.tiles_d; tt /= p.tiles_d;
    const int b = tt;
#pragma unroll
    for (int h = 0; h < NH; ++h) {
      const int r64 = 64 * (PP ? h : wg);   // first row of this 64-row half of the M tile
      if constexpr (XP) {
        // TW == 32: row == tile column inside each 32-row line, so the W neighbours' partial sums are rows r -+ 1
        // (the line's first and last rows are halo columns, never stored)
        const int row = r64 + 16 * warp4 + (lane >> 2) + 8 * ((lane & 3) >> 1);
        const int rw = row % 32;
        const int rh = (row / 32) % p.TH;
        const int rd = row / (32 * p.TH);
        const int od = td * p.TD + rd, oh = th * p.TH + rh, ow = tw * 30 + rw - 1;
        const XpRows rows{{true, true}, {true, true},
                          od < p.epi.OD && oh < p.epi.OH && ow < p.epi.OW && rw >= 1 && rw <= 30, od, oh, ow};
        epilogue_xp<T, N>(p.epi, acc[h], st, 1 + wg, warp4, lane, 1, rows, b);
      } else {
        const int row = r64 + (t >> 1);
        const int rw = row % p.TW;
        const int rh = (row / p.TW) % p.TH;
        const int rd = row / (p.TW * p.TH);
        const int od = td * p.TD + rd, oh = th * p.TH + rh, ow = tw * p.TW + rw;
        const bool valid = od < p.epi.OD && oh < p.epi.OH && ow < p.epi.OW;
        epilogue_rows<T, N, LD>(p.epi, acc[h], st, 1 + wg, warp4, lane, t, valid, b, od, oh, ow, nt * N,
                                p.n_groups > 1 ? p.grp_oadd[tgrp] : nullptr);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Halo-tile variant for stride-1 3x3x3 convolutions with few channels (the full-resolution head):
// the per-tap TMA boxes of conv_tc_kernel re-load every input row 27 times and the TMA unit becomes the limiter.
// Here each CTA tile loads ONE zero-filled halo box (PD x PH x PW positions, rows of one K chunk) and feeds all 27
// taps from row-shifted views of that box: with smem rows linearised as r = (pd*PH + ph)*PW + pw, the A operand of
// tap (a,b,c) for output rows [R, R+64) is simply rows [R + (a*PH + b)*PW + c, ...) -- a different wgmma start
// address, same data.  Rows that fall in the halo produce garbage accumulator rows that the epilogue never stores.
// Dilation d runs the same scheme on the d^3 sub-sampled grids (TMA traversal stride d), so the halo is always one
// position.  Weights for all taps stay resident in shared memory.
struct HaloParams {
  ConvEpi epi;
  int d;                      // dilation (== padding)
  int D, H, W;                // full grid (== output grid)
  int BD, BH, BW, PD, PH, PW;  // valid box / halo box (sub-sampled coordinates)
  int src_d0;                 // plane offset of the interior inside a halo-margin source buffer
  int hd, hh, hw;             // 1 where the taps reach into that dimension (halo of one sub-sampled position)
  int tilesD, tilesH, tilesW;
  int nM, R0;                 // M tiles per CTA tile, first valid row
  int box_bytes;              // bytes one TMA box delivers
  int a_stage_bytes;          // allocated per stage (box + slack rows read by garbage outputs)
  int stages;
  int n_taps;
  int N_tile, rb;
  int b_stride, w_bytes;
  int tap_off16[27];          // (R0 + (a*PH + b)*PW + c) * row_bytes / 16: A-descriptor advance per tap
  int pdl;                    // see TcParams::pdl
};

// N: the N tile (== p.N_tile == Cout_pad)
template <typename T, int N>
__global__ void __launch_bounds__(kTcThreads, 1)
conv_halo_kernel(const __grid_constant__ HaloParams p, const __grid_constant__ CUtensorMap tmA,
                 const __grid_constant__ CUtensorMap tmW) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem_base = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_w = smem_base;                                   // [n_taps][b_stride] resident weights
  const uint32_t smem_a = smem_w + (uint32_t)p.w_bytes;                 // [stages][a_stage_bytes]
  constexpr int LD = kStageHalo;
  const uint32_t smem_st = smem_a + (uint32_t)p.stages * p.a_stage_bytes;
  const uint32_t bar_base = smem_st + (uint32_t)staging_bytes(LD);
  const uint32_t full_bar = bar_base;            // [4]
  const uint32_t empty_bar = bar_base + 32u;     // [4]
  const uint32_t w_bar = bar_base + 64u;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int d = p.d;
  const int per_res = p.tilesD * p.tilesH * p.tilesW;
  const int num_tiles = p.epi.B * d * d * d * per_res;
  const int RB = p.rb;

  if (threadIdx.x == 0) {
    tc::prefetch_tmap(&tmA);
    tc::prefetch_tmap(&tmW);
    for (int s = 0; s < p.stages; ++s) {
      tc::mbar_init(full_bar + 8u * s, 1);
      tc::mbar_init(empty_bar + 8u * s, kEmptyArrivals);
    }
    tc::mbar_init(w_bar, 1);
    tc::fence_barrier_init();
  }
  __syncthreads();
  pdl_prologue_done(p.pdl);

  // tile -> (batch, residue class, sub-grid tile origin)
  auto decode = [&](int tile, int& b, int& ra, int& rb, int& rc, int& td, int& th, int& tw) {
    int t = tile;
    tw = t % p.tilesW; t /= p.tilesW;
    th = t % p.tilesH; t /= p.tilesH;
    td = t % p.tilesD; t /= p.tilesD;
    rc = t % d; t /= d;
    rb = t % d; t /= d;
    ra = t % d; t /= d;
    b = t;
  };

  if (warp < 4) {
    tc::reg_dealloc<40>();
    if (warp == 0 && lane == 0) {
      // ===== TMA producer: resident weights once, then one halo box per tile =====
      tc::mbar_expect_tx(w_bar, (uint32_t)(p.n_taps * N * RB));
      for (int tp = 0; tp < p.n_taps; ++tp)
        tc::tma_load_2d(smem_w + (uint32_t)tp * p.b_stride, &tmW, w_bar, 0, tp * N);
      int s = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int b, ra, rb, rc, td, th, tw;
        decode(tile, b, ra, rb, rc, td, th, tw);
        tc::mbar_wait(empty_bar + 8u * s, ph ^ 1u);
        tc::mbar_expect_tx(full_bar + 8u * s, (uint32_t)p.box_bytes);
        tc::tma_load_5d(smem_a + (uint32_t)s * p.a_stage_bytes, &tmA, full_bar + 8u * s, 0,
                        (tw * p.BW - p.hw) * d + rc, (th * p.BH - p.hh) * d + rb,
                        (td * p.BD - p.hd) * d + ra + p.src_d0, b);
        if (++s == p.stages) { s = 0; ph ^= 1u; }
      }
    }
    return;
  }

  // ===== MMA + epilogue warpgroups: M tile m, rows [64 wg, 64 wg + 64) =====
  tc::reg_alloc<232>();
  const int wg = (warp >> 2) - 1;
  const int warp4 = warp & 3;
  const int t = threadIdx.x & 127;
  float* st = reinterpret_cast<float*>(smem_raw + (smem_st - tc::smem_u32(smem_raw))) + wg * 64 * LD;
  const int nmma = RB / 32;
  const uint64_t db_w = tc::make_sdesc(smem_w, RB);
  const int w_step16 = p.b_stride / 16;
  float acc[1][N / 2];
  tc::mbar_wait(w_bar, 0);
  int s = 0;
  uint32_t ph = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int b, ra, rb, rc, td, th, tw;
    decode(tile, b, ra, rb, rc, td, th, tw);
    tc::mbar_wait(full_bar + 8u * s, ph);
    // descriptors advance by plain 64-bit adds on the 16-byte-unit address field (smem < 256 KB: no carry out of
    // the 14-bit field)
    const uint64_t da_stage = tc::make_sdesc(smem_a + (uint32_t)s * p.a_stage_bytes, RB) +
                              (uint64_t)(64 * wg * RB / 16);
    for (int m = 0; m < p.nM; ++m) {
      const uint64_t da_m = da_stage + (uint64_t)(m * (128 * RB / 16));
      for (int tp = 0; tp < p.n_taps; ++tp)
        mma_item<T, N, 1>(acc, da_m + (uint64_t)p.tap_off16[tp], db_w + (uint64_t)(tp * w_step16), 0, nmma,
                          tp == 0);
      tc::wg_wait<0>();
      if (m == p.nM - 1 && lane == 0) tc::mbar_arrive(empty_bar + 8u * s);   // the box is no longer read
      acc_fence(acc);
      const int R = p.R0 + m * 128 + 64 * wg + t;   // epilogue threads t < 64: one row each
      const int pw = R % p.PW;
      const int phh = (R / p.PW) % p.PH;
      const int pd = R / (p.PW * p.PH);
      const int od = (td * p.BD + pd - p.hd) * d + ra, oh = (th * p.BH + phh - p.hh) * d + rb,
                ow = (tw * p.BW + pw - p.hw) * d + rc;
      const bool valid = pd >= p.hd && pd < p.hd + p.BD && phh >= p.hh && phh < p.hh + p.BH && pw >= p.hw &&
                         pw < p.hw + p.BW && od < p.D && oh < p.H && ow < p.W;
      epilogue_rows<T, N, LD>(p.epi, acc[0], st, 1 + wg, warp4, lane, t, valid, b, od, oh, ow, 0, nullptr);
    }
    if (++s == p.stages) { s = 0; ph ^= 1u; }
  }
}


// ------------------------------------------------------------------------------------------------
// x-packed halo kernel for grids whose innermost extent W is one warp wide or narrower (W in {8, 16, 32}: every
// 3-D activation of this network -- Z = 32 / 16 / 8).  A 32-output-channel conv issued tap by tap keeps the tensor
// core at N = 32; here the three W taps (dx = -d, 0, +d) of each (dz, dy) pair share ONE instruction: its B operand
// stacks the three taps' weights along N (N = 3 * Cout_pad: three consecutive tap slices of the ordinary weight
// tensor), its A operand is the un-shifted rows, and the accumulator holds
//     Q_c[r] = sum_{a,b} W[a][b][c] . in[r + (a*PH + b)*PW]      c = 0, 1, 2
// from which the epilogue forms out[r] = Q_0[r - d] + Q_1[r] + Q_2[r + d].  Smem rows are linearised with W
// fastest and PW == W divides 32, so r +- d stays inside one line of the tile, masked where the neighbour would fall
// outside [0, W) -- which is exactly the convolution's zero padding, so the W axis needs no halo columns and no
// sub-sampling.  D and H keep the halo-tile scheme (one zero-filled halo position per side on the d-sub-sampled
// grids, TMA traversal stride d).  27 taps become 9 instructions per 32 bytes of K.
struct HaloxParams {
  ConvEpi epi;
  int d;                      // dilation (== padding) of the taps
  int D, H;                   // output grid (W == PW)
  int BD, BH, PD, PH, PW;     // valid box / halo box in sub-sampled (D, H) coordinates; PW == W
  int hd, hh;                 // 1 where the taps reach into D / H
  int src_d0;
  int tilesD, tilesH;
  int nM;                     // M tiles (128 smem rows = 128 / PW h-rows of one plane) per CTA tile, <= 2
  int mt_row[2], mt_pd[2], mt_ph0[2];
  int box_bytes, a_stage_bytes, stages;
  int n_groups;               // (dz, dy) groups = n_taps / 3
  int CP, N_tile, rb;         // padded output channels, N_tile = 3 * CP, bytes per K chunk row
  int b_stride, w_bytes;
  int grp_off[9];             // (a*PH + b)*PW: smem row offset of a group's A operand relative to the M tile
  int pdl;
  // plane-ring mode (ring == 1; chosen when the halo box leaves room for ONE stage only, i.e. the TF32 head whose
  // resident weights take 110 KB): the output planes of all columns (image, residue class, H tile) form one sequence
  // of n_cols * sD M tiles; every CTA takes a contiguous, equal share of it (at most one column change inside).  The
  // four stages are a ring of single input planes, output plane z reads ring planes z-1, z, z+1, so every M tile costs
  // ONE new plane (prefetched a plane ahead) instead of a whole box loaded while the tensor core waits
  int ring, sD, n_cols;
  int pp;                     // ping-pong schedule (else cooperative), see kTcThreads
  signed char grp_dz[9];      // -1 / 0 / +1: which ring plane a group reads
  short grp_row[9];           // (hh + dy) * PW: its row offset inside the plane
};

// N: the N tile (== p.N_tile == 3 * CP)
template <typename T, int N, bool PP>
__global__ void __launch_bounds__(kTcThreads, 1)
conv_halox_kernel(const __grid_constant__ HaloxParams p, const __grid_constant__ CUtensorMap tmA,
                  const __grid_constant__ CUtensorMap tmW) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem_base = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_w = smem_base;                                   // [n_groups][b_stride] resident weights
  const uint32_t smem_a = smem_w + (uint32_t)p.w_bytes;                 // [stages][a_stage_bytes]
  static_assert(!PP || ping_pong(N), "ping-pong holds N accumulator registers per thread");
  constexpr int NH = PP ? 2 : 1;
  const uint32_t smem_st = smem_a + (uint32_t)p.stages * p.a_stage_bytes;   // neighbour exchange (xp_xchg_bytes)
  const uint32_t bar_base = smem_st + (uint32_t)xp_xchg_bytes(p.d);
  const uint32_t full_bar = bar_base;            // [4]
  const uint32_t empty_bar = bar_base + 32u;     // [4]
  const uint32_t w_bar = bar_base + 64u;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int d = p.d;
  const int RB = p.rb;
  const int num_tiles = p.epi.B * d * d * p.tilesD * p.tilesH;
  // ring mode: this CTA's share [ring_lo, ring_hi) of the n_cols * sD output planes
  const long long ring_total = (long long)p.n_cols * p.sD;
  const long long ring_lo = p.ring ? ring_total * blockIdx.x / gridDim.x : 0;
  const long long ring_hi = p.ring ? ring_total * (blockIdx.x + 1) / gridDim.x : 0;

  if (threadIdx.x == 0) {
    tc::prefetch_tmap(&tmA);
    tc::prefetch_tmap(&tmW);
    for (int s = 0; s < p.stages; ++s) {
      tc::mbar_init(full_bar + 8u * s, 1);
      tc::mbar_init(empty_bar + 8u * s, kEmptyArrivals);
    }
    tc::mbar_init(w_bar, 1);
    tc::fence_barrier_init();
  }
  __syncthreads();
  pdl_prologue_done(p.pdl);

  // tile -> (batch, (D, H) residue class, sub-grid tile origin)
  auto decode = [&](int tile, int& b, int& ra, int& rb, int& td, int& th) {
    int t = tile;
    th = t % p.tilesH; t /= p.tilesH;
    td = t % p.tilesD; t /= p.tilesD;
    rb = t % d; t /= d;
    ra = t % d; t /= d;
    b = t;
  };

  // ring mode: position in the plane sequence -> (batch, residue class, H tile) and the run of planes [z0, z1) this CTA
  // takes from that column
  auto decode_ring = [&](long long pos, int& b, int& ra, int& rb, int& th, int& z0, int& z1) {
    const int ip = (int)pos;   // < n_cols * sD, an M-tile count (int, like num_tiles): a 32-bit division
    int t = ip / p.sD;
    z0 = ip - t * p.sD;
    const long long left = ring_hi - pos;
    z1 = (long long)(p.sD - z0) < left ? p.sD : z0 + (int)left;
    th = t % p.tilesH; t /= p.tilesH;
    rb = t % d; t /= d;
    ra = t % d; t /= d;
    b = t;
  };

  if (warp < 4) {
    tc::reg_dealloc<40>();
    if (warp == 0 && lane == 0) {
      // ===== TMA producer: resident weights once, then (ring) planes z0-1 .. z1 of every unit, one ring slot each,
      // or (box) one halo box per tile =====
      tc::mbar_expect_tx(w_bar, (uint32_t)(p.n_groups * N * RB));
      for (int g = 0; g < p.n_groups; ++g)
        tc::tma_load_2d(smem_w + (uint32_t)g * p.b_stride, &tmW, w_bar, 0, g * N);
      if (p.ring) {
        uint32_t n = 0;
        for (long long pos = ring_lo; pos < ring_hi;) {
          int b, ra, rb, th, z0, z1;
          decode_ring(pos, b, ra, rb, th, z0, z1);
          pos += z1 - z0;
          for (int z = z0 - 1; z <= z1; ++z, ++n) {
            const uint32_t slot = n & 3u;
            tc::mbar_wait(empty_bar + 8u * slot, ((n >> 2) & 1u) ^ 1u);
            tc::mbar_expect_tx(full_bar + 8u * slot, (uint32_t)p.box_bytes);
            tc::tma_load_5d(smem_a + slot * (uint32_t)p.a_stage_bytes, &tmA, full_bar + 8u * slot, 0, 0,
                            (th * p.BH - p.hh) * d + rb, z * d + ra + p.src_d0, b);
          }
        }
      } else {
        int s = 0;
        uint32_t ph = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
          int b, ra, rb, td, th;
          decode(tile, b, ra, rb, td, th);
          tc::mbar_wait(empty_bar + 8u * s, ph ^ 1u);
          tc::mbar_expect_tx(full_bar + 8u * s, (uint32_t)p.box_bytes);
          tc::tma_load_5d(smem_a + (uint32_t)s * p.a_stage_bytes, &tmA, full_bar + 8u * s, 0, 0,
                          (th * p.BH - p.hh) * d + rb, (td * p.BD - p.hd) * d + ra + p.src_d0, b);
          if (++s == p.stages) { s = 0; ph ^= 1u; }
        }
      }
    }
    return;
  }

  // ===== MMA + epilogue warpgroups: ping-pong (whole M tiles, alternately) or cooperative (rows [64 wg, 64 wg + 64)
  // of every M tile) =====
  tc::reg_alloc<232>();
  const int wg = (warp >> 2) - 1;
  const int warp4 = warp & 3;
  float* xb = reinterpret_cast<float*>(smem_raw + (smem_st - tc::smem_u32(smem_raw))) + wg * xp_xchg_floats(d);
  const int nmma = RB / 32;
  const uint64_t db_w = tc::make_sdesc(smem_w, RB);
  const int w_step16 = p.b_stride / 16;
  const uint64_t a_half = (uint64_t)(64 * RB / 16);
  const int row0 = PP ? 0 : 64 * wg;       // first M-tile row of this warpgroup's MMAs
  float acc[NH][N / 2];
  // epilogue of this warpgroup's rows of an M tile at output plane od whose first h-row is oh_base (sub-sampled)
  auto tile_epilogue = [&](int b, int ra, int rb, int od, int oh_base) {
#pragma unroll
    for (int h = 0; h < NH; ++h) {
      const int r0 = 64 * (PP ? h : wg) + 16 * warp4 + (lane >> 2);   // the thread's first row inside the M tile
      const int pw0 = r0 % p.PW, pw1 = (r0 + 8) % p.PW;                // == output w
      const int rr = r0 + 8 * ((lane & 3) >> 1);                         // the row it stores
      const int hr = rr / p.PW;                // h-row inside the M tile
      const int oh = (oh_base + hr) * d + rb;
      const XpRows rows{{pw0 >= d, pw1 >= d}, {pw0 + d < p.PW, pw1 + d < p.PW}, od < p.D && oh < p.H, od, oh,
                        rr - hr * p.PW};
      epilogue_xp<T, N>(p.epi, acc[h], xb, 1 + wg, warp4, lane, d, rows, b);
    }
  };
  tc::mbar_wait(w_bar, 0);
  if (p.ring) {
    // one M tile (one plane, 128 / PW h-rows) per output plane
    const int total = (int)(ring_hi - ring_lo);   // this CTA's planes; ping-pong: plane q belongs to warpgroup q & 1
    int q = 0;
    uint32_t n0 = 0;     // ring index of this unit's first plane (z0 - 1)
    for (long long pos = ring_lo; pos < ring_hi;) {
      int b, ra, rb, th, z0, z1;
      decode_ring(pos, b, ra, rb, th, z0, z1);
      pos += z1 - z0;
      const int K = z1 - z0;
      for (int k = 0; k < K; ++k, ++q) {
        if (PP && (q & 1) != wg) continue;
        if (PP) turn_take(wg, q);
        // cooperative: planes z-1 and z were waited for by plane z-1
        for (uint32_t i = (PP || k == 0 ? 0u : 2u); i < 3u; ++i) {
          const uint32_t n = n0 + (uint32_t)k + i;
          tc::mbar_wait(full_bar + 8u * (n & 3u), (n >> 2) & 1u);
        }
        const uint32_t r = n0 + (uint32_t)k + 1u;                 // ring index of plane z
        for (int g = 0; g < p.n_groups; ++g) {
          const uint32_t slot = (r + (uint32_t)p.grp_dz[g]) & 3u;
          const uint64_t da = tc::make_sdesc(smem_a + slot * (uint32_t)p.a_stage_bytes, RB) +
                              (uint64_t)((p.grp_row[g] + row0) * (RB / 16));
          mma_item<T, N, NH>(acc, da, db_w + (uint64_t)(g * w_step16), a_half, nmma, g == 0);
        }
        if (PP) turn_pass(wg, q + 1 < total);
        tc::wg_wait<0>();
        if (lane == 0) {
          // ring planes n0 + k .. n0 + k + 2 are read by the unit's output planes k - 2 .. k + 2; a plane's slot is
          // free after 8 arrivals, one per MMA warp, each given when its warpgroup's last reader of it has retired
          const uint32_t nz = n0 + (uint32_t)k;
          if (PP) {
            // this warpgroup's next plane is k + 2, which reads only n0 + k + 2 of these; the other warpgroup owns
            // planes k - 1 and k + 1.  A plane the other warpgroup never reads gets both warpgroups' arrivals here
            const bool o_prev = k >= 1, o_next = k + 1 < K;
            tc::mbar_arrive(empty_bar + 8u * (nz & 3u), o_prev ? 1u : 2u);
            tc::mbar_arrive(empty_bar + 8u * ((nz + 1u) & 3u), (o_prev || o_next) ? 1u : 2u);
            if (k + 2 >= K) tc::mbar_arrive(empty_bar + 8u * ((nz + 2u) & 3u), o_next ? 1u : 2u);
          } else {
            tc::mbar_arrive(empty_bar + 8u * (nz & 3u));                          // plane z-1 is done with
            if (k == K - 1) {                                                     // ... and the unit's last two
              tc::mbar_arrive(empty_bar + 8u * ((nz + 1u) & 3u));
              tc::mbar_arrive(empty_bar + 8u * ((nz + 2u) & 3u));
            }
          }
        }
        acc_fence(acc);
        tile_epilogue(b, ra, rb, (z0 + k) * d + ra, th * p.BH);
      }
      n0 += (uint32_t)K + 2u;
    }
    return;
  }
  // box mode: M tile m of CTA tile i is number q = i * nM + m of the CTA; ping-pong: it belongs to warpgroup q & 1
  const int total = ((num_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x) * p.nM;
  int q = 0;
  int s = 0;
  uint32_t ph = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int b, ra, rb, td, th;
    decode(tile, b, ra, rb, td, th);
    const uint64_t da_stage = tc::make_sdesc(smem_a + (uint32_t)s * p.a_stage_bytes, RB);
    for (int m = 0; m < p.nM; ++m, ++q) {
      if (PP && (q & 1) != wg) continue;
      if (PP) turn_take(wg, q);
      tc::mbar_wait(full_bar + 8u * s, ph);
      for (int g = 0; g < p.n_groups; ++g) {
        const uint64_t da = da_stage + (uint64_t)((p.mt_row[m] + p.grp_off[g] + row0) * (RB / 16));
        mma_item<T, N, NH>(acc, da, db_w + (uint64_t)(g * w_step16), a_half, nmma, g == 0);
      }
      if (PP) turn_pass(wg, q + 1 < total);
      tc::wg_wait<0>();
      // the box is free after 8 arrivals, one per MMA warp that read it (ping-pong with nM == 1: one warpgroup)
      if (lane == 0) {
        if (PP) tc::mbar_arrive(empty_bar + 8u * s, p.nM == 2 ? 1u : 2u);
        else if (m == p.nM - 1) tc::mbar_arrive(empty_bar + 8u * s);
      }
      acc_fence(acc);
      tile_epilogue(b, ra, rb, (td * p.BD + p.mt_pd[m] - p.hd) * d + ra, th * p.BH + p.mt_ph0[m] - p.hh);
    }
    if (++s == p.stages) { s = 0; ph ^= 1u; }
  }
}

// The N tiles compiled for each kernel: every width a plan can select.  Plan creation refuses any other N.
template <int... Ns> struct NTiles {
  static constexpr bool has(int n) { return ((n == Ns) || ...); }
};
// per-tap: a divisor of Cout_pad
using TcTiles = NTiles<16, 32, 48, 64, 80, 96, 112, 128, 144, 160, 176, 192, 208, 224, 240, 256>;
using TcxTiles = NTiles<48, 96, 144, 192, 240>;      // 3 * Cout_pad, Cout_pad in {16, ..., 80}
using HaloxTiles = NTiles<48, 96, 144, 192, 240>;    // 3 * Cout_pad, Cout_pad in {16, ..., 80}
using HaloTiles = NTiles<16, 32, 48, 64>;            // Cout_pad

struct SimtParams {
  ConvEpi epi;
  int n_src, n_taps;
  const void* src[OCCD_CONV_MAX_SRC];
  int src_C[OCCD_CONV_MAX_SRC], src_cstride[OCCD_CONV_MAX_SRC], src_coff[OCCD_CONV_MAX_SRC];
  int ID, IH, IW, src_d0;
  int stride[3];
  const void* weight;
  int Cout_pad, Kpad;
  int w_batch_rows;
  signed char tap_src[OCCD_CONV_MAX_TAPS];
  short tap_dz[OCCD_CONV_MAX_TAPS], tap_dy[OCCD_CONV_MAX_TAPS], tap_dx[OCCD_CONV_MAX_TAPS];
};

}  // namespace occd_conv

struct occd_conv_plan {
  int impl;
  int dtype;
  int esize;
  int kc;   // channels per K chunk
  int rb;   // bytes per K chunk row (kc * esize): 128 / 64 / 32 == the swizzle mode
  occd_conv::TcParams tc;
  occd_conv::HaloParams halo;
  occd_conv::HaloxParams halox;
  occd_conv::SimtParams simt;
  CUtensorMap tmA[OCCD_CONV_MAX_SRC];
  CUtensorMap tmW;
  dim3 grid;
  size_t smem;
};

namespace occd_conv {

template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, int threads, size_t smem, cudaStream_t st,
                       Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = dim3((unsigned)threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

template <auto kernel, typename... Args>
int launch_conv(const occd_conv_plan* pl, int pdl, cudaStream_t st, Args&&... args) {
  static bool attr_set[64] = {false};  // per instantiation, per device (the attribute is per device)
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  cudaError_t e = cudaSuccess;
  if (!attr_set[dev]) {
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) { occd_set_last_error(cudaGetErrorString(e)); return OCCD_ERR_CUDA; }
    attr_set[dev] = true;
  }
  if (pdl) {
    e = launch_pdl(kernel, pl->grid, kTcThreads, pl->smem, st, std::forward<Args>(args)...);
    if (e != cudaSuccess) { occd_set_last_error(cudaGetErrorString(e)); return OCCD_ERR_CUDA; }
    return OCCD_OK;
  }
  kernel<<<pl->grid, kTcThreads, pl->smem, st>>>(std::forward<Args>(args)...);
  OCCD_CHECK_LAUNCH();
  return OCCD_OK;
}

// launch the kernel compiled for the plan's N tile and schedule (plan creation has checked that there is one)
template <typename T, int N, bool XP>
int run_tc_n(const occd_conv_plan* pl, cudaStream_t st) {
  if constexpr (ping_pong(N)) {
    if (pl->tc.pp)
      return launch_conv<conv_tc_kernel<T, N, XP, true>>(pl, pl->tc.pdl, st, pl->tc, pl->tmA[0], pl->tmA[1],
                                                         pl->tmA[2], pl->tmW);
  }
  return launch_conv<conv_tc_kernel<T, N, XP, false>>(pl, pl->tc.pdl, st, pl->tc, pl->tmA[0], pl->tmA[1], pl->tmA[2],
                                                      pl->tmW);
}
template <typename T, bool XP, int... Ns>
int run_tc(const occd_conv_plan* pl, cudaStream_t st, NTiles<Ns...>) {
  int rc = OCCD_ERR_UNSUPPORTED;
  (void)((pl->tc.N_tile == Ns && (rc = run_tc_n<T, Ns, XP>(pl, st), true)) || ...);
  if (rc == OCCD_ERR_UNSUPPORTED) occd_set_last_error("occd_conv_run: no kernel compiled for the plan's N tile");
  return rc;
}
template <typename T, int... Ns>
int run_halo(const occd_conv_plan* pl, cudaStream_t st, NTiles<Ns...>) {
  int rc = OCCD_ERR_UNSUPPORTED;
  (void)((pl->halo.N_tile == Ns &&
          (rc = launch_conv<conv_halo_kernel<T, Ns>>(pl, pl->halo.pdl, st, pl->halo, pl->tmA[0], pl->tmW), true)) ||
         ...);
  if (rc == OCCD_ERR_UNSUPPORTED) occd_set_last_error("occd_conv_run: no kernel compiled for the plan's N tile");
  return rc;
}
template <typename T, int N>
int run_halox_n(const occd_conv_plan* pl, cudaStream_t st) {
  if constexpr (ping_pong(N)) {
    if (pl->halox.pp)
      return launch_conv<conv_halox_kernel<T, N, true>>(pl, pl->halox.pdl, st, pl->halox, pl->tmA[0], pl->tmW);
  }
  return launch_conv<conv_halox_kernel<T, N, false>>(pl, pl->halox.pdl, st, pl->halox, pl->tmA[0], pl->tmW);
}
template <typename T, int... Ns>
int run_halox(const occd_conv_plan* pl, cudaStream_t st, NTiles<Ns...>) {
  int rc = OCCD_ERR_UNSUPPORTED;
  (void)((pl->halox.N_tile == Ns && (rc = run_halox_n<T, Ns>(pl, st), true)) || ...);
  if (rc == OCCD_ERR_UNSUPPORTED) occd_set_last_error("occd_conv_run: no kernel compiled for the plan's N tile");
  return rc;
}

// the launchers of one element type: TC / TCX plans (conv_tc_f32.cu, conv_tc_bf16.cu), HALO / HALOX plans
// (conv_halo.cu)
template <typename T>
int run_tc_family(const occd_conv_plan* pl, cudaStream_t st) {
  return pl->impl == OCCD_CONV_IMPL_TCX ? run_tc<T, true>(pl, st, TcxTiles{}) : run_tc<T, false>(pl, st, TcTiles{});
}
template <typename T>
int run_halo_family(const occd_conv_plan* pl, cudaStream_t st) {
  return pl->impl == OCCD_CONV_IMPL_HALOX ? run_halox<T>(pl, st, HaloxTiles{}) : run_halo<T>(pl, st, HaloTiles{});
}
extern template int run_tc_family<float>(const occd_conv_plan*, cudaStream_t);
extern template int run_tc_family<__nv_bfloat16>(const occd_conv_plan*, cudaStream_t);
extern template int run_halo_family<float>(const occd_conv_plan*, cudaStream_t);
extern template int run_halo_family<__nv_bfloat16>(const occd_conv_plan*, cudaStream_t);

}  // namespace occd_conv
