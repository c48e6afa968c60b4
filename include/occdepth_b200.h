/*
 * occdepth_b200 -- C ABI of the H100 (sm_90a) kernels behind the OccDepth forward hot path.
 *
 * The reference (megvii-research/OccDepth) has no FFI: its "operator interface" for this path is the
 * sequence of PyTorch library calls inside occdepth/models/*.py.  Each entry point below names the
 * reference call sequence it replaces (file:line relative to the reference tree).
 *
 * Conventions
 *   - plain pointers + sizes only; all pointers are DEVICE pointers unless stated otherwise
 *   - nothing allocates or synchronises; kernels are enqueued on `stream` (a cudaStream_t cast to void*)
 *   - return 0 on success, an OCCD_ERR_* code otherwise; occd_last_error() returns a static message
 *   - activations are "channels-last": [B][D][H][W][C] with C contiguous (D == 1 for 2-D maps)
 */
#ifndef OCCDEPTH_B200_H
#define OCCDEPTH_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define OCCD_ABI_VERSION 2

/* Activation / GEMM-operand element types.  Every kernel that touches channels-last activations takes one of:    */
/*   OCCD_DTYPE_F32  : fp32 storage holding TF32-representable values (each store rounds to the 10-bit TF32        */
/*                     mantissa, round-to-nearest-away); convolutions run as wgmma .tf32 with fp32          */
/*                     accumulation -- the reference-precision mode (the reference's fp32 nn.Conv*d under PyTorch's */
/*                     CUDA default, TF32 tensor cores)                                                             */
/*   OCCD_DTYPE_BF16 : bf16 storage, wgmma .bf16 -- the throughput mode                                       */
/* One channel "vector" is 8 consecutive channels (32 / 16 bytes): cstride, coff and C are multiples of 8.         */
#define OCCD_DTYPE_F32 0
#define OCCD_DTYPE_BF16 1
/* Element types of class maps and labels (occd_ssc_confusion only); a float32 label is OCCD_DTYPE_F32.           */
#define OCCD_DTYPE_U8 2
#define OCCD_DTYPE_U16 3
#define OCCD_DTYPE_I64 4

/* -------------------------------------------------------------------------------------------- */
/* library                                                                                      */
int occd_abi_version(void);
const char* occd_last_error(void);

/* -------------------------------------------------------------------------------------------- */
/* Stereo-SFA lift (the memory-bound 2D->3D gather)                                              */
/* replaces SFA.forward (occdepth/models/SFA.py:12-106) x len(project_res) as driven by          */
/* OccDepth._forward_2d_to_3d (occdepth/models/OccDepth.py:262-298) and the FlospDepth product   */
/* x3ds * x3ds_depth * 100 (OccDepth.py:339).                                                    */
#define OCCD_SFA_MAX_SCALES 4
#define OCCD_SFA_OUT_F32_PLANAR 0 /* [C][N]   == reference (C,X,Y,Z) fp32                  */
#define OCCD_SFA_OUT_BF16_CL 1    /* [N][cstride] bf16 channels-last (feeds the 3D net)    */
#define OCCD_SFA_OUT_F32_CL 2     /* [N][cstride] fp32 channels-last                       */
#define OCCD_SFA_OUT_TF32_CL 3    /* [N][cstride] fp32 channels-last, values rounded to TF32 (feeds the 3D net) */

typedef struct {
  const void* feat[OCCD_SFA_MAX_SCALES]; /* per scale: [V][h][w][C] channels-last, feat_dtype      */
  int h[OCCD_SFA_MAX_SCALES];
  int w[OCCD_SFA_MAX_SCALES];
  int div[OCCD_SFA_MAX_SCALES]; /* projected_pix // div (floor), OccDepth.py:286-294               */
  long long vstride[OCCD_SFA_MAX_SCALES]; /* elements between consecutive views; 0 = dense (h*w*C)    */
  int n_scales;                 /* 1..4                                                            */
  int n_views;                  /* V, 1..4                                                         */
  int C;                        /* channels, multiple of 4 (f32) / 8 (bf16), <= 256                */
  int feat_dtype;               /* OCCD_DTYPE_*                                                    */
  const int64_t* pix;           /* [V][N][P][2] (x,y) int64 -- batch["projected_pix_s"][i]         */
  const uint8_t* fov;           /* [V][N][P] bool          -- batch["fov_mask_s"][i]               */
  long long N;                  /* voxels                                                          */
  int P;                        /* pattern points per voxel (1 for pattern_id 0)                   */
  void* out;
  int out_mode;    /* OCCD_SFA_OUT_*                                                               */
  int out_cstride; /* channel stride of channels-last outputs (>= C)                               */
  int perm_nyu;    /* 1: voxel n=(i*S2+k)*S1+j is written at (i*S1+j)*S2+k (SFA.py:90-97)          */
  int S1, S2;
  const float* prior; /* optional [N] per-voxel multiplier (FlospDepth occupancy prior), or NULL   */
  float scale_const;  /* out = out * prior * scale_const when prior != NULL                        */
} occd_sfa_params;

int occd_sfa_lift_fwd(const occd_sfa_params* p, void* stream);

/* layout helpers at the module boundary: NCHW/NCDHW fp32 <-> channels-last (f32 or bf16)          */
/* in: [B][C][S] planar fp32, out: [B][S][cstride] channels-last (pad channels zero-filled), each   */
/* value rounded to the activation type: bf16 (round-to-nearest-even) or, for OCCD_DTYPE_F32, TF32  */
/* (cvt.rna.tf32.f32) like every other F32 activation store                                        */
int occd_planar_to_cl(const float* in, void* out, int out_dtype, long long B, int C, long long S,
                      int cstride, void* stream);
/* in: [B][S][cstride] channels-last, out: [B][C][S] planar fp32                                   */
int occd_cl_to_planar(const void* in, int in_dtype, float* out, long long B, int C, long long S,
                      int cstride, void* stream);


/* -------------------------------------------------------------------------------------------- */
/* Generalised N-d convolution as implicit GEMM on wgmma (sm_90a)                              */
/* replaces, with BatchNorm folded into weights/bias and the activation / residual adds fused:    */
/*   nn.Conv3d / nn.Conv2d (+BN +ReLU/LeakyReLU/SiLU)  modules.py:6-48,51-235; DDR.py:51-139;      */
/*     unet2d.py:24-46,65-165; CRP3D.py:22-52; flosp_depth.py:201-257; geffnet 1x1 convs           */
/*   nn.ConvTranspose3d k3 s2 (modules.py:278-296) as 8 sub-pixel phase launches                   */
/*   AvgPool3d + 1x1x1 conv (DDR.py:95-109, modules.py:329-339) as strided multi-tap convs          */
/*   torch.bmm of CRP3D.py:81 (as a 1x1x1 conv whose weights are the mega-context)                 */
/* The GEMM:  M = output positions (tile of 128 = TDxTHxTW box), N = output channels,              */
/*            K = sum over "taps" of the source channels.  A tap = (source tensor, integer offset) */
/* so dilation, padding, multi-branch accumulation (ASPP: three sources, three dilations, one      */
/* accumulator) and concat-free skip connections are all tap lists.                                */
#define OCCD_CONV_MAX_TAPS 81
#define OCCD_CONV_MAX_SRC 3
#define OCCD_CONV_MAX_GROUPS 8
#define OCCD_ACT_NONE 0
#define OCCD_ACT_RELU 1
#define OCCD_ACT_LEAKY 2 /* slope 0.01 */
#define OCCD_ACT_SILU 3
#define OCCD_ACT_SIGMOID 4
#define OCCD_CONV_IMPL_TC 0   /* wgmma + TMA implicit GEMM                                       */
#define OCCD_CONV_IMPL_SIMT 1 /* CUDA-core direct convolution (cross-check / odd shapes)           */
#define OCCD_CONV_IMPL_HALO 2 /* wgmma, halo tile loaded once + row-shifted smem views per tap:    */
                              /* stride-1 {-d,0,d}-tap convs, Cin <= 64, resident weights; returns  */
                              /* OCCD_ERR_UNSUPPORTED from plan_create when the shape does not fit   */
#define OCCD_CONV_IMPL_HALOX 3 /* halo tile for grids whose innermost extent W is 8 / 16 / 32 (one warp row): the   */
                              /* three W taps of each (dz,dy) pair packed into ONE MMA (N = 3*Cout_pad <= 256),  */
                              /* epilogue sums the lane-shifted partials (masked lanes == zero padding); taps in  */
                              /* lexicographic (dz,dy,dx) order, one K chunk, stride 1                           */
#define OCCD_CONV_IMPL_TCX 4  /* per-tap kernel, the three W taps of each (src,dz,dy) group packed into    */
                              /* ONE MMA (N = 3*Cout_pad <= 256): taps ordered as groups of dx = -1,0,+1,   */
                              /* W stride 1, tiles 32 wide (30 outputs), epilogue sums lane-shifted partials */
#define OCCD_CONV_IMPL_AUTO 5 /* the library picks the kernel: the first of HALOX, then HALO (convs of 3..27 {-d,0,d}  */
                              /* taps, Cout_pad <= 64, one K chunk) or else TCX (Cout_pad >= 48), then TC, whose    */
                              /* plan accepts the shape; TC for tap groups and per-image weights.  When all refuse, */
                              /* TC's refusal is returned.  occd_conv_plan_impl reports the kernel chosen           */
#define OCCD_OUT1_NONE 0
#define OCCD_OUT1_CL 1         /* pre-activation copy, channels-last in the plan's dtype            */
#define OCCD_OUT1_BF16_CL OCCD_OUT1_CL
#define OCCD_OUT1_F32_PLANAR 2 /* pre-activation copy, fp32 [B][C][positions] (reference layout)   */
#define OCCD_OUT1_CLASS_U16 3  /* class map, uint16 [B][positions] (positions = ODf*OHf*OWf, the planar mode's      */
                               /* spatial index): the FIRST index of the largest pre-activation value over the Cout */
                               /* channels (a NaN in channel 0 wins, later NaNs are skipped), i.e. exactly what     */
                               /* occd_argmax_classes returns for the OCCD_OUT1_F32_PLANAR logits of the same       */
                               /* descriptor; optional label remap: occd_conv_plan_set_class_lut.  Needs every     */
                               /* channel in one N tile and no tap groups (else OCCD_ERR_UNSUPPORTED)               */
#define OCCD_OUT1_CLASS_U16_CONF 4 /* class map and its confidence, uint16 [2][B][positions]: [0] the map of      */
                                   /* OCCD_OUT1_CLASS_U16, [1] the float16 bits of the top class's softmax          */
                                   /* probability, 1 / sum_c exp(l_c - max l), computed in fp32 and rounded once;   */
                                   /* NaN where a value is NaN or +inf.  The map is bit-identical to mode 3's, the   */
                                   /* lut does not touch the confidence, and the same refusals apply                */
#define OCCD_OUT1_CLASS_U16_PROBS 5 /* class map and every class's probability: uint16 [B][positions], the map of */
                                    /* OCCD_OUT1_CLASS_U16, then float16 [B][Cout][positions] (the planar mode's    */
                                    /* layout), p_c = exp(l_c - m) / s rounded once from fp32, with m and s of mode  */
                                    /* 4 (the probability at the map's class is mode 4's confidence, bit for bit);   */
                                    /* NaN in every channel where a value is NaN or +inf.  The map is bit-identical  */
                                    /* to mode 3's, the lut remaps the map only, and the same refusals apply         */
#define OCCD_CLASS_LUT_MAX 64

typedef struct {
  int src;        /* which source tensor                                                          */
  int dz, dy, dx; /* input coordinate = output coordinate * stride + (dz,dy,dx) (padding folded)  */
} occd_conv_tap;

typedef struct {
  int impl; /* OCCD_CONV_IMPL_*                                                                   */
  int dtype; /* OCCD_DTYPE_*: element type of sources, weights, out0, res1, res2 and a channels-last */
             /* out1.  F32 = TF32 operands (K chunk 32/16/8 channels), BF16 (K chunk 64/32/16)       */
  /* sources: channels-last [B][ID][IH][IW][cstride], channels [coff, coff+C) are read             */
  int n_src;
  const void* src[OCCD_CONV_MAX_SRC];
  int src_C[OCCD_CONV_MAX_SRC];
  int src_cstride[OCCD_CONV_MAX_SRC];
  int src_coff[OCCD_CONV_MAX_SRC];
  int B, ID, IH, IW; /* shared by all sources                                                      */
  int src_d0;        /* plane offset added to every source D coordinate: sources that carry halo   */
                     /* margins ([ID] = slab + 2*margin planes, X-slab multi-GPU partition) are     */
                     /* addressed relative to their interior; 0 for ordinary tensors               */
  int stride[3];     /* (sd, sh, sw)                                                               */
  int n_taps;
  occd_conv_tap taps[OCCD_CONV_MAX_TAPS];
  /* weights: dtype [n_taps][Cout_pad][Kpad], K contiguous, zero padded (F32: pre-rounded to TF32);  */
  /* bias fp32 [Cout_pad]                                                                           */
  const void* weight;
  const float* bias;
  int Cout, Cout_pad, Kpad;
  int weight_per_image; /* 1: weight holds B consecutive [n_taps][Cout_pad][Kpad] sets, image b uses set b   */
                        /* (SE gate folded into the projection weights of each image); TC impl only        */
  /* iteration space of the launch and its mapping to output coordinates: o_full = o*omul + oadd    */
  int OD, OH, OW;
  int omul[3], oadd[3];
  int ODf, OHf, OWf; /* full output grid (== OD,OH,OW unless omul != 1)                            */
  /* out0: channels-last.  v = acc + bias + res1 (+ res2 if !res2_post); out1 = v;                  */
  /*       out0 = act(v) (+ res2 if res2_post)                                                      */
  void* out0;
  int out0_cstride, out0_coff;
  int act;
  int out0_exact;   /* 1: F32 plans store out0 without the TF32 rounding (a tensor that is only ever */
                    /* a residual input, never a GEMM operand); no effect for BF16                   */
  const void* res1; /* channels-last on the full output grid, or NULL                              */
  int res1_cstride, res1_coff;
  const void* res2;
  int res2_cstride, res2_coff;
  int res2_post; /* 1: res2 is added AFTER the activation (modules.py Upsample + skip)            */
  /* out1: optional second output holding the PRE-activation value (or its class map, see above)      */
  int out1_mode;
  void* out1;
  int out1_cstride, out1_coff; /* channels-last mode                                               */
  int out1_C;                  /* planar mode: channels of the planar tensor, written at coff+n    */
  /* tap groups (OCCD_CONV_IMPL_TC only; 0 or 1 = off): n_groups convolutions over the same sources, iteration    */
  /* space, weights tensor and bias in ONE launch.  Group g uses taps [group_tap0[g], group_tap0[g+1]) and writes   */
  /* o_full = o*omul + group_oadd[g] (`oadd` is ignored): the 8 sub-pixel phases of ConvTranspose3d(k3, s2, p1,     */
  /* op1) (modules.py:278-296).  Order the groups by descending tap count.  Needs out1_mode == NONE and at most     */
  /* one residual (res1, or res2 with res2_post).                                                                  */
  int n_groups;
  int group_tap0[OCCD_CONV_MAX_GROUPS + 1];
  int group_oadd[OCCD_CONV_MAX_GROUPS][3];
} occd_conv_desc;

typedef struct occd_conv_plan occd_conv_plan;

/* Validates the descriptor, encodes the TMA tensor maps (pointers are baked in: buffers must stay  */
/* allocated and in place) and picks the tiling.  Host call; needs a current CUDA context for TC.   */
int occd_conv_plan_create(const occd_conv_desc* desc, occd_conv_plan** plan);
int occd_conv_plan_destroy(occd_conv_plan* plan);
int occd_conv_run(const occd_conv_plan* plan, void* stream);
/* class-map plans (OCCD_OUT1_CLASS_U16): lut (HOST pointer, n == Cout <= 64 ints) or NULL: the map holds     */
/* uint16(lut[class]) -- the inv_map remap of occd_argmax_classes -- from the next occd_conv_run on             */
int occd_conv_plan_set_class_lut(occd_conv_plan* plan, const int* lut, int n);
/* introspection for tests / profiling: tile box (TD,TH,TW), N tile, K chunk, stages, grid, and      */
/* info8[7]: TC / TCX plans the number of output tiles; HALO / HALOX plans 1 when the x-packed halo   */
/* kernel runs its plane ring, 0 when it runs the box mainloop (HALO: always 0); SIMT plans 0        */
int occd_conv_plan_info(const occd_conv_plan* plan, int* info8);
/* the kernel (OCCD_CONV_IMPL_*, never _AUTO) the plan runs on                                      */
int occd_conv_plan_impl(const occd_conv_plan* plan, int* impl);
/* how the plan's tensor-core kernel shares M tiles between its two MMA warpgroups (fixed by the N tile):    */
/* ping-pong (whole tiles, alternately: one tile's epilogue runs under the next tile's MMAs) or cooperative   */
/* (both on every tile); OCCD_CONV_SCHED_NONE for the SIMT kernel                                            */
#define OCCD_CONV_SCHED_NONE 0
#define OCCD_CONV_SCHED_COOPERATIVE 1
#define OCCD_CONV_SCHED_PINGPONG 2
int occd_conv_plan_schedule(const occd_conv_plan* plan, int* schedule);
/* debug: plans created while a device buffer ([64][8] int64) is set stamp per-role clock64 values of CTA 0  */
/* into it (tools/conv_trace.py); NULL switches tracing off                                               */
int occd_conv_debug_trace(long long* device_buf);

/* -------------------------------------------------------------------------------------------- */
/* small channels-last helpers                                                                   */
/* nn.Softmax(dim=1) over C<=32 planar fp32 channels, written as a channels-last channel window   */
/* of element type `dtype` (the torch.cat([x_in, softmax(x_occ)]) of modules.py:168-171)           */
int occd_softmax_planar_to_cl(const float* in, void* out, int dtype, long long B, int C, long long S, int cstride,
                              int coff, void* stream);
/* out[b][c][p] = in[b][p][coff+c]: turns a channels-last activation into a K-major GEMM weight  */
/* (the mega-context operand of torch.bmm, CRP3D.py:62-63,81); out rows have leading dim ldo      */
int occd_cl_transpose(const void* in, void* out, int dtype, int B, int P, int C, int cstride, int coff, int ldo,
                      long long out_bstride, void* stream);
/* class map of the callers' post-processing: uint16 out[b][s] = first index of the largest of the   */
/* C planar fp32 logits in[b][c][s] (np.argmax(softmax(ssc_logit), 1).astype(uint16),               */
/* scripts/generate_output.py:94-97; softmax is monotonic, so it is never evaluated).  lut (HOST      */
/* pointer, C ints, C <= 64) or NULL: out = uint16(lut[class]), the inv_map remap of                  */
/* scripts/generate_kitti_submission.py:79 (data/semantic_kitti/io_data.py:99-113)                    */
int occd_argmax_classes(const float* in, void* out, long long B, int C, long long S, const int* lut, void* stream);
/* occd_argmax_classes plus the top class's softmax probability: conf (2-byte aligned) gets the float16 bits of   */
/* max_c softmax(in[b][:][s]) as OCCD_OUT1_CLASS_U16_CONF's second half holds them (NaN where a logit is NaN or  */
/* +inf); out as occd_argmax_classes writes it, lut applied to the class only                                   */
int occd_argmax_classes_conf(const float* in, void* out, void* conf, long long B, int C, long long S, const int* lut,
                             void* stream);
/* occd_argmax_classes plus every class's softmax probability: probs (2-byte aligned) gets the float16 bits of      */
/* softmax(in[b][:][s]) at probs[b][c][s], OCCD_OUT1_CLASS_U16_PROBS's arithmetic with the channels taken in      */
/* ascending order by one thread: the same bytes as a conv epilogue that takes them so, within one float16 ulp of  */
/* one that merges two threads' sums (NaN in every channel where a logit is NaN or +inf); map as                   */
/* occd_argmax_classes writes it, lut applied to the map only                                                      */
int occd_class_probs(const float* logits, void* map, void* probs, long long B, int C, long long S, const int* lut,
                     void* stream);
/* copy a channel window (C % 8 == 0) between channels-last buffers (torch.cat of CRP3D.py:90)    */
int occd_copy_channels(const void* in, void* out, int dtype, long long positions, int C, int in_cstride,
                       int in_coff, int out_cstride, int out_coff, void* stream);

/* -------------------------------------------------------------------------------------------- */
/* Data pipeline (SURVEY 8f row 2): voxel-centre -> pixel indices on the device, bit for bit what     */
/* occdepth/data/utils/helpers.py:94-169 `vox2pix` returns (vox2world fusion.py:201-217, rigid_transform */
/* :518-522 in float64 with OpenBLAS' sequential-FMA dot order, cam2allpixs :236-343).                 */
/* HOST pointers: cam_E 4x4 row-major (first 3 rows used), float64 or -- pose_is_f32 != 0 -- float32: */
/* the reference multiplies in the pose's own precision; cam_k 3x3 float32 row-major (the reference's   */
/* intr.astype(float32)), vox_origin 3 float32, pattern P x 2 int (dx, dy).                             */
/* DEVICE pointers: pix int64 [N][P][2] (x, y), fov bool [N][P], pix_z [N] in the pose's precision or   */
/* NULL; N = X*Y*Z voxels in C order.  pix may be NULL: then only fov (and pix_z, if given) is written, */
/* the same bytes as with pix (a FOV mask alone needs no [N][P][2] index scratch).  fov is required.    */
int occd_vox2pix_fwd(const void* cam_E, int pose_is_f32, const float* cam_k, const float* vox_origin,
                     double voxel_size, int X, int Y, int Z, int img_W, int img_H, const int* pattern, int P,
                     long long* pix, unsigned char* fov, void* pix_z, void* stream);
/* the same for voxels [v0, v0 + n) of that C order only (0 <= v0, 1 <= n, v0 + n <= X*Y*Z), written to pix [n][P][2], */
/* fov [n][P], pix_z [n]: bit for bit that slice of occd_vox2pix_fwd's outputs.  An X-slab [x0, x1) of the grid is  */
/* v0 = x0*Y*Z, n = (x1 - x0)*Y*Z.  pix may be NULL, as for occd_vox2pix_fwd.                                      */
int occd_vox2pix_range_fwd(const void* cam_E, int pose_is_f32, const float* cam_k, const float* vox_origin,
                           double voxel_size, int X, int Y, int Z, int img_W, int img_H, const int* pattern, int P,
                           long long* pix, unsigned char* fov, void* pix_z, long long v0, long long n, void* stream);

/* uint8 RGB HWC image [H0][W0][3] (device) -> float32 CHW [3][H][W] of the top-left H x W crop:     */
/* ((u8 / 255) - mean[c]) / std[c] in float32 = np.array(img, float32) / 255.0, crop, ToTensor,        */
/* Normalize of the datasets (data/semantic_kitti/kitti_dataset.py:164-171,376-402); mean/std: HOST    */
int occd_normalize_rgb_u8(const void* in, float* out, int H0, int W0, int H, int W, const float* mean,
                          const float* stdv, void* stream);
/* the same pre-processing written straight into the forward's channels-last image buffer: n uint8 RGB images     */
/* (device; image i, row y starts at in + i*img_stride + y*row_stride bytes, pixels are 3 contiguous bytes) of     */
/* raw size H0 x W0 -> out [n][H][W][cstride] of out_dtype (OCCD_DTYPE_F32: TF32 values, OCCD_DTYPE_BF16), the top- */
/* left H x W crop.  Bit for bit occd_planar_to_cl(occd_normalize_rgb_u8(image i)) for every image; channels        */
/* [3, cstride) are written as zeros.  cstride: multiple of 8; out 16-byte aligned; mean/std: HOST                  */
int occd_stage_rgb_u8_cl(const void* in, long long img_stride, long long row_stride, int n, int H0, int W0, int H,
                         int W, const float* mean, const float* stdv, void* out, int out_dtype, int cstride,
                         void* stream);
/* the same staging from what cameras and video decoders deliver, bit for bit what OpenCV makes on the host:         */
/*   OCCD_PIX_RGB  as occd_stage_rgb_u8_cl; OCCD_PIX_BGR  pixels B, G, R (cv::cvtColor COLOR_BGR2RGB);                */
/*   OCCD_PIX_NV12 a luma plane of H0 rows, then H0/2 rows of interleaved U, V at in + i*img_stride + uv_offset, both */
/*                 with row_stride (cv::cvtColor COLOR_YUV2RGB_NV12: BT.601 limited range; H0, W0 even).             */
/* maps (DEVICE float32, or NULL): per image [2][H][W] source x then y of every output pixel, image i's at            */
/* maps + i*map_stride floats, 4-byte aligned: the converted image is rectified as cv::remap(INTER_LINEAR,           */
/* BORDER_CONSTANT 0) does, each of the four taps converted first; taps outside H0 x W0 read 0.  The crop H x W is   */
/* then the maps' size, and H0, W0 < 32767.  Without maps it is the top-left H x W of the image, as for RGB.         */
#define OCCD_PIX_RGB 0
#define OCCD_PIX_BGR 1
#define OCCD_PIX_NV12 2
int occd_stage_camera_u8_cl(const void* in, int format, long long img_stride, long long row_stride,
                            long long uv_offset, int n, int H0, int W0, int H, int W, const float* maps,
                            long long map_stride, const float* mean, const float* stdv, void* out, int out_dtype,
                            int cstride, void* stream);
/* NYU's depth map (data/NYU/nyu_dataset.py:42-48 load_depth): out[i] = float32(in[i] / divisor) (the division in   */
/* float64), clamped to [0, max_depth] in float32; in: n uint16 (device), out: n float32 (device)                  */
int occd_depth_u16_to_f32(const void* in, float* out, long long n, double divisor, float max_depth, void* stream);

/* -------------------------------------------------------------------------------------------- */
/* EfficientNet / decoder bandwidth kernels (channels-last 2-D maps of element type `dtype`)       */
/* depthwise KxK (K = 3|5) conv + folded BN + activation; optionally accumulates the per-channel    */
/* spatial SUM of the output into pool[B][C] (squeeze of geffnet SqueezeExcite) as 64-bit FIXED-    */
/* POINT integers in units of 2^-24 (integer atomics: bit-reproducible); explicit top/left padding  */
/* implements TF "SAME" (bottom/right implied by OH/OW). w: fp32 [K*K][C].                          */
int occd_dwconv2d_fwd(const void* in, const float* w, const float* bias, void* out, long long* pool, int dtype,
                      int B, int H, int W, int OH, int OW, int C, int cs_in, int cs_out, int K, int stride,
                      int pad_top, int pad_left, int act, void* stream);
/* same contract, shared-memory-tiled variant: one zero-filled input halo tile per CTA staged with    */
/* cp.async, FMA loop out of shared memory (results equal up to fp32 summation order)                */
int occd_dwconv2d_tiled_fwd(const void* in, const float* w, const float* bias, void* out, long long* pool, int dtype,
                            int B, int H, int W, int OH, int OW, int C, int cs_in, int cs_out, int K, int stride,
                            int pad_top, int pad_left, int act, void* stream);
/* gate[b][c] = sigmoid(W2 silu(W1 (pool[b] 2^-24 / HW) + b1) + b2); zeroes pool. w1 [R][C],       */
/* w2t [R][C]; `gate` must hold B*C + B*R floats (the hidden layer is staged behind the gates)     */
int occd_se_gate_fwd(long long* pool, float inv_hw, const float* w1, const float* b1, const float* w2t,
                     const float* b2, float* gate, int B, int C, int R, void* stream);
/* fused path: squeeze-excite MLP + gate folded into one projection-weight set per image:          */
/* wout[b][row][k] = wdtype(master[row][k] * gate[b][k]) (bf16 / TF32-rounded fp32 GEMM weights);   */
/* hidden: B*R floats of scratch; zeroes pool                                                       */
int occd_se_gate_fold_fwd(long long* pool, float inv_hw, const float* w1, const float* b1, const float* w2t,
                          const float* b2, float* hidden, const float* master, void* wout, int wdtype, int B, int C,
                          int R, int rows, int Kpad, void* stream);
/* out[row][k] = wdtype(master[row][k] * gate[k]): folds x * gate into the next 1x1 conv's weights */
int occd_scale_weights(const float* master, const float* gate, void* out, int wdtype, int rows, int Kpad, int C,
                       void* stream);
/* F.interpolate(mode="bilinear", align_corners=True) of UpSampleBN.forward (unet2d.py:39-44)      */
int occd_upsample_bilinear_ac(const void* in, void* out, int dtype, int B, int h, int w, int OH, int OW, int C,
                              int cs_in, int in_off, int cs_out, int out_off, void* stream);
/* UpSampleBN conv1 with the resize behind the 3x3 taps. y: [B][h][w][cs_y], tap t = (dy+1)*3+(dx+1) */
/* of the coarse per-tap products at channels y_off + t*tap_stride + [0, C).  For every fine pixel p: */
/* out[b][p][c] = act(pre[b][p][c] + sum_t [p+t inside OH x OW] bilinear_ac(Y_t)(p+t)[c]), fp32 sums;  */
/* pre may be NULL or equal to out (in place); act is an OCCD_ACT_* code                            */
int occd_upsample_tapsum_ac(const void* y, const void* pre, void* out, int dtype, int B, int h, int w, int OH,
                            int OW, int C, int cs_y, int y_off, int tap_stride, int cs_pre, int pre_off, int cs_out,
                            int out_off, int act, void* stream);

/* -------------------------------------------------------------------------------------------- */
/* FlospDepth (the "OAD" depth branch, configs with trans_2d_to_3d: "flosp_depth")                */
/* frustum grid generation fused with the trilinear sampling of the depth distribution and of the */
/* all-ones mask volume + per-camera masked mean: FrustumGridGenerator (f2v/frustum_grid_         */
/* generator.py:70-152), bin_depths LID (f2v/utils/depth_utils.py:24-26), normalize_coords        */
/* (f2v/utils/grid_utils.py:4-19), F.grid_sample (f2v/sampler.py:49-65), flosp_depth.py:563-602.   */
/* depth: [V][Dn][h][w] fp32 probabilities; cams: V x 40 floats {T[12], K[12], ida[16]} where T =  */
/* rows 0..2 of lidar_to_cam @ grid_to_lidar; out: [X*Y*Z] fp32 (perm_xzy: written as [X][Z][Y])  */
int occd_frustum_sample_fwd(const float* depth, const float* cams, int V, int Dn, int h, int w, int X, int Y,
                            int Z, float img_w, float img_h, float dmin, float dmax, int mean_mode, float* out,
                            int perm_xzy, void* stream);
/* the infer_mode / ONNX-export route of the same step (OccDepth.py:310-317, flosp_depth.py:564-565, custom  */
/* GridSample symbolic f2v/sampler.py:9-34): the caller supplies the sampling grids, grids: [V][X*Y*Z][3] fp32 */
/* normalised (x, y, z) coordinates of F.grid_sample(bilinear, zeros, align_corners=False)                    */
int occd_grid_sample_prior_fwd(const float* depth, const float* grids, int V, int Dn, int h, int w, int X, int Y,
                               int Z, int mean_mode, float* out, int perm_xzy, void* stream);
/* X windows of the two entry points above, for the X-slab partition of one frame: the prior of planes        */
/* [x0, x0 + Xl) of the X-plane grid, written densely as [Xl*Y*Z] in the local voxel order (perm_xzy: as       */
/* [Xl][Z][Y]).  Voxel coordinates and the index into `grids` ([V][X*Y*Z][3], read at full-grid indices; only  */
/* the window's rows are read) are those of the whole grid, so a window equals the matching slice of the whole  */
/* grid's output bit for bit; x0 = 0, Xl = X is the whole grid.  Refused: Xl < 1, x0 < 0, x0 + Xl > X.         */
int occd_frustum_sample_window_fwd(const float* depth, const float* cams, int V, int Dn, int h, int w, int X, int Y,
                                   int Z, int x0, int Xl, float img_w, float img_h, float dmin, float dmax,
                                   int mean_mode, float* out, int perm_xzy, void* stream);
int occd_grid_sample_prior_window_fwd(const float* depth, const float* grids, int V, int Dn, int h, int w, int X,
                                      int Y, int Z, int x0, int Xl, int mean_mode, float* out, int perm_xzy,
                                      void* stream);
/* softmax over the C planar channels of [B][C][S] fp32 (depth_feature.softmax(1), flosp_depth.py:548) */
int occd_softmax_planar(const float* in, float* out, long long B, int C, long long S, void* stream);
/* out[b] = act(W in[b] + bias): the Linear / 1x1-on-a-vector layers of DepthNet.mlp and SELayer    */
int occd_fc_fwd(const float* in, const float* w, const float* bias, float* out, int B, int n_in, int n_out,
                int act, void* stream);
/* x[b][pos][c] *= gate[b][c] in place (SELayer: x * gate(x_se), flosp_depth.py:195-199)            */
int occd_channel_scale(void* x, const float* gate, int dtype, long long B, long long S, int C, int cstride,
                       void* stream);

/* -------------------------------------------------------------------------------------------- */
/* Evaluation: the SSC metrics' confusion matrix (SSCMetrics.add_batch, loss/sscMetrics.py:70-91, as     */
/* OccDepth.step calls it, OccDepth.py:526-529).  pred: class map of pred_dtype OCCD_DTYPE_U16 (what       */
/* occd_argmax_classes and the class-map epilogue write) or OCCD_DTYPE_I64 (a torch argmax); label: of     */
/* label_dtype OCCD_DTYPE_F32 (KITTI's float32 targets; a value that is not an integer is no class),       */
/* OCCD_DTYPE_U8 (NYU) or OCCD_DTYPE_I64.  Both contiguous, n elements (B frames are one flat array).      */
/* counts: n_classes^2 + 1 int64, ACCUMULATED (never cleared): counts[g*n_classes + p] += voxels with       */
/* label g and prediction p; label 255 is skipped; counts[n_classes^2] += invalid voxels (a label outside  */
/* [0, n_classes) that is not 255, or a prediction outside [0, n_classes) where the label is not 255).     */
/* n_classes <= 64.                                                                                        */
int occd_ssc_confusion(const void* pred, int pred_dtype, const void* label, int label_dtype, long long n,
                       int n_classes, long long* counts, void* stream);

/* -------------------------------------------------------------------------------------------- */
/* Evaluation: the sums behind the losses of the reference's evaluation step (OccDepth.step,              */
/* OccDepth.py:378-533).  Each entry point ADDS its sums (float64, never cleared) to `sums`, so frames,   */
/* batches and later slabs compose by addition; occdepth_b200/losses.py forms the losses from them.       */
/* Per-element math is fp32; each block writes one row of fp64 partials to `work` (work_len doubles, at   */
/* least OCCD_LOSS_WORK_BLOCKS rows of the entry point's sum count), and the rows are added in block      */
/* order: the same inputs give bit-identical sums.                                                        */
#define OCCD_LOSS_WORK_BLOCKS 264
#define OCCD_SSC_LOSS_MAX_CLASSES 64
#define OCCD_SSC_LOSS_MAX_FRUSTUMS 64
#define OCCD_SSC_LOSS_SUMS(C, F) (6 + 3 * (C) + (F) * (C))
/* logits: fp32 [B][C][S] (channel-planar, the ssc_logit layout); label: [B][S] of label_dtype F32, U8 or */
/* I64 (255 = ignore; decoded as occd_ssc_confusion does); weight: fp32 [C].  Over the voxels whose label */
/* is not 255, with t the label and p = softmax(logits) (fp32, max-subtracted):                           */
/*   sums[0] += sum w[t] * (logsumexp - x_t)   sums[1] += sum w[t]     (labels in [0, C) only)            */
/*   sums[2] += #voxels                        sums[3] += #invalid (label outside [0, C) or not integer)  */
/*   sums[6 + c] += sum p_c   sums[6 + C + c] += sum p_c [t == c]   sums[6 + 2C + c] += #[t == c]         */
/* occ_logits / occ_weight (optional, together): fp32 [B][2][S] and [2] against the cascade target        */
/* (labels other than 0 and 255 become 1): sums[4] += sum w_occ[t'] * (logsumexp - x_t'), sums[5] += sum */
/* w_occ[t'].  frustum_masks (optional, n_frustums > 0): uint8 / bool [B][F][S]; over EVERY voxel,        */
/* sums[6 + 3C + f*C + c] += sum mask_f * p_c.  C <= 64, F <= 64.                                         */
int occd_ssc_loss_sums(const float* logits, const void* label, int label_dtype, int B, int n_classes, long long S,
                       const float* weight, const float* occ_logits, const float* occ_weight,
                       const uint8_t* frustum_masks, int n_frustums, double* sums, double* work, long long work_len,
                       void* stream);
/* CRP relation loss (compute_super_CP_multilabel_loss, loss/CRP_loss.py:4-25): P_logits fp32 [B][R][M][N] */
/* against CP_mega_matrices uint8 [B][R][N][M] (note the transpose).  Per relation r, x a logit, y its     */
/* entry:  sums[4r] += sum y softplus(-x)   sums[4r+1] += sum (1-y) softplus(x)   sums[4r+2] += sum y      */
/*         sums[4r+3] += #[y == 0].   R <= 16.                                                             */
#define OCCD_CRP_MAX_RELATIONS 16
int occd_crp_relation_sums(const float* P_logits, const uint8_t* cp, int B, int R, int M, int N, double* sums,
                           double* work, long long work_len, void* stream);
/* Depth classification loss (DepthClsLoss.get_depth_loss, loss/depth_loss.py:14-87): gt fp32 [n][H][W],  */
/* prob fp32 [n][D][h][w].  Per pixel of the (h, w) map: nearest resize of gt to (h*factor, w*factor)     */
/* (PyTorch's index rule and float scale), smallest nonzero depth of the factor x factor patch (1e5 if    */
/* none), bin = trunc((d - (d0 - step)) / step) kept if 0 <= bin < D + 1; the pixel is foreground when    */
/* 1 <= bin <= D:  sums[0] += sum over foreground pixels of sum_d BCE(prob_d, [d == bin - 1]) (logs       */
/* clamped at -100), sums[1] += #foreground.  D <= 1024, factor <= 64.                                    */
#define OCCD_DEPTH_MAX_BINS 1024
int occd_depth_cls_sums(const float* gt, int n_maps, int H, int W, const float* prob, int D, int h, int w,
                        int factor, double d0, double step, double* sums, double* work, long long work_len,
                        void* stream);

/* -------------------------------------------------------------------------------------------- */
/* Occupied-voxel list of a class map: what the visualisation scripts build on the host from `y_pred` and     */
/* `fov_mask_1` (scripts/visualization/kitti_vis_pred.py:9-32, 69-89; kitti_vis_pred_batch.py, NYU_vis_pred.py). */
/* class_map: uint16 [B][N], N = X*Y*Z in C order (what the class-map epilogue / occd_argmax_classes write, with */
/* or without a remap); fov_mask: numpy bool bytes [B][N] or NULL (then every voxel counts as inside).  A voxel is */
/* occupied when empty < class < ignore (the scripts' 0 < class < 255).  Per frame b:                            */
/*   count[b][2]        occupied voxels inside / outside the FOV (the true counts, whatever cap is)               */
/*   hist[b][n_classes] occupied voxels per class id below n_classes (<= 64); larger ids are listed, not counted  */
/*   index[b][cap], cls[b][cap], xyz[b][cap][3] (xyz may be NULL): one row per occupied voxel, the voxels inside   */
/*     the FOV first, then the others, each group in ascending flat index -- the order of numpy's boolean        */
/*     indexing.  Only the first min(cap, total) rows are written; nothing else of the three arrays is touched.   */
/* index = index0 + the voxel's flat index in its frame (index0: the flat index of this map's first voxel in a    */
/* larger grid, e.g. x_lo*Y*Z for an X-slab; 0 otherwise).  xyz = the centre of voxel (x, y, z) = the unravelled  */
/* index: float32(((double)x * voxel_size + voxel_size / 2) + origin[0]) and likewise y, z -- a float64 product    */
/* and sums, rounded once; without `origin` (HOST pointer to 3 doubles, or NULL) these are the rows of            */
/* get_grid_coords([X, Y, Z], voxel_size) cast to float32, for the X == Y grids the scripts call it with.         */
/* work: OCCD_VOXEL_WORK_LEN(B, N) uint32, 8-byte aligned, contents irrelevant before and after.  hist is cleared */
/* by the call.  Three launches on `stream`; the same inputs give the same bytes.                                 */
#define OCCD_VOXEL_TILE 2048
#define OCCD_VOXEL_WORK_LEN(B, N) (2LL * (B) * (((N) + OCCD_VOXEL_TILE - 1) / OCCD_VOXEL_TILE))
int occd_occupied_voxels(const uint16_t* class_map, const uint8_t* fov_mask, int B, int X, int Y, int Z, int index0,
                         int empty, int ignore, int n_classes, int cap, uint32_t* count, uint32_t* hist,
                         int32_t* index, uint16_t* cls, float* xyz, double voxel_size, const double* origin,
                         uint32_t* work, long long work_len, void* stream);

/* -------------------------------------------------------------------------------------------- */
/* Scene maps: frames' class probabilities fused into one persistent voxel map (naive Bayes: the per-voxel       */
/* posterior is proportional to prod_t p_t(c), so its log is a sum of ln p_t(c) and softmax over that sum is the */
/* normalised posterior).  A map is an axis-aligned grid in a caller-chosen map frame: origin (3 float64), voxel */
/* (float64 edge), dims MX x MY x MZ, holding acc fp32 [C][MX][MY][MZ] (summed log-probabilities, start 0) and   */
/* count int32 [MX][MY][MZ] (frames that observed the voxel, start 0).  acc is a logits tensor:                 */
/* occd_argmax_classes / _conf / occd_class_probs read it as [1][C][MX*MY*MZ].                                   */
/* Integrating one frame.  probs: DEVICE float16, C class planes of a frame grid with origin grid_origin (HOST, 3 */
/* float64), edge grid_voxel and dims GX x GY x GZ along its own x, y, z; strides (HOST, 4 long long): elements   */
/* between classes, then between x, y and z neighbours inside a plane (KITTI's output is [x][y][z]; NYU's is      */
/* [x][z][y]).  R (HOST, 12 float64): rows 0..2 of inverse(T), T the rigid 4x4 frame grid's frame -> map frame   */
/* (KITTI: world <- velodyne_t; NYU: map <- world).  For each map voxel (i, j, k) in box (HOST, 6 int: i_lo, i_hi, */
/* j_lo, j_hi, k_lo, k_hi, half-open, inside the map), in float64 without FMA contraction:                       */
/*   c = ((idx + 0.5) * voxel) + origin;  q_r = ((R[r][0] c_x + R[r][1] c_y) + R[r][2] c_z) + R[r][3];           */
/*   f = floor((q - grid_origin) / grid_voxel)                                                                    */
/* The voxel is observed when 0 <= f < (GX, GY, GZ), fov_mask (DEVICE bytes at the class plane's offsets, or     */
/* NULL) is nonzero at f, and none of its C probabilities is NaN.  Then, in fp32 with full-precision logf,       */
/* acc[c] += logf(fmaxf(p_c, min_prob)) for every class, and count += 1.  Nothing else is written.  The box only  */
/* bounds the launch: any box holding every observed voxel gives the same bytes, the whole map included         */
/* ({0, MX, 0, MY, 0, MZ}); the smallest safe one is the frame grid's 8 corners taken to the map frame, their   */
/* bounding box in map indices widened by one voxel and clipped to the map.  n_classes <= 64, min_prob in       */
/* (0, 1].  One launch, one writer per voxel: the same inputs give the same bytes.                               */
int occd_scene_map_integrate(float* acc, int32_t* count, int n_classes, int MX, int MY, int MZ, double voxel,
                             const double* origin, const void* probs, const long long* strides,
                             const uint8_t* fov_mask, int GX, int GY, int GZ, const double* grid_origin,
                             double grid_voxel, const double* R, float min_prob, const int* box, void* stream);
/* Shift by whole voxels d (HOST, 3 int): voxel idx of (acc_out, count_out) is voxel idx + d of (acc, count), and */
/* voxels that come into view hold acc = 0, count = 0.  Out of place (the outputs must be other buffers of the    */
/* same shape); the caller moves the origin by d * voxel.  One launch.                                           */
int occd_scene_map_shift(const float* acc, const int32_t* count, float* acc_out, int32_t* count_out, int n_classes,
                         int MX, int MY, int MZ, const int* d, void* stream);
/* map (uint16 [n], e.g. occd_argmax_classes of acc) = unknown (a uint16 id) wherever count == 0: an unobserved */
/* voxel's acc is all zero and would read as class 0.  One launch.                                               */
int occd_scene_map_mark_unobserved(void* map, const int32_t* count, long long n, int unknown, void* stream);

/* -------------------------------------------------------------------------------------------- */
/* Camera views: each pixel's first visible voxel in a class map, as the camera sees it (the views the           */
/* visualisation scripts draw from, scripts/visualization/kitti_vis_pred.py, NYU_vis_pred.py).  class_map: DEVICE */
/* uint16 [B][GX*GY*GZ] (e.g. what occd_model_run_frames or occd_argmax_classes wrote, or a scene map's classes); */
/* the grid's x, y, z have dims GX, GY, GZ, corner origin (HOST, 3 float64) and edge voxel; strides (HOST, 3     */
/* long long): elements between x, y and z neighbours inside one map (KITTI [x][y][z]: {GY*GZ, GZ, 1}; NYU        */
/* [x][z][y]: {GZ*GY, 1, GY}).  cameras (HOST, B*V*12 float64): camera v of map b at (b*V + v)*12, M row-major   */
/* (3x3) then o (3): M = R^-1 K^-1 and o = -R^-1 t for E = [R | t] taking the grid frame to the camera frame     */
/* (KITTI T_velo_2_cam, NYU world -> cam; R^-1 = R^T for a rigid E), K with last row (0, 0, 1), so o is the      */
/* camera centre and a ray's parameter t is camera-frame z.  Pixel (u, v), u the column, is the image point (u, v) */
/* (pixel centres at integers, as the reference's cam2pix rounds).  In float64 without FMA contraction:          */
/*   d_r = ((M[r][0] u + M[r][1] v) + M[r][2]);  boundary i of axis a at t_a(i) = ((origin_a + i voxel) - o_a) r_a, */
/*   r_a = 1 / d_a, recomputed from the integer index every time.  An axis with d_a == 0 is never stepped and keeps */
/*   the ray only if origin_a <= o_a < origin_a + G_a voxel.  [t_lo, t_hi]: the slab test over the other axes;     */
/*   t0 = max(t_lo, near), t_end = min(t_hi, far), a miss if t0 >= t_end.  First voxel: floor((o + t0 d - origin) */
/*   / voxel) clamped into [0, G_a - 1].  Walk: a voxel of class c with c != empty and c != ignore is the hit;    */
/*   else step the axis with the least next boundary time (ties: x, then y, then z), a miss when that time is >=   */
/*   t_end, when the index leaves the grid, or after GX + GY + GZ + 3 voxels.  Entry time: t0 for the first voxel,  */
/*   max(the previous entry time, the crossed boundary's time) after it.  Every min / max is a plain comparison.  */
/* Outputs [B][V][H][W], each optional (NULL; at least one): cls uint16 = the hit's class (empty on a miss), depth  */
/* float32 = its entry time rounded once (+inf on a miss), index int32 = its element offset in its map            */
/* i*s_x + j*s_y + k*s_z, the flat index occd_occupied_voxels lists (-1 on a miss).  B*V <= 32 cameras travel in  */
/* the kernel parameters (no host-to-device copy: the launch captures into a CUDA graph); at most 2^31 - 1 voxels */
/* per map; near finite >= 0, far > near (+inf allowed).  One launch on `stream`; the same inputs give the same   */
/* bytes.                                                                                                          */
#define OCCD_RENDER_MAX_CAMERAS 32
int occd_render_classes(const uint16_t* class_map, int B, int GX, int GY, int GZ, const long long* strides,
                        const double* origin, double voxel, int V, const double* cameras, int W, int H, int empty,
                        int ignore, double near_t, double far_t, uint16_t* cls, float* depth, int32_t* index,
                        void* stream);
/* Soft camera views: each ray composited front to back through per-voxel class probabilities instead of stopping  */
/* at the first arg-max hit.  probs: DEVICE float16 [B][C][GX*GY*GZ] (what occd_model_run_frames_probs or          */
/* occd_class_probs wrote), class planes contiguous, strides inside a plane as above; 1 <= C <= 64, channel `empty` */
/* (< C) is the probability that the voxel is free.  class_map: DEVICE uint16 [B][GX*GY*GZ] with the same layout, or */
/* NULL; a voxel whose class there is `ignore` is skipped (a scene map's unobserved voxels).  The walk is            */
/* occd_render_classes' (same voxels, order, entry times t, near / far, exit and step cap), and no voxel stops it   */
/* on its class.  Per visited voxel, in float32 with one correctly rounded operation per step (no FMA), T = 1,      */
/* D = -0 (addition's identity, so a lone term keeps its sign) and S[c] = 0 at the start:                           */
/*   skip it if class_map holds `ignore` there; e = p[empty]; skip it if e == 1 (no other channel is read);         */
/*   S[c] = S[c] + T p[c] for every c != empty;  Tn = T e, w = T - Tn, D = D + w (float)t, T = Tn;                   */
/*   stop after it once T <= t_min (t_min in [0, 1); 0 walks every voxel that does not empty T).                    */
/* Voxel i is occupied with probability 1 - p_i(empty), independently, and then has class c with weight p_i(c): T   */
/* is the chance the ray got past every voxel so far, T p_i(c) the chance voxel i is the first occupied one and has */
/* class c, so the channels below sum to 1 when each voxel's probabilities do.  Probabilities are not clamped to    */
/* [0, 1]; NaN propagates.  Outputs [B][V][H][W], each optional (NULL; at least one): opacity float32 = 1 - T;      */
/* depth float32 = D / opacity, the expected entry depth of the first surface (+inf where opacity <= 0); probs_out */
/* float16 [B][V][C][H][W]: channel empty = T (the ray leaves unblocked), channel c = S[c], each rounded once; cls */
/* uint16 = the first largest float32 channel (from channel 0, replaced only on a strict >), remapped to           */
/* uint16(lut[cls]) when lut (HOST, C ints) is given, as occd_argmax_classes remaps.  On one-hot probabilities with */
/* the arg-max map as class_map this is occd_render_classes' cls and depth bit for bit, opacity 1 on a hit and 0   */
/* on a miss.  Cameras, W, H, near and far as occd_render_classes.  One launch on `stream`; the same inputs give   */
/* the same bytes.                                                                                                   */
int occd_render_probs(const void* probs, int B, int C, int GX, int GY, int GZ, const long long* strides,
                      const uint16_t* class_map, int ignore, int empty, const double* origin, double voxel, int V,
                      const double* cameras, int W, int H, double near_t, double far_t, float t_min, const int* lut,
                      uint16_t* cls, float* depth, float* opacity, void* probs_out, void* stream);

/* virtual right view for single-view RGB-D inputs: OccDepth.generate_virtual_img (OccDepth.py:233-260). */
/* in/out: channels-last [B][h][w][cs] of `dtype`; depth: fp32 [dh][dw] of batch item 0; bf_scale = bf / scale_2d */
int occd_virtual_view_fwd(const void* in, void* out, const float* depth, int dtype, int B, int h, int w, int C,
                          int cs_in, int cs_out, int dh, int dw, float bf_scale, void* stream);
/* the same with one depth map per batch item: item b reads the fp32 [dh][dw] map at depth + b * depth_stride floats.  */
/* depth_stride 0 is occd_virtual_view_fwd exactly (item 0's map for every item); otherwise it must be >= dh * dw.    */
int occd_virtual_view_items_fwd(const void* in, void* out, const float* depth, int dtype, int B, int h, int w, int C,
                                int cs_in, int cs_out, int dh, int dw, float bf_scale, long long depth_stride,
                                void* stream);

/* -------------------------------------------------------------------------------------------- */
/* Model files: one camera frame in, the class map out, without Python.  occdepth_b200.deploy.export writes the   */
/* launch list of a model's class-map plan (OccDepth.predict_frame) with its weights and constant tables; the      */
/* calls below load it and replay it (file layout: DESIGN.md section 9).                                          */
#define OCCD_OK 0
#define OCCD_ERR_ARG 1         /* bad argument                                                    */
#define OCCD_ERR_CUDA 2        /* CUDA runtime / driver error                                     */
#define OCCD_ERR_UNSUPPORTED 3 /* e.g. a model file of another format or ABI version              */
#define OCCD_ERR_FORMAT 4      /* not a model file: bad magic, truncated, unknown entry point,    */
                               /* an index or pointer fix-up outside its table or buffer          */
#define OCCD_ERR_IO 5          /* the file cannot be opened or read                              */
#define OCCD_MODEL_FORMAT_VERSION 1
#define OCCD_FRAME_NO_GRAPH 1  /* occd_frame.flags: launch the records one by one, no CUDA graph  */

typedef struct occd_model occd_model;

typedef struct {
  int precision;          /* OCCD_DTYPE_F32 (tf32 plan) or OCCD_DTYPE_BF16                             */
  int dataset;            /* 0 KITTI, 1 NYU                                                            */
  int V;                  /* images per frame                                                          */
  int img_h, img_w;       /* the crop the network sees (raw images may be larger)                     */
  int project_scale;
  int X, Y, Z;            /* the output class map: uint16 [X][Y][Z]                                   */
  int n_classes;
  int has_depth;          /* NYU virtual right view: occd_frame.depth is required                     */
  int depth_h, depth_w;
  int flosp_depth;        /* the FlospDepth prior: camera tables are rebuilt with the calibration     */
  int graph;              /* 1 once the replay has been captured into a CUDA graph                    */
  long long device_bytes; /* device memory the model holds                                            */
  double voxel_size, vox_origin[3], scene_size[3]; /* the default geometry (vox_origin: KITTI's)     */
} occd_model_geom;

typedef struct {
  const void* images;           /* DEVICE uint8 RGB (V, H0, W0, 3); image i, row y at images + i*img_stride + */
  long long img_stride;         /* y*row_stride bytes; pixels are 3 contiguous bytes                         */
  long long row_stride;
  int H0, W0;                   /* raw size, >= the model's img_h x img_w                                   */
  const void* cam_k;            /* HOST: KITTI (V, 3, 3); NYU (3, 3) or NULL for the dataset's default      */
  const void* pose;             /* HOST: KITTI T_velo_2_cam (V, 4, 4); NYU T_world_2_cam (4, 4), the inverse */
                                /* of the camera pose (the dataset's np.linalg.inv(cam_pose))               */
  int calib_f32;                /* cam_k and pose are float32 (1) or float64 (0)                            */
  const double* vox_origin;     /* HOST 3 doubles; required for NYU; NULL: the model's default             */
  const double* scene_size;     /* HOST 3 doubles or NULL: the model's                                      */
  double voxel_size;            /* 0: the model's                                                           */
  const uint16_t* depth;        /* DEVICE uint16 depth PNG (depth_h, depth_w), when geom.has_depth          */
  int depth_h, depth_w;
  int flags;                    /* OCCD_FRAME_*                                                             */
} occd_frame;

/* Reads and validates the whole file before touching a device, then allocates and uploads on the current device   */
/* and creates the convolution plans.  On failure *m is NULL and nothing is left allocated.                          */
int occd_model_load(const char* path, occd_model** m);
int occd_model_info(const occd_model* m, occd_model_geom* geom);
/* One frame -> class_map (DEVICE uint16 [X][Y][Z], the caller's) on `stream`: the images are cropped and normalised */
/* into the plan's input buffer, NYU's depth map converted, and -- when the calibration differs from the last       */
/* frame's, and for every NYU frame -- the projection indices and FlospDepth camera tables are rebuilt.  Then the   */
/* records are replayed: the first run launches them one by one and captures them into a CUDA graph, later runs     */
/* launch the graph (OCCD_FRAME_NO_GRAPH: always one by one).  Allocates nothing per frame; calls on one model must  */
/* not overlap.                                                                                                    */
int occd_model_run_frame(occd_model* m, const occd_frame* frame, uint16_t* class_map, void* stream);
/* occd_model_run_frame plus the class map's confidence: conf (DEVICE float16 [X][Y][Z], 2-byte aligned) gets the  */
/* top class's softmax probability of every voxel (OCCD_OUT1_CLASS_U16_CONF).  OCCD_ERR_UNSUPPORTED for a model    */
/* exported without confidence; occd_model_run_frame on a model exported with it writes the map only.              */
int occd_model_run_frame_conf(occd_model* m, const occd_frame* frame, uint16_t* class_map, void* conf, void* stream);
/* Batched model files (exported from a list of frames, OccDepth.predict_frames): one plan runs up to B frames.     */
/* *batch = B, or 1 for a file exported from one frame.                                                             */
int occd_model_batch(const occd_model* m, int* batch);
/* frames[0..n) -> class_maps + i*X*Y*Z (DEVICE uint16), 1 <= n <= B, and with conf (DEVICE float16, or NULL for the */
/* maps only; OCCD_ERR_UNSUPPORTED for a file without confidence) their confidences at conf + i*X*Y*Z.  Each item    */
/* keeps its own calibration cache; items [n, B) keep what their buffers hold and their results are not copied.  The */
/* B-frame plan runs whatever n is, with the graph rules of occd_model_run_frame.  On an unbatched file this is      */
/* occd_model_run_frame(_conf) with n = 1.                                                                          */
int occd_model_run_frames(occd_model* m, const occd_frame* frames, int n, uint16_t* class_maps, void* conf,
                          void* stream);
/* A frame in any camera format of occd_stage_camera_u8_cl.  frame.images holds the V images as that format lays     */
/* them out: OCCD_PIX_RGB / OCCD_PIX_BGR (V, H0, W0, 3); OCCD_PIX_NV12 each image's luma rows (H0 x W0 bytes,         */
/* H0 and W0 even), its interleaved U, V rows at images + i*img_stride + uv_offset, both with row_stride.  A model    */
/* exported with rectification maps (DESIGN.md section 9) remaps every frame with them; the crop is then the maps'. */
typedef struct {
  occd_frame frame;
  int pixel_format;             /* OCCD_PIX_*                                                               */
  long long uv_offset;          /* NV12: bytes from an image's first luma row to its chroma plane           */
} occd_frame_ex;
/* occd_model_run_frames for frames of any camera format; occd_model_run_frame(s/_conf) are this call with RGB.      */
int occd_model_run_frames_ex(occd_model* m, const occd_frame_ex* frames, int n, uint16_t* class_maps, void* conf,
                             void* stream);
/* occd_model_run_frames_ex plus every class's probability: probs (DEVICE float16 [n][C][X][Y][Z], 2-byte aligned,  */
/* C = occd_model_geom.n_classes) gets the float16 softmax of each item (OCCD_OUT1_CLASS_U16_PROBS).  Only for a    */
/* file exported with probabilities (header flag bit 8), else OCCD_ERR_UNSUPPORTED; the other run calls on such a  */
/* file copy only the map.  On a slab rank other than 0 class_maps and probs may be NULL.                          */
int occd_model_run_frames_probs(occd_model* m, const occd_frame_ex* frames, int n, uint16_t* class_maps, void* probs,
                                void* stream);
/* The occupied-voxel list (occd_occupied_voxels) of the maps the model's last run left on the device: items [0, n)  */
/* of that run (1 <= n <= its n), empty = 0, ignore = 255, the labels remapped when the file has a class LUT.  The  */
/* rows of each item are split by its fov_mask_1: vox2pix of the first view of the item's last staged calibration  */
/* at the output resolution (voxel size / project_scale, the img_w x img_h crop, the centre pixel), computed on the */
/* first listing after that calibration changed and kept otherwise.  NYU has no mask: every row counts as inside.   */
/* Under the X-slab partition rank 0 (also a local group's, after occd_model_run_frame_group) lists the whole       */
/* gathered map; the other ranks hold no map and are refused.  The mask (B x N bytes) and the work array are        */
/* allocated at the first listing and held until occd_model_destroy (counted in device_bytes); nothing is allocated */
/* per call.  Launches on `stream` only, outside the graph; nothing synchronises with the host.                    */
typedef struct {
  int capacity;        /* rows per frame, >= 0                                                                    */
  double voxel_size;   /* edge of an output voxel for xyz; 0: 0.2 for KITTI, 0.08 for NYU                         */
  const double* origin;/* HOST 3 doubles added to the centres, or NULL                                            */
  int32_t* count;      /* DEVICE [n][2] in-FOV / out-of-FOV occupied voxels (the true counts, whatever capacity is) */
  int32_t* hist;       /* DEVICE [n][64] occupied voxels per class id                                             */
  int32_t* index;      /* DEVICE [n][capacity] flat voxel index                                                   */
  uint16_t* cls;       /* DEVICE [n][capacity]                                                                    */
  float* xyz;          /* DEVICE [n][capacity][3] voxel centres, or NULL: no coordinates                          */
} occd_voxel_out;
int occd_model_list_voxels(occd_model* m, int n, const occd_voxel_out* out, void* stream);
int occd_model_destroy(occd_model* m);

/* Model files under the X-slab partition (DESIGN.md section 9): one file per rank, each holding that rank's plan of */
/* predict_frame(slab_output="root").  The ranks' collectives are launches on an occd_comm, created and destroyed   */
/* through include/occdepth_b200_comm.h (NCCL, one rank per process and device; or `world` local ranks on one       */
/* device).  Each is enqueued on `stream` only, so it replays inside a CUDA graph.  A NULL communicator is refused.  */
typedef struct occd_comm occd_comm;
/* halo exchange of one halo-carrying activation: planes [halo, halo + planes) of `base` (plane_bytes each) are      */
/* this rank's; min(halo, planes) planes go to each X-neighbour, and the neighbours' come back into the margins      */
/* [halo - min(halo, planes), halo) and [halo + planes, halo + planes + min(halo, planes))                           */
int occd_comm_halo_exchange(occd_comm* comm, void* base, long long plane_bytes, int halo, int planes, void* stream);
/* dst (world * bytes) = every rank's src (bytes), in rank order                                                     */
int occd_comm_all_gather(occd_comm* comm, const void* src, void* dst, long long bytes, void* stream);
/* rank 0's dst gets every rank's planes: bounds (HOST, 2 * world ints) holds rank r's [lo, hi) at bounds[2r],       */
/* bounds[2r + 1]; src holds this rank's hi - lo planes of plane_bytes each.  dst is ignored on the other ranks.     */
int occd_comm_gather_root(occd_comm* comm, const void* src, void* dst, const int* bounds, long long plane_bytes,
                          void* stream);
/* occd_comm_gather_root of `items` arrays at once: src holds items x (hi - lo) planes, item-major, and rank 0's dst  */
/* items x X planes (X = bounds[2 * world - 1]), so item i of rank r lands at planes [i * X + lo, i * X + hi).  One  */
/* grouped exchange; items == 1 is occd_comm_gather_root                                                           */
int occd_comm_gather_root_items(occd_comm* comm, const void* src, void* dst, const int* bounds, long long plane_bytes,
                                int items, void* stream);

/* FlospDepth's per-camera tables on the host (FlospDepth.camera_tables of occdepth_b200, flosp_depth.py:466-541),  */
/* bit for bit: cams[v] = {rows 0..2 of T[v] @ grid_to_lidar, rows 0..2 of K4[v], identity ida} (40 floats) and      */
/* scaled_pixel_size[v] = |(1/fx, 1/fy)| * 1000, all float32 after casting cam_k (n_cams 3x3) and T (n_cams 4x4)     */
/* from float64, or float32 when inputs_f32.  grid_to_lidar: 16 floats, or NULL with nyu_vox_origin (3 doubles):     */
/* NYU's grid from that origin (extent 4.8 x 4.8 x 2.88 m, 0.08 m voxels / project_scale).  voxel_num (3 ints, or   */
/* NULL) receives the NYU grid's dimensions.  HOST pointers only.                                                    */
int occd_flosp_camera_tables(int n_cams, const void* cam_k, const void* T, int inputs_f32, const float* grid_to_lidar,
                             const double* nyu_vox_origin, int project_scale, float* cams, float* scaled_pixel_size,
                             int* voxel_num);

#ifdef __cplusplus
}
#endif
#endif /* OCCDEPTH_B200_H */
