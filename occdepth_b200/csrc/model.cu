// Model files: load an exported camera-frame class-map plan (occdepth_b200/deploy.py) and replay it from C.
//
// A model file is the launch list of one `Plan` with the plan's buffers: the records name an entry point of this
// library and carry its arguments typed by the header prototype; device pointers are (buffer, offset) pairs into
// one device arena, host structs are byte blobs with pointer fix-ups, convolution plans are created at load.  The
// layout is documented field by field in DESIGN.md section 9; the Python writer is the only producer.
#include "common.cuh"
#include "comm.cuh"
#include "../../include/occdepth_b200.h"
#include "../../include/occdepth_b200_comm.h"

#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <type_traits>
#include <utility>
#include <vector>

namespace {

// ---- replayable entry points: the signature is derived from the header prototype -------------------------------------
union Arg {
  void* p;
  int i;
  long long l;
  float f;
  double d;
};

template <typename T>
struct ArgOf {  // pointer parameters
  static_assert(std::is_pointer<T>::value, "replayable entry points take pointers, int, long long, float, double");
  static constexpr char tag = 'p';
  static T get(const Arg& a) { return static_cast<T>(a.p); }
};
template <>
struct ArgOf<occd_model*> {  // a model handle cannot be stored in a file: only NULL is recorded (the call then refuses)
  static constexpr char tag = 'n';
  static occd_model* get(const Arg&) { return nullptr; }
};
template <>
struct ArgOf<const occd_model*> {
  static constexpr char tag = 'n';
  static const occd_model* get(const Arg&) { return nullptr; }
};
template <>
struct ArgOf<occd_comm*> {  // the model's communicator (tag 'm'), filled in by occd_model_load_slab; or NULL ('n')
  static constexpr char tag = 'm';
  static occd_comm* get(const Arg& a) { return static_cast<occd_comm*>(a.p); }
};
template <>
struct ArgOf<int> {
  static constexpr char tag = 'i';
  static int get(const Arg& a) { return a.i; }
};
template <>
struct ArgOf<long long> {
  static constexpr char tag = 'l';
  static long long get(const Arg& a) { return a.l; }
};
template <>
struct ArgOf<float> {
  static constexpr char tag = 'f';
  static float get(const Arg& a) { return a.f; }
};
template <>
struct ArgOf<double> {
  static constexpr char tag = 'd';
  static double get(const Arg& a) { return a.d; }
};

typedef void (*AnyFn)();
typedef int (*Invoke)(AnyFn, const Arg*);

template <typename... A, size_t... I>
int call_with(int (*f)(A...), const Arg* a, std::index_sequence<I...>) {
  return f(ArgOf<A>::get(a[I])...);
}

template <typename... A>
int invoke(AnyFn fn, const Arg* a) {
  return call_with(reinterpret_cast<int (*)(A...)>(fn), a, std::index_sequence_for<A...>());
}

template <typename... A>
struct Sig {
  static constexpr char str[sizeof...(A) + 1] = {ArgOf<A>::tag..., 0};
};

struct Entry {
  const char* name;
  const char* sig;  // one tag per parameter: p i l f d, m (a communicator)
  AnyFn fn;
  Invoke call;
};

template <typename... A>
Entry entry(const char* name, int (*f)(A...)) {
  return Entry{name, Sig<A...>::str, reinterpret_cast<AnyFn>(f), &invoke<A...>};
}

#define OCCD_ENTRY(fn) entry(#fn, &fn)
// every launch entry point of the header (they end in `void* stream`); occd_conv_run takes a plan by index
const Entry kEntries[] = {
    OCCD_ENTRY(occd_sfa_lift_fwd),          OCCD_ENTRY(occd_planar_to_cl),
    OCCD_ENTRY(occd_cl_to_planar),          OCCD_ENTRY(occd_conv_run),
    OCCD_ENTRY(occd_softmax_planar_to_cl),  OCCD_ENTRY(occd_cl_transpose),
    OCCD_ENTRY(occd_argmax_classes),        OCCD_ENTRY(occd_copy_channels),
    OCCD_ENTRY(occd_vox2pix_fwd),           OCCD_ENTRY(occd_normalize_rgb_u8),
    OCCD_ENTRY(occd_stage_rgb_u8_cl),       OCCD_ENTRY(occd_depth_u16_to_f32),
    OCCD_ENTRY(occd_dwconv2d_fwd),          OCCD_ENTRY(occd_dwconv2d_tiled_fwd),
    OCCD_ENTRY(occd_se_gate_fwd),           OCCD_ENTRY(occd_se_gate_fold_fwd),
    OCCD_ENTRY(occd_scale_weights),         OCCD_ENTRY(occd_upsample_bilinear_ac),
    OCCD_ENTRY(occd_upsample_tapsum_ac),    OCCD_ENTRY(occd_frustum_sample_fwd),
    OCCD_ENTRY(occd_grid_sample_prior_fwd), OCCD_ENTRY(occd_frustum_sample_window_fwd),
    OCCD_ENTRY(occd_grid_sample_prior_window_fwd), OCCD_ENTRY(occd_softmax_planar),
    OCCD_ENTRY(occd_fc_fwd),                OCCD_ENTRY(occd_channel_scale),
    OCCD_ENTRY(occd_ssc_confusion),         OCCD_ENTRY(occd_ssc_loss_sums),
    OCCD_ENTRY(occd_crp_relation_sums),     OCCD_ENTRY(occd_depth_cls_sums),
    OCCD_ENTRY(occd_occupied_voxels),       OCCD_ENTRY(occd_virtual_view_fwd),
    OCCD_ENTRY(occd_vox2pix_range_fwd),     OCCD_ENTRY(occd_argmax_classes_conf),
    OCCD_ENTRY(occd_virtual_view_items_fwd), OCCD_ENTRY(occd_stage_camera_u8_cl),
    OCCD_ENTRY(occd_class_probs),
    // take a stream like the launches (occd_model_batch is bound like them), so they have a signature here; their
    // model handle can only be NULL
    OCCD_ENTRY(occd_model_run_frame_conf),  OCCD_ENTRY(occd_model_run_frames),
    OCCD_ENTRY(occd_model_batch),           OCCD_ENTRY(occd_model_run_frames_ex),
    OCCD_ENTRY(occd_model_list_voxels),     OCCD_ENTRY(occd_model_run_frames_probs),
    // the X-slab partition's collectives: the lock-step runner of a local group stops after each
    OCCD_ENTRY(occd_comm_halo_exchange),    OCCD_ENTRY(occd_comm_all_gather),
    OCCD_ENTRY(occd_comm_gather_root),     OCCD_ENTRY(occd_comm_gather_root_items),
};

bool is_collective(const Entry* e) { return strncmp(e->name, "occd_comm_", 10) == 0; }

const Entry* find_entry(const std::string& name) {
  for (const Entry& e : kEntries)
    if (name == e.name) return &e;
  return nullptr;
}

// ---- the file -----------------------------------------------------------------------------------------------------
const char kMagic[8] = {'O', 'C', 'C', 'D', 'M', 'O', 'D', 'L'};
enum Role { ROLE_IMG, ROLE_PIX, ROLE_FOV, ROLE_PIX_Z, ROLE_DEPTH, ROLE_CAMS, ROLE_SPS, ROLE_CLASSES, N_ROLES };
const char* kRoleNames[N_ROLES] = {"image", "pix", "fov", "pix_z", "depth", "camera tables", "scaled_pixel_size",
                                   "class map"};
enum { FLAG_FLOSP_DEPTH = 1, FLAG_VIRTUAL = 2, FLAG_CONF = 4,   // FLAG_CONF: the class-map role holds the map, then its
       FLAG_SLAB = 16, FLAG_BATCH = 32, FLAG_MAPS = 64,           // float16 confidence (OCCD_OUT1_CLASS_U16_CONF);
       FLAG_PROBS = 256 };                                       // FLAG_PROBS: the class-map role holds the B maps,
                                                                 // then the B x C float16 probability planes
                                                                 // (OCCD_OUT1_CLASS_U16_PROBS);
                                                                 // FLAG_SLAB: one rank's plan, a slab block follows;
                                                                 // FLAG_BATCH: a B-frame plan, a batch block follows
                                                                 // the roles (bit 3 stays unassigned); FLAG_MAPS: a
                                                                 // rectification-maps role follows the roles
const uint32_t kMaxBatch = 1024;
const uint32_t kMaxWorld = 64;
const size_t kArenaAlign = 512;  // the caching allocator's block alignment, which the plans were built with

struct Reader {
  const uint8_t* p;
  size_t n, pos = 0;
  bool ok = true;
  const uint8_t* take(size_t k) {
    if (!ok || k > n - pos) {
      ok = false;
      return nullptr;
    }
    const uint8_t* r = p + pos;
    pos += k;
    return r;
  }
  template <typename T>
  T get() {
    T v;
    const uint8_t* s = take(sizeof(T));
    if (!s) return T(0);
    memcpy(&v, s, sizeof(T));  // little-endian host (x86-64, aarch64)
    return v;
  }
};

struct Fixup {
  uint64_t at;
  uint32_t buffer;
  uint64_t off;
};
struct Blob {
  std::vector<uint8_t> bytes;
  std::vector<Fixup> fix;
};
struct PlanRec {
  uint32_t desc_blob;
  int32_t lut_blob;
  uint32_t lut_n;
};
struct RawArg {
  char tag;
  uint32_t id;  // buffer / blob / plan
  uint64_t off;
  Arg v;
};
struct Record {
  const Entry* e;
  std::vector<RawArg> raw;
  std::vector<Arg> args;     // resolved at load
  std::vector<int> streams;  // argument slots that take the stream
};
struct RoleRef {
  int32_t buffer;
  uint64_t off, len;
};

}  // namespace

struct occd_model {
  // header
  uint32_t precision, dataset, flags, V, img_h, img_w, ps;
  uint32_t grid[3], out[3], P, n_classes, has_lut, depth_h, depth_w, n_cams, img_cstride;
  uint32_t flosp_vn[3];  // FlospDepth's (X, Y, Z) at export, in its own axis order (NYU: not the lift grid's)
  int32_t pattern[64][2], lut[OCCD_CLASS_LUT_MAX];  // the label remap the class-map records apply (informative)
  double voxel_size, vox_origin[3], scene_size[3], virtual_bf;
  float G[16];
  RoleRef roles[N_ROLES];
  RoleRef maps{-1, 0, 0};  // FLAG_MAPS: the staged views' float32 [2][img_h][img_w] rectification maps
  // sections
  std::vector<uint64_t> buf_size, buf_off;
  std::vector<const uint8_t*> buf_data;  // into `file` (nullptr: zeros); only valid while loading
  std::vector<Blob> blobs;
  std::vector<PlanRec> plan_recs;
  std::vector<Record> recs;
  std::vector<uint8_t> file;
  // device state
  uint8_t* arena = nullptr;
  size_t arena_bytes = 0;
  std::vector<occd_conv_plan*> plans;
  cudaStream_t capture_stream = nullptr;
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t graph_exec = nullptr;
  // per batch item: the calibration its index buffers hold (KITTI), and its FlospDepth tables on the host
  uint32_t batch = 1;
  std::vector<std::vector<uint8_t>> calib;
  std::vector<char> calib_valid;
  std::vector<float> cams, sps;
  std::vector<occd_frame_ex> frames_ex;      // the RGB occd_frame_ex of each frame an occd_frame entry point is given
  // the X-slab partition (FLAG_SLAB): this rank, every rank's [lo, hi) planes of the lift grid, this rank's window of
  // the lift's voxel order, the one view it stages (-1: every view) and the whole map's X extent (rank 0's output)
  uint32_t rank = 0, world = 1, map_x = 0;
  std::vector<uint32_t> bounds;
  uint64_t n_lo = 0, n_len = 0;
  int32_t view_sel = -1;
  occd_comm* comm = nullptr;                 // not owned
  std::vector<occd_model*> graph_ranks;      // a local group's graph (held by rank 0): the models it was captured over
  // occd_model_list_voxels: the last run's n (0: none, or it failed), per item the first view's calibration as staged
  // (KITTI) and whether the item's output-resolution FOV mask was computed from it; the mask [batch][N_out] and the
  // listing's work array, allocated at the first listing
  struct ViewCalib {
    int f32;
    double E[16];
    float Ef[16], k32[9];
    double origin[3], scene[3], voxel;
  };
  int last_n = 0;
  std::vector<ViewCalib> view0;
  std::vector<char> mask_valid;
  uint8_t* list_mask = nullptr;
  uint32_t* list_work = nullptr;
  size_t list_bytes = 0;

  bool slab() const { return (flags & FLAG_SLAB) != 0; }
  void* dev(int role) const { return arena + buf_off[roles[role].buffer] + roles[role].off; }
  // item b's part of an input role, which holds `batch` items of equal length
  void* dev(int role, uint32_t b) const { return static_cast<uint8_t*>(dev(role)) + roles[role].len / batch * b; }
  uint64_t map_bytes() const { return (uint64_t)out[0] * out[1] * out[2] * 2; }   // one uint16 class map
  // map-sized planes per item in the class-map role: the map, and its confidence or its C probabilities
  uint64_t maps_per_item() const {
    return (flags & FLAG_PROBS) ? 1 + (uint64_t)n_classes : (flags & FLAG_CONF) ? 2 : 1;
  }
  void* dev_maps() const { return arena + buf_off[maps.buffer] + maps.off; }
};

namespace {

int fail(int code, const std::string& msg) {
  occd_set_last_error(msg.c_str());
  return code;
}

int cuda_fail(cudaError_t e, const char* what) {
  return fail(OCCD_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

// everything below only reads `file`: no device is touched until the whole file has been validated
int parse(occd_model* m) {
  Reader r{m->file.data(), m->file.size()};
  const uint8_t* magic = r.take(8);
  if (!magic || memcmp(magic, kMagic, 8) != 0) return fail(OCCD_ERR_FORMAT, "occd_model_load: not a model file (magic)");
  uint32_t fmt = r.get<uint32_t>(), abi = r.get<uint32_t>();
  if (!r.ok) return fail(OCCD_ERR_FORMAT, "occd_model_load: truncated file (header)");
  if (fmt != OCCD_MODEL_FORMAT_VERSION)
    return fail(OCCD_ERR_UNSUPPORTED, "occd_model_load: model file format version " + std::to_string(fmt) +
                                          ", this library reads version " + std::to_string(OCCD_MODEL_FORMAT_VERSION));
  if (abi != OCCD_ABI_VERSION)
    return fail(OCCD_ERR_UNSUPPORTED, "occd_model_load: model file written for ABI version " + std::to_string(abi) +
                                          ", this library is version " + std::to_string(OCCD_ABI_VERSION));
  m->precision = r.get<uint32_t>();
  m->dataset = r.get<uint32_t>();
  m->flags = r.get<uint32_t>();
  m->V = r.get<uint32_t>();
  m->img_h = r.get<uint32_t>();
  m->img_w = r.get<uint32_t>();
  m->ps = r.get<uint32_t>();
  for (int k = 0; k < 3; ++k) m->grid[k] = r.get<uint32_t>();
  for (int k = 0; k < 3; ++k) m->out[k] = r.get<uint32_t>();
  m->P = r.get<uint32_t>();
  for (int k = 0; k < 64; ++k) {
    m->pattern[k][0] = r.get<int32_t>();
    m->pattern[k][1] = r.get<int32_t>();
  }
  m->voxel_size = r.get<double>();
  for (int k = 0; k < 3; ++k) m->vox_origin[k] = r.get<double>();
  for (int k = 0; k < 3; ++k) m->scene_size[k] = r.get<double>();
  m->n_classes = r.get<uint32_t>();
  m->has_lut = r.get<uint32_t>();
  for (int k = 0; k < OCCD_CLASS_LUT_MAX; ++k) m->lut[k] = r.get<int32_t>();
  m->virtual_bf = r.get<double>();
  m->depth_h = r.get<uint32_t>();
  m->depth_w = r.get<uint32_t>();
  m->n_cams = r.get<uint32_t>();
  for (int k = 0; k < 3; ++k) m->flosp_vn[k] = r.get<uint32_t>();
  for (int k = 0; k < 16; ++k) m->G[k] = r.get<float>();
  m->img_cstride = r.get<uint32_t>();
  for (int k = 0; k < N_ROLES; ++k) {
    m->roles[k].buffer = r.get<int32_t>();
    m->roles[k].off = r.get<uint64_t>();
    m->roles[k].len = r.get<uint64_t>();
  }
  if (m->flags & FLAG_MAPS) {
    m->maps.buffer = r.get<int32_t>();
    m->maps.off = r.get<uint64_t>();
    m->maps.len = r.get<uint64_t>();
    if (!r.ok) return fail(OCCD_ERR_FORMAT, "occd_model_load: truncated file (maps role)");
  }
  if (m->flags & FLAG_BATCH) {
    m->batch = r.get<uint32_t>();
    if (!r.ok) return fail(OCCD_ERR_FORMAT, "occd_model_load: truncated file (batch block)");
    if (m->batch < 1 || m->batch > kMaxBatch)
      return fail(OCCD_ERR_FORMAT, "occd_model_load: batch of " + std::to_string(m->batch) + " frames out of range");
    if (m->flags & FLAG_SLAB)
      return fail(OCCD_ERR_FORMAT, "occd_model_load: a batched file has no X-slab partition (flag bits 4 and 5)");
  }
  if (m->flags & FLAG_SLAB) {
    m->rank = r.get<uint32_t>();
    m->world = r.get<uint32_t>();
    if (!r.ok) return fail(OCCD_ERR_FORMAT, "occd_model_load: truncated file (slab block)");
    if (m->world < 1 || m->world > kMaxWorld || m->rank >= m->world)
      return fail(OCCD_ERR_FORMAT, "occd_model_load: slab rank " + std::to_string(m->rank) + " of " +
                                       std::to_string(m->world) + " out of range");
    m->bounds.resize(2 * m->world);
    for (uint32_t& b : m->bounds) b = r.get<uint32_t>();
    m->n_lo = r.get<uint64_t>();
    m->n_len = r.get<uint64_t>();
    m->view_sel = r.get<int32_t>();
    m->map_x = r.get<uint32_t>();
    if (!r.ok) return fail(OCCD_ERR_FORMAT, "occd_model_load: truncated file (slab block)");
  }
  uint32_t n_buf = r.get<uint32_t>(), n_blob = r.get<uint32_t>(), n_plan = r.get<uint32_t>(),
           n_rec = r.get<uint32_t>();
  if (!r.ok) return fail(OCCD_ERR_FORMAT, "occd_model_load: truncated file (header)");
  if ((m->precision != OCCD_DTYPE_F32 && m->precision != OCCD_DTYPE_BF16) || m->dataset > 1 || m->V < 1 ||
      m->V > 4 || m->P < 1 || m->P > 64 || m->n_cams > 4 || m->img_cstride % 8 != 0)
    return fail(OCCD_ERR_FORMAT, "occd_model_load: header field out of range");
  if (m->flags & ~(uint32_t)(FLAG_FLOSP_DEPTH | FLAG_VIRTUAL | FLAG_CONF | FLAG_SLAB | FLAG_BATCH | FLAG_MAPS |
                             FLAG_PROBS))
    return fail(OCCD_ERR_FORMAT, "occd_model_load: unknown header flag bits");
  if ((m->flags & FLAG_PROBS) && (m->flags & FLAG_CONF))
    return fail(OCCD_ERR_FORMAT, "occd_model_load: header flag bits 2 (confidence) and 8 (probabilities) together: "
                                 "the confidence is the probability at the map's class");
  if ((m->flags & FLAG_PROBS) && (m->n_classes < 1 || m->n_classes > 65535))
    return fail(OCCD_ERR_FORMAT, "occd_model_load: class probabilities need 1 to 65535 classes");
  if (m->slab()) {
    // every rank's slab, in rank order, tiles the lift grid's X planes; this rank's window is its slab's voxels
    const uint64_t plane = (uint64_t)m->grid[1] * m->grid[2];
    bool tiles = m->bounds[0] == 0 && m->bounds[2 * m->world - 1] == m->grid[0];
    for (uint32_t k = 0; k < m->world; ++k)
      tiles = tiles && m->bounds[2 * k + 1] > m->bounds[2 * k] && (k == 0 || m->bounds[2 * k] == m->bounds[2 * k - 1]);
    if (!tiles)
      return fail(OCCD_ERR_FORMAT, "occd_model_load: the slab bounds do not tile the " + std::to_string(m->grid[0]) +
                                       " X planes of the grid");
    if (m->n_lo != m->bounds[2 * m->rank] * plane || m->n_len != (m->bounds[2 * m->rank + 1] - m->bounds[2 * m->rank]) * plane)
      return fail(OCCD_ERR_FORMAT, "occd_model_load: the index window is not rank " + std::to_string(m->rank) +
                                       "'s slab");
    if (m->view_sel < -1 || m->view_sel >= (int32_t)m->V || (m->view_sel >= 0 && (m->flags & FLAG_VIRTUAL)))
      return fail(OCCD_ERR_FORMAT, "occd_model_load: staged view " + std::to_string(m->view_sel) + " outside [-1, " +
                                       std::to_string(m->V) + ")");
    if (m->map_x != m->out[0])
      return fail(OCCD_ERR_FORMAT, "occd_model_load: the slab block's map extent is not the header's");
    if (m->dataset == 1 && (m->flags & FLAG_FLOSP_DEPTH))
      return fail(OCCD_ERR_UNSUPPORTED, "occd_model_load: NYU with the FlospDepth prior has no X-slab partition");
  }
  // counts are bounded by what the file can hold before anything is sized from them
  const size_t left = r.n - r.pos;
  if (n_buf > left / 12 || n_blob > left / 12 || n_plan > left / 12 || n_rec > left / 6)
    return fail(OCCD_ERR_FORMAT, "occd_model_load: truncated file (section counts)");

  m->buf_size.resize(n_buf);
  m->buf_data.resize(n_buf);
  for (uint32_t i = 0; i < n_buf; ++i) {
    uint64_t n = r.get<uint64_t>();
    uint32_t kind = r.get<uint32_t>();
    if (kind > 1) return fail(OCCD_ERR_FORMAT, "occd_model_load: buffer " + std::to_string(i) + ": unknown kind");
    m->buf_size[i] = n;
    m->buf_data[i] = kind ? r.take(n) : nullptr;
    if (!r.ok) return fail(OCCD_ERR_FORMAT, "occd_model_load: truncated file (buffer " + std::to_string(i) + ")");
  }
  auto in_buffer = [&](uint32_t b, uint64_t off, uint64_t len) {
    return b < n_buf && off <= m->buf_size[b] && len <= m->buf_size[b] - off;
  };
  m->blobs.resize(n_blob);
  for (uint32_t i = 0; i < n_blob; ++i) {
    uint64_t n = r.get<uint64_t>();
    const uint8_t* s = r.take(n);
    uint32_t nf = r.get<uint32_t>();
    if (!r.ok || nf > (r.n - r.pos) / 20)
      return fail(OCCD_ERR_FORMAT, "occd_model_load: truncated file (host blob " + std::to_string(i) + ")");
    m->blobs[i].bytes.assign(s, s + n);
    for (uint32_t k = 0; k < nf; ++k) {
      Fixup f;
      f.at = r.get<uint64_t>();
      f.buffer = r.get<uint32_t>();
      f.off = r.get<uint64_t>();
      if (!r.ok) return fail(OCCD_ERR_FORMAT, "occd_model_load: truncated file (fix-ups)");
      if (f.at > n || n - f.at < 8)
        return fail(OCCD_ERR_FORMAT, "occd_model_load: host blob " + std::to_string(i) + ": fix-up outside the blob");
      if (f.buffer >= n_buf)
        return fail(OCCD_ERR_FORMAT, "occd_model_load: host blob " + std::to_string(i) + ": buffer id " +
                                         std::to_string(f.buffer) + " out of range");
      if (f.off >= m->buf_size[f.buffer])
        return fail(OCCD_ERR_FORMAT, "occd_model_load: host blob " + std::to_string(i) + ": fix-up outside buffer " +
                                         std::to_string(f.buffer));
      m->blobs[i].fix.push_back(f);
    }
  }
  m->plan_recs.resize(n_plan);
  for (uint32_t i = 0; i < n_plan; ++i) {
    PlanRec& p = m->plan_recs[i];
    p.desc_blob = r.get<uint32_t>();
    p.lut_blob = r.get<int32_t>();
    p.lut_n = r.get<uint32_t>();
    if (!r.ok) return fail(OCCD_ERR_FORMAT, "occd_model_load: truncated file (convolution plans)");
    if (p.desc_blob >= n_blob || m->blobs[p.desc_blob].bytes.size() != sizeof(occd_conv_desc) ||
        (p.lut_blob >= 0 && ((uint32_t)p.lut_blob >= n_blob || p.lut_n > OCCD_CLASS_LUT_MAX ||
                             m->blobs[p.lut_blob].bytes.size() != 4ull * p.lut_n)))
      return fail(OCCD_ERR_FORMAT, "occd_model_load: convolution plan " + std::to_string(i) + ": bad descriptor");
  }
  m->recs.resize(n_rec);
  for (uint32_t i = 0; i < n_rec; ++i) {
    Record& rec = m->recs[i];
    uint16_t nl = r.get<uint16_t>();
    const uint8_t* s = r.take(nl);
    uint32_t na = r.get<uint32_t>();
    if (!r.ok) return fail(OCCD_ERR_FORMAT, "occd_model_load: truncated file (record " + std::to_string(i) + ")");
    std::string name(reinterpret_cast<const char*>(s), nl);
    rec.e = find_entry(name);
    if (!rec.e) return fail(OCCD_ERR_FORMAT, "occd_model_load: record " + std::to_string(i) +
                                                 ": unknown entry point '" + name + "'");
    if (na != strlen(rec.e->sig))
      return fail(OCCD_ERR_FORMAT, "occd_model_load: record " + std::to_string(i) + " (" + name + "): " +
                                       std::to_string(na) + " arguments, the entry point takes " +
                                       std::to_string(strlen(rec.e->sig)));
    rec.raw.resize(na);
    for (uint32_t k = 0; k < na; ++k) {
      RawArg& a = rec.raw[k];
      a.tag = (char)r.get<uint8_t>();
      a.id = 0;
      a.off = 0;
      a.v.l = 0;
      switch (a.tag) {
        case 'p': a.id = r.get<uint32_t>(); a.off = r.get<uint64_t>(); break;
        case 'h': case 'c': a.id = r.get<uint32_t>(); break;
        case 'i': a.v.i = r.get<int32_t>(); break;
        case 'l': a.v.l = r.get<int64_t>(); break;
        case 'f': a.v.f = r.get<float>(); break;
        case 'd': a.v.d = r.get<double>(); break;
        case 'n': case 's': case 'm': break;
        default: return fail(OCCD_ERR_FORMAT, "occd_model_load: record " + std::to_string(i) + ": bad argument tag");
      }
      if (!r.ok) return fail(OCCD_ERR_FORMAT, "occd_model_load: truncated file (record " + std::to_string(i) + ")");
      const char want = rec.e->sig[k];
      const bool ptr_tag = a.tag == 'p' || a.tag == 'h' || a.tag == 'c' || a.tag == 'n' || a.tag == 's';
      if (want == 'p' ? !ptr_tag : want == 'm' ? (a.tag != 'm' && a.tag != 'n') : a.tag != want)
        return fail(OCCD_ERR_FORMAT, "occd_model_load: record " + std::to_string(i) + " (" + name + "): argument " +
                                         std::to_string(k) + " has the wrong type");
      const std::string where = "occd_model_load: record " + std::to_string(i) + " (" + name + ") argument " +
                                std::to_string(k) + ": ";
      if (a.tag == 'p' && a.id >= n_buf) return fail(OCCD_ERR_FORMAT, where + "buffer id out of range");
      if (a.tag == 'p' && a.off >= m->buf_size[a.id]) return fail(OCCD_ERR_FORMAT, where + "pointer outside its buffer");
      if (a.tag == 'h' && a.id >= n_blob) return fail(OCCD_ERR_FORMAT, where + "host blob id out of range");
      if (a.tag == 'c' && a.id >= n_plan) return fail(OCCD_ERR_FORMAT, where + "convolution plan id out of range");
      if (a.tag == 's') rec.streams.push_back((int)k);
      if (a.tag == 'm' && !m->slab()) return fail(OCCD_ERR_FORMAT, where + "a communicator in a file without the slab partition");
    }
  }
  if (r.pos != r.n) return fail(OCCD_ERR_FORMAT, "occd_model_load: trailing bytes after the records");

  // under the slab partition: the staged view only, this rank's window of the indices, the whole map on rank 0 only;
  // a batched file holds `batch` items of each
  const bool need[N_ROLES] = {true, true, true, true, (m->flags & FLAG_VIRTUAL) != 0,
                              (m->flags & FLAG_FLOSP_DEPTH) != 0, (m->flags & FLAG_FLOSP_DEPTH) != 0, m->rank == 0};
  const uint64_t N = m->slab() ? m->n_len : (uint64_t)m->grid[0] * m->grid[1] * m->grid[2];
  const uint32_t VL = (m->flags & FLAG_VIRTUAL) ? 2 : m->V;
  const uint64_t want_len[N_ROLES] = {
      (uint64_t)(m->view_sel >= 0 ? 1 : m->V) * m->img_h * m->img_w * m->img_cstride *
          (m->precision == OCCD_DTYPE_F32 ? 4 : 2),
      (uint64_t)VL * N * m->P * 16, (uint64_t)VL * N * m->P, N * 8, (uint64_t)m->depth_h * m->depth_w * 4,
      (uint64_t)m->n_cams * 160, (uint64_t)m->n_cams * 4, m->map_bytes() * m->maps_per_item()};
  for (int k = 0; k < N_ROLES; ++k) {
    const RoleRef& ro = m->roles[k];
    if (!need[k]) continue;
    if (ro.buffer < 0 || !in_buffer((uint32_t)ro.buffer, ro.off, ro.len) || ro.len != want_len[k] * m->batch)
      return fail(OCCD_ERR_FORMAT, std::string("occd_model_load: the ") + kRoleNames[k] +
                                       " buffer does not match the header");
  }
  if (m->flags & FLAG_MAPS) {
    // one set of maps for every batch item: the staged views' [2][img_h][img_w] float32, 4-byte aligned in the arena
    const RoleRef& ro = m->maps;
    if (ro.buffer < 0)
      return fail(OCCD_ERR_FORMAT, "occd_model_load: header flag bit 6 (rectification maps) without a maps buffer");
    if (!in_buffer((uint32_t)ro.buffer, ro.off, ro.len) || ro.off % 4 != 0 ||
        ro.len != (uint64_t)(m->view_sel >= 0 ? 1 : m->V) * 2 * m->img_h * m->img_w * 4)
      return fail(OCCD_ERR_FORMAT, "occd_model_load: the rectification maps buffer does not match the header");
  }
  m->frames_ex.assign(m->batch, occd_frame_ex{});
  m->calib.assign(m->batch, std::vector<uint8_t>());
  m->calib_valid.assign(m->batch, 0);
  m->view0.assign(m->batch, occd_model::ViewCalib{});
  m->mask_valid.assign(m->batch, 0);
  m->cams.assign((size_t)m->batch * 4 * 40, 0.f);
  m->sps.assign((size_t)m->batch * 4, 0.f);
  return OCCD_OK;
}

void release(occd_model* m) {
  if (m->graph_exec) cudaGraphExecDestroy(m->graph_exec);
  if (m->graph) cudaGraphDestroy(m->graph);
  for (occd_conv_plan* p : m->plans)
    if (p) occd_conv_plan_destroy(p);
  if (m->arena) cudaFree(m->arena);
  if (m->list_mask) cudaFree(m->list_mask);
  if (m->list_work) cudaFree(m->list_work);
  if (m->capture_stream) cudaStreamDestroy(m->capture_stream);
  delete m;
}

int upload(occd_model* m) {
  size_t total = 0;
  m->buf_off.resize(m->buf_size.size());
  for (size_t i = 0; i < m->buf_size.size(); ++i) {
    m->buf_off[i] = total;
    total += (m->buf_size[i] + kArenaAlign - 1) / kArenaAlign * kArenaAlign;
  }
  cudaError_t e = cudaMalloc(&m->arena, total ? total : kArenaAlign);
  if (e != cudaSuccess) {
    m->arena = nullptr;
    return cuda_fail(e, "occd_model_load: cudaMalloc");
  }
  m->arena_bytes = total ? total : kArenaAlign;
  if ((e = cudaMemset(m->arena, 0, m->arena_bytes)) != cudaSuccess) return cuda_fail(e, "occd_model_load: cudaMemset");
  for (size_t i = 0; i < m->buf_size.size(); ++i)
    if (m->buf_data[i] && m->buf_size[i] &&
        (e = cudaMemcpy(m->arena + m->buf_off[i], m->buf_data[i], m->buf_size[i], cudaMemcpyHostToDevice)) != cudaSuccess)
      return cuda_fail(e, "occd_model_load: upload");
  for (Blob& b : m->blobs)
    for (const Fixup& f : b.fix) {
      void* p = m->arena + m->buf_off[f.buffer] + f.off;
      memcpy(b.bytes.data() + f.at, &p, sizeof(p));
    }
  m->plans.assign(m->plan_recs.size(), nullptr);
  for (size_t i = 0; i < m->plan_recs.size(); ++i) {
    const PlanRec& pr = m->plan_recs[i];
    int rc = occd_conv_plan_create(reinterpret_cast<const occd_conv_desc*>(m->blobs[pr.desc_blob].bytes.data()),
                                   &m->plans[i]);
    if (rc != OCCD_OK) return rc;
    if (pr.lut_blob >= 0 &&
        (rc = occd_conv_plan_set_class_lut(m->plans[i],
                                           reinterpret_cast<const int*>(m->blobs[pr.lut_blob].bytes.data()),
                                           (int)pr.lut_n)) != OCCD_OK)
      return rc;
  }
  for (Record& rec : m->recs) {
    rec.args.resize(rec.raw.size());
    for (size_t k = 0; k < rec.raw.size(); ++k) {
      const RawArg& a = rec.raw[k];
      Arg& v = rec.args[k];
      v = a.v;
      if (a.tag == 'p') v.p = m->arena + m->buf_off[a.id] + a.off;
      if (a.tag == 'h') v.p = m->blobs[a.id].bytes.data();
      if (a.tag == 'c') v.p = m->plans[a.id];
      if (a.tag == 'n' || a.tag == 's') v.p = nullptr;
      if (a.tag == 'm') v.p = m->comm;
    }
  }
  if ((e = cudaStreamCreateWithFlags(&m->capture_stream, cudaStreamNonBlocking)) != cudaSuccess) {
    m->capture_stream = nullptr;
    return cuda_fail(e, "occd_model_load: cudaStreamCreate");
  }
  return OCCD_OK;
}

int call(Record& rec, cudaStream_t st) {
  for (int k : rec.streams) rec.args[k].p = st;
  return rec.e->call(rec.e->fn, rec.args.data());
}

int replay(occd_model* m, cudaStream_t st) {
  for (Record& rec : m->recs) {
    int rc = call(rec, st);
    if (rc != OCCD_OK) return rc;
  }
  return OCCD_OK;
}

// the ranks of a local group on one stream, as parallel.SimSlabGroup.run_lockstep runs them: each rank up to and
// including its next collective (a local collective only posts its arguments), the last rank's post then enqueues that
// collective's copies for all ranks
int replay_lockstep(occd_model* const* ms, int world, cudaStream_t st) {
  std::vector<size_t> pos(world, 0);
  for (;;) {
    int ended = 0;
    for (int r = 0; r < world; ++r) {
      std::vector<Record>& recs = ms[r]->recs;
      bool at_collective = false;
      while (pos[r] < recs.size() && !at_collective) {
        Record& rec = recs[pos[r]++];
        int rc = call(rec, st);
        if (rc != OCCD_OK) {
          occd_comm_reset(ms[0]->comm);
          return rc;
        }
        at_collective = is_collective(rec.e);
      }
      ended += at_collective ? 0 : 1;
    }
    if (ended == world) return OCCD_OK;
    if (ended) {
      occd_comm_reset(ms[0]->comm);
      return fail(OCCD_ERR_ARG, "occd_model_run_frame_group: the ranks' files hold different numbers of collectives");
    }
  }
}

template <typename T>
void load_as_f32(const void* src, int n, float* dst) {
  const T* s = static_cast<const T*>(src);
  for (int i = 0; i < n; ++i) dst[i] = (float)s[i];
}

// the datasets' camera-frame staging (OccDepth._stage_frames) of frame `f` into batch item b: images, depth, and -- for
// a calibration other than the item's last -- the projection indices and the FlospDepth tables
int stage(occd_model* m, const occd_frame_ex* fx, uint32_t b, cudaStream_t st) {
  static const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
  const occd_frame* f = &fx->frame;
  const bool nyu = m->dataset == 1;
  // under the partition's view sharding the rank stages its one view (a slab file's maps are that view's)
  const void* images = static_cast<const uint8_t*>(f->images) + (m->view_sel > 0 ? m->view_sel * f->img_stride : 0);
  const float* maps = (m->flags & FLAG_MAPS) ? static_cast<const float*>(m->dev_maps()) : nullptr;
  int rc = occd_stage_camera_u8_cl(images, fx->pixel_format, f->img_stride, f->row_stride, fx->uv_offset,
                                   m->view_sel >= 0 ? 1 : (int)m->V, f->H0, f->W0, (int)m->img_h, (int)m->img_w, maps,
                                   2LL * m->img_h * m->img_w, mean, stdv, m->dev(ROLE_IMG, b), (int)m->precision,
                                   (int)m->img_cstride, st);
  if (rc != OCCD_OK) return rc;
  if (m->flags & FLAG_VIRTUAL) {
    OCCD_CHECK_ARG(f->depth != nullptr && f->depth_h == (int)m->depth_h && f->depth_w == (int)m->depth_w,
                   "occd_model_run_frame: the model takes a uint16 depth map of the size it was exported with");
    rc = occd_depth_u16_to_f32(f->depth, static_cast<float*>(m->dev(ROLE_DEPTH, b)), (long long)m->depth_h * m->depth_w,
                               8000.0, 10.0f, st);
    if (rc != OCCD_OK) return rc;
  }
  OCCD_CHECK_ARG(f->pose != nullptr && (f->cam_k != nullptr || nyu), "occd_model_run_frame: no calibration");
  OCCD_CHECK_ARG(!nyu || f->vox_origin != nullptr, "occd_model_run_frame: an NYU frame needs vox_origin");
  const int nv = nyu ? 1 : (int)m->V;
  double K[4][9], E[4][16];
  static const double nyu_k[9] = {518.8579, 0, 320, 0, 518.8579, 240, 0, 0, 1};
  for (int v = 0; v < nv; ++v) {
    for (int i = 0; i < 9; ++i)
      K[v][i] = !f->cam_k ? nyu_k[i]
                : f->calib_f32 ? (double)static_cast<const float*>(f->cam_k)[v * 9 + i]
                               : static_cast<const double*>(f->cam_k)[v * 9 + i];
  }
  const double* origin = f->vox_origin ? f->vox_origin : m->vox_origin;
  const double* scene = f->scene_size ? f->scene_size : m->scene_size;
  const double voxel = f->voxel_size > 0 ? f->voxel_size : m->voxel_size;
  if (!nyu) {
    // a KITTI sequence keeps one calibration: the indices and tables stay in place while its bytes do
    const size_t es = f->calib_f32 ? 4 : 8;
    std::vector<uint8_t> key;
    auto put = [&](const void* p, size_t n) {
      const uint8_t* b = static_cast<const uint8_t*>(p);
      key.insert(key.end(), b, b + n);
    };
    put(&f->calib_f32, sizeof(int));
    put(f->cam_k, es * 9 * nv);
    put(f->pose, es * 16 * nv);
    put(origin, 24);
    put(scene, 24);
    put(&voxel, 8);
    if (m->calib_valid[b] && key == m->calib[b]) return OCCD_OK;
    m->calib_valid[b] = 0;
    m->calib[b].swap(key);
    // what occd_model_list_voxels projects the item's FOV mask from: the key above covers all of it, so an unchanged
    // calibration (the early return) keeps both this copy and the mask made from it
    occd_model::ViewCalib& c = m->view0[b];
    c.f32 = f->calib_f32;
    for (int i = 0; i < 16; ++i) {
      if (f->calib_f32) c.Ef[i] = static_cast<const float*>(f->pose)[i];
      else c.E[i] = static_cast<const double*>(f->pose)[i];
    }
    for (int i = 0; i < 9; ++i) c.k32[i] = (float)K[0][i];
    for (int k = 0; k < 3; ++k) {
      c.origin[k] = origin[k];
      c.scene[k] = scene[k];
    }
    c.voxel = voxel;
    m->mask_valid[b] = 0;
  }
  int dims[3];
  for (int k = 0; k < 3; ++k) dims[k] = (int)ceil(((origin[k] + scene[k]) - origin[k]) / voxel);  // volume_dims
  OCCD_CHECK_ARG((long long)dims[0] * dims[1] * dims[2] == (long long)m->grid[0] * m->grid[1] * m->grid[2],
                 "occd_model_run_frame: the geometry gives another voxel count than the model lifts into");
  const float o32[3] = {(float)origin[0], (float)origin[1], (float)origin[2]};
  // the poses vox2pix applies: KITTI's views; NYU's camera, and for the virtual right view T_cam0_2_cam1 @ T
  int f32_pose[4];
  const int n_views = nyu ? ((m->flags & FLAG_VIRTUAL) ? 2 : 1) : nv;
  float Ef[4][16];
  for (int v = 0; v < nv; ++v) {
    f32_pose[v] = f->calib_f32;
    for (int i = 0; i < 16; ++i) {
      if (f->calib_f32) Ef[v][i] = static_cast<const float*>(f->pose)[v * 16 + i];
      else E[v][i] = static_cast<const double*>(f->pose)[v * 16 + i];
    }
  }
  if (nyu && n_views == 2) {
    // np.array([[1,0,0,-0.1],...]) @ T in float64 whatever T's type: rows 1..3 unchanged, row 0 as a dgemm
    // accumulates it, fused multiply-adds over k.  For an inverted rigid pose the last row is exactly (0, 0, 0, 1),
    // so every product is exact and any summation order gives the same row; other last rows follow the FMA order
    for (int i = 0; i < 16; ++i) E[1][i] = f->calib_f32 ? (double)Ef[0][i] : E[0][i];
    for (int j = 0; j < 4; ++j)
      E[1][j] = fma(-0.1, E[1][12 + j], fma(0.0, E[1][8 + j], fma(0.0, E[1][4 + j], E[1][j])));
    f32_pose[1] = 0;
  }
  float k32[4][9];
  for (int v = 0; v < n_views; ++v)
    for (int i = 0; i < 9; ++i) k32[v][i] = (float)K[nyu ? 0 : v][i];
  // under the slab partition every pose's indices of this rank's window [n_lo, n_lo + n_len) only
  const long long N = m->slab() ? (long long)m->n_len : (long long)m->grid[0] * m->grid[1] * m->grid[2];
  for (int v = 0; v < n_views; ++v) {
    const void* pose = f32_pose[v] ? (const void*)Ef[v] : (const void*)E[v];
    long long* pix = static_cast<long long*>(m->dev(ROLE_PIX, b)) + (long long)v * N * m->P * 2;
    unsigned char* fov = static_cast<unsigned char*>(m->dev(ROLE_FOV, b)) + (long long)v * N * m->P;
    if (m->slab())
      rc = occd_vox2pix_range_fwd(pose, f32_pose[v], k32[v], o32, voxel, dims[0], dims[1], dims[2], (int)m->img_w,
                                  (int)m->img_h, &m->pattern[0][0], (int)m->P, pix, fov, m->dev(ROLE_PIX_Z, b),
                                  (long long)m->n_lo, N, st);
    else
      rc = occd_vox2pix_fwd(pose, f32_pose[v], k32[v], o32, voxel, dims[0], dims[1], dims[2], (int)m->img_w,
                            (int)m->img_h, &m->pattern[0][0], (int)m->P, pix, fov, m->dev(ROLE_PIX_Z, b), st);
    if (rc != OCCD_OK) return rc;
  }
  if (m->flags & FLAG_FLOSP_DEPTH) {
    // the intrinsics (the frame's, or NYU's default) in the pose's type: one type flag covers both matrices
    float kf[4 * 9];
    double kd[4 * 9];
    for (int v = 0; v < (int)m->n_cams; ++v)
      for (int i = 0; i < 9; ++i) {
        kd[v * 9 + i] = K[v][i];
        kf[v * 9 + i] = (float)K[v][i];
      }
    int vn[3];
    float* cams = m->cams.data() + (size_t)b * m->n_cams * 40;
    float* sps = m->sps.data() + (size_t)b * m->n_cams;
    rc = occd_flosp_camera_tables((int)m->n_cams, f->calib_f32 ? (const void*)kf : (const void*)kd, f->pose,
                                  f->calib_f32, nyu ? nullptr : m->G, nyu ? origin : nullptr, (int)m->ps, cams, sps,
                                  vn);
    if (rc != OCCD_OK) return rc;
    // NYU re-derives FlospDepth's grid from each frame's origin; it must be the one the plan was built for (in
    // FlospDepth's own axis order, which is not the lift grid's)
    if (nyu)
      OCCD_CHECK_ARG((unsigned)vn[0] == m->flosp_vn[0] && (unsigned)vn[1] == m->flosp_vn[1] &&
                         (unsigned)vn[2] == m->flosp_vn[2],
                     "occd_model_run_frame: this vox_origin gives FlospDepth another voxel grid than the model's");
    cudaError_t e;
    if ((e = cudaMemcpyAsync(m->dev(ROLE_CAMS, b), cams, m->n_cams * 160, cudaMemcpyHostToDevice, st)) != cudaSuccess ||
        (e = cudaMemcpyAsync(m->dev(ROLE_SPS, b), sps, m->n_cams * 4, cudaMemcpyHostToDevice, st)) != cudaSuccess)
      return cuda_fail(e, "occd_model_run_frame: camera tables");
  }
  if (!nyu) m->calib_valid[b] = 1;
  return OCCD_OK;
}

// float32 4x4 product in the order of the CPU sgemm torch calls for `T @ G`: per element, the k = 0 product rounded,
// then fused multiply-adds over k = 1, 2, 3
void matmul4_f32(const float* A, const float* B, float* C) {
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      float acc = A[i * 4] * B[j];
      for (int k = 1; k < 4; ++k) acc = fmaf(A[i * 4 + k], B[k * 4 + j], acc);
      C[i * 4 + j] = acc;
    }
}

}  // namespace

extern "C" int occd_flosp_camera_tables(int n_cams, const void* cam_k, const void* T, int inputs_f32,
                                        const float* grid_to_lidar, const double* nyu_vox_origin, int project_scale,
                                        float* cams, float* scaled_pixel_size, int* voxel_num) {
  OCCD_CHECK_ARG(n_cams >= 1 && n_cams <= 4 && cam_k && T && cams && scaled_pixel_size,
                 "occd_flosp_camera_tables: bad arguments");
  OCCD_CHECK_ARG((grid_to_lidar != nullptr) != (nyu_vox_origin != nullptr) && project_scale >= 1,
                 "occd_flosp_camera_tables: give grid_to_lidar or nyu_vox_origin");
  float G[16];
  if (grid_to_lidar) {
    memcpy(G, grid_to_lidar, sizeof(G));
  } else {
    // FlospDepth._grid_to_lidar: bounds [o, o + extent, 0.08] in float64, corners and sizes in float32
    static const double ext[3] = {4.8, 4.8, 2.88};
    memset(G, 0, sizeof(G));
    G[15] = 1.f;
    for (int k = 0; k < 3; ++k) {
      const double lo = nyu_vox_origin[k], hi = lo + ext[k];
      const int vn = (int)((hi - lo) / 0.08 / project_scale);
      if (voxel_num) voxel_num[k] = vn;
      const float lo32 = (float)lo, hi32 = (float)hi;
      G[k * 5] = (hi32 - lo32) / (float)vn;
      G[k * 4 + 3] = lo32;
    }
  }
  for (int v = 0; v < n_cams; ++v) {
    float K[9], Tv[16], M[16];
    if (inputs_f32) {
      load_as_f32<float>(static_cast<const float*>(cam_k) + v * 9, 9, K);
      load_as_f32<float>(static_cast<const float*>(T) + v * 16, 16, Tv);
    } else {
      load_as_f32<double>(static_cast<const double*>(cam_k) + v * 9, 9, K);
      load_as_f32<double>(static_cast<const double*>(T) + v * 16, 16, Tv);
    }
    // torch.inverse(K4) of an upper-triangular K4 has diagonal 1 / K[i][i] (one IEEE division); torch.norm of the
    // two values is sqrt(fma(b, b, a * a))
    const float a = 1.f / K[0], b = 1.f / K[4];
    scaled_pixel_size[v] = sqrtf(fmaf(b, b, a * a)) * 1000.0f;
    matmul4_f32(Tv, G, M);
    float* c = cams + v * 40;
    for (int i = 0; i < 12; ++i) c[i] = M[i];
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) c[12 + i * 4 + j] = K[i * 3 + j];
      c[12 + i * 4 + 3] = 0.f;
    }
    for (int i = 0; i < 16; ++i) c[24 + i] = (i % 5 == 0) ? 1.f : 0.f;
  }
  return OCCD_OK;
}

namespace {

// reads and validates the file (no device touched), then -- when `accept` agrees -- uploads it
int load(const char* path, occd_comm* comm, occd_model** out, int (*accept)(const occd_model*, const occd_comm*)) {
  *out = nullptr;
  FILE* fp = fopen(path, "rb");
  if (!fp) return fail(OCCD_ERR_IO, std::string("occd_model_load: cannot open ") + path);
  occd_model* m = new occd_model();
  bool io_ok = fseek(fp, 0, SEEK_END) == 0;
  long size = io_ok ? ftell(fp) : -1;
  io_ok = io_ok && size >= 0 && fseek(fp, 0, SEEK_SET) == 0;
  if (io_ok) {
    m->file.resize((size_t)size);
    io_ok = fread(m->file.data(), 1, m->file.size(), fp) == m->file.size();
  }
  fclose(fp);
  if (!io_ok) {
    delete m;
    return fail(OCCD_ERR_IO, std::string("occd_model_load: cannot read ") + path);
  }
  m->comm = comm;
  int rc = parse(m);
  if (rc == OCCD_OK) rc = accept(m, comm);
  if (rc == OCCD_OK) rc = upload(m);
  m->buf_data.clear();
  std::vector<uint8_t>().swap(m->file);
  if (rc != OCCD_OK) {
    std::string msg = occd_last_error();  // release() may overwrite it
    release(m);
    occd_set_last_error(msg.c_str());
    return rc;
  }
  *out = m;
  return OCCD_OK;
}

int accept_plain(const occd_model* m, const occd_comm*) {
  if (m->slab())
    return fail(OCCD_ERR_UNSUPPORTED, "occd_model_load: the file is rank " + std::to_string(m->rank) + " of an X-slab "
                                      "partition over " + std::to_string(m->world) + " ranks; load it with "
                                      "occd_model_load_slab");
  return OCCD_OK;
}

int accept_slab(const occd_model* m, const occd_comm* c) {
  if (!m->slab())
    return fail(OCCD_ERR_UNSUPPORTED, "occd_model_load_slab: the file holds no X-slab partition; load it with "
                                      "occd_model_load");
  int rank, world, kind;
  occd_comm_describe(c, &rank, &world, &kind);
  if ((uint32_t)rank != m->rank || (uint32_t)world != m->world)
    return fail(OCCD_ERR_ARG, "occd_model_load_slab: the file is rank " + std::to_string(m->rank) + " of " +
                                  std::to_string(m->world) + ", the communicator rank " + std::to_string(rank) +
                                  " of " + std::to_string(world));
  return OCCD_OK;
}

}  // namespace

extern "C" int occd_model_load(const char* path, occd_model** out) {
  OCCD_CHECK_ARG(path && out, "occd_model_load: null argument");
  return load(path, nullptr, out, accept_plain);
}

extern "C" int occd_model_load_slab(const char* path, occd_comm* comm, occd_model** out) {
  OCCD_CHECK_ARG(path && comm && out, "occd_model_load_slab: null argument");
  return load(path, comm, out, accept_slab);
}

extern "C" int occd_model_info(const occd_model* m, occd_model_geom* g) {
  OCCD_CHECK_ARG(m && g, "occd_model_info: null argument");
  memset(g, 0, sizeof(*g));
  g->precision = (int)m->precision;
  g->dataset = (int)m->dataset;
  g->V = (int)m->V;
  g->img_h = (int)m->img_h;
  g->img_w = (int)m->img_w;
  g->project_scale = (int)m->ps;
  g->X = (int)m->out[0];
  g->Y = (int)m->out[1];
  g->Z = (int)m->out[2];
  g->n_classes = (int)m->n_classes;
  g->has_depth = (m->flags & FLAG_VIRTUAL) ? 1 : 0;
  g->depth_h = (int)m->depth_h;
  g->depth_w = (int)m->depth_w;
  g->flosp_depth = (m->flags & FLAG_FLOSP_DEPTH) ? 1 : 0;
  g->graph = m->graph_exec ? 1 : 0;
  g->device_bytes = (long long)(m->arena_bytes + m->list_bytes);
  g->voxel_size = m->voxel_size;
  for (int k = 0; k < 3; ++k) {
    g->vox_origin[k] = m->vox_origin[k];
    g->scene_size[k] = m->scene_size[k];
  }
  return OCCD_OK;
}

namespace {

void drop_graph(occd_model* m) {
  if (m->graph_exec) cudaGraphExecDestroy(m->graph_exec);
  if (m->graph) cudaGraphDestroy(m->graph);
  m->graph_exec = nullptr;
  m->graph = nullptr;
}

// replays the records (through `owner`'s graph when there is one) on `stream`: rep(stream) launches them one by one
template <typename Replay>
int execute(occd_model* owner, int flags, cudaStream_t st, Replay rep) {
  int rc;
  cudaError_t e;
  if ((flags & OCCD_FRAME_NO_GRAPH) || owner->graph_exec == nullptr) {
    if ((rc = rep(st)) != OCCD_OK) return rc;
    if (!(flags & OCCD_FRAME_NO_GRAPH)) {
      // the first run is also the warm-up (module loading, function attributes); the graph is captured after it
      if ((e = cudaStreamBeginCapture(owner->capture_stream, cudaStreamCaptureModeThreadLocal)) != cudaSuccess)
        return cuda_fail(e, "occd_model_run_frame: cudaStreamBeginCapture");
      cudaGraph_t graph = nullptr;
      rc = rep(owner->capture_stream);
      e = cudaStreamEndCapture(owner->capture_stream, &graph);
      if (rc == OCCD_OK && e == cudaSuccess && (e = cudaGraphInstantiate(&owner->graph_exec, graph, 0)) == cudaSuccess) {
        owner->graph = graph;
      } else {
        // nothing half-made stays behind: a later run captures afresh
        owner->graph_exec = nullptr;
        if (graph) cudaGraphDestroy(graph);
        if (rc != OCCD_OK) return rc;
        return cuda_fail(e, "occd_model_run_frame: graph capture");
      }
    }
  } else if ((e = cudaGraphLaunch(owner->graph_exec, st)) != cudaSuccess) {
    return cuda_fail(e, "occd_model_run_frame: cudaGraphLaunch");
  }
  return OCCD_OK;
}

// stages frames[0..n) into items [0, n) and replays the records (through the graph when there is one) on `stream`
int run_records(occd_model* m, const occd_frame_ex* frames, int n, cudaStream_t st) {
  if (m->comm) {
    int rank, world, kind;
    occd_comm_describe(m->comm, &rank, &world, &kind);
    if (kind == OCCD_COMM_LOCAL)
      return fail(OCCD_ERR_UNSUPPORTED, "occd_model_run_frame: a model on a local communicator runs with its group "
                                        "through occd_model_run_frame_group");
  }
  m->last_n = 0;  // a failed run leaves nothing to list
  for (int i = 0; i < n; ++i) {
    int rc = stage(m, &frames[i], (uint32_t)i, st);
    if (rc != OCCD_OK) return rc;
  }
  int rc = execute(m, frames[0].frame.flags, st, [m](cudaStream_t s) { return replay(m, s); });
  if (rc == OCCD_OK) m->last_n = n;
  return rc;
}

// the occd_frame entry points: frames[0..n) as RGB occd_frame_ex, in the model's own array (nothing allocated)
const occd_frame_ex* rgb_frames(occd_model* m, const occd_frame* frames, int n) {
  for (int i = 0; i < n; ++i) m->frames_ex[i] = occd_frame_ex{frames[i], OCCD_PIX_RGB, 0};
  return m->frames_ex.data();
}

// the whole maps of items [0, n) (and their confidences or probabilities) of a model whose plan outputs them: every
// unpartitioned model, rank 0 of a slab.  The class-map role is [B][map], [2][B][map] with the confidence, or
// [B][map] then [B][C][map] with the probabilities
int copy_out(const occd_model* m, uint16_t* class_map, void* conf, int n, cudaStream_t st, const char* what,
             void* probs = nullptr) {
  if (m->rank != 0) return OCCD_OK;
  const char* roles = static_cast<const char*>(m->dev(ROLE_CLASSES));
  cudaError_t e;
  if ((e = cudaMemcpyAsync(class_map, roles, m->map_bytes() * n, cudaMemcpyDeviceToDevice, st)) != cudaSuccess)
    return cuda_fail(e, (std::string(what) + ": class map copy").c_str());
  if (conf && (e = cudaMemcpyAsync(conf, roles + m->map_bytes() * m->batch, m->map_bytes() * n,
                                   cudaMemcpyDeviceToDevice, st)) != cudaSuccess)
    return cuda_fail(e, (std::string(what) + ": confidence copy").c_str());
  if (probs && (e = cudaMemcpyAsync(probs, roles + m->map_bytes() * m->batch, m->map_bytes() * m->n_classes * n,
                                    cudaMemcpyDeviceToDevice, st)) != cudaSuccess)
    return cuda_fail(e, (std::string(what) + ": probabilities copy").c_str());
  return OCCD_OK;
}

}  // namespace

extern "C" int occd_model_run_frame(occd_model* m, const occd_frame* f, uint16_t* class_map, void* stream) {
  OCCD_CHECK_ARG(m && f && f->images && (class_map || m->rank != 0), "occd_model_run_frame: null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = run_records(m, rgb_frames(m, f, 1), 1, st);
  if (rc != OCCD_OK) return rc;
  return copy_out(m, class_map, nullptr, 1, st, "occd_model_run_frame");
}

extern "C" int occd_model_run_frame_conf(occd_model* m, const occd_frame* f, uint16_t* class_map, void* conf,
                                         void* stream) {
  OCCD_CHECK_ARG(m && f && f->images && ((class_map && conf) || m->rank != 0),
                 "occd_model_run_frame_conf: null argument");
  if (!(m->flags & FLAG_CONF)) {
    occd_set_last_error("occd_model_run_frame_conf: the model was exported without confidence");
    return OCCD_ERR_UNSUPPORTED;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = run_records(m, rgb_frames(m, f, 1), 1, st);
  if (rc != OCCD_OK) return rc;
  return copy_out(m, class_map, conf, 1, st, "occd_model_run_frame_conf");
}

extern "C" int occd_model_batch(const occd_model* m, int* batch) {
  OCCD_CHECK_ARG(m && batch, "occd_model_batch: null argument");
  *batch = (int)m->batch;
  return OCCD_OK;
}

namespace {

int run_frames(const char* who, occd_model* m, const occd_frame* frames, const occd_frame_ex* frames_ex, int n,
               uint16_t* class_maps, void* conf, void* stream, void* probs = nullptr) {
  const std::string w(who);
  if (!(m && (frames || frames_ex) && (class_maps || m->rank != 0))) return fail(OCCD_ERR_ARG, w + ": null argument");
  if (n < 1 || (uint32_t)n > m->batch)
    return fail(OCCD_ERR_ARG, w + ": " + std::to_string(n) + " frames, the model runs 1 to " +
                                  std::to_string(m->batch));
  for (int i = 0; i < n; ++i)
    if (!(frames ? frames[i].images : frames_ex[i].frame.images)) return fail(OCCD_ERR_ARG, w + ": a frame without images");
  if (conf && !(m->flags & FLAG_CONF)) return fail(OCCD_ERR_UNSUPPORTED, w + ": the model was exported without confidence");
  if (probs && !(m->flags & FLAG_PROBS))
    return fail(OCCD_ERR_UNSUPPORTED, w + ": the model was exported without probabilities");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = run_records(m, frames ? rgb_frames(m, frames, n) : frames_ex, n, st);
  if (rc != OCCD_OK) return rc;
  return copy_out(m, class_maps, conf, n, st, who, probs);
}

}  // namespace

extern "C" int occd_model_run_frames(occd_model* m, const occd_frame* frames, int n, uint16_t* class_maps, void* conf,
                                     void* stream) {
  return run_frames("occd_model_run_frames", m, frames, nullptr, n, class_maps, conf, stream);
}

extern "C" int occd_model_run_frames_ex(occd_model* m, const occd_frame_ex* frames, int n, uint16_t* class_maps,
                                        void* conf, void* stream) {
  return run_frames("occd_model_run_frames_ex", m, nullptr, frames, n, class_maps, conf, stream);
}

extern "C" int occd_model_run_frames_probs(occd_model* m, const occd_frame_ex* frames, int n, uint16_t* class_maps,
                                           void* probs, void* stream) {
  if (m && !probs && m->rank == 0) return fail(OCCD_ERR_ARG, "occd_model_run_frames_probs: null argument");
  if (m && !(m->flags & FLAG_PROBS))
    return fail(OCCD_ERR_UNSUPPORTED, "occd_model_run_frames_probs: the model was exported without probabilities");
  return run_frames("occd_model_run_frames_probs", m, nullptr, frames, n, class_maps, nullptr, stream, probs);
}

namespace {

int run_frame_group(const char* who, occd_model* const* ms, int world, const occd_frame* f, uint16_t* class_map,
                    void* conf, void* probs, void* stream) {
  const std::string w(who);
  if (!(ms && world >= 1 && f && f->images && class_map)) return fail(OCCD_ERR_ARG, w + ": null argument");
  for (int r = 0; r < world; ++r) {
    if (!(ms[r] && ms[r]->comm))
      return fail(OCCD_ERR_ARG, w + ": every rank's model, loaded with a local communicator, is needed");
    int rank, wr, kind;
    occd_comm_describe(ms[r]->comm, &rank, &wr, &kind);
    if (!(kind == OCCD_COMM_LOCAL && rank == r && wr == world &&
          occd_comm_group(ms[r]->comm) == occd_comm_group(ms[0]->comm)))
      return fail(OCCD_ERR_ARG, w + ": models[r] must be rank r of one local group of `world` ranks");
  }
  if (conf && !(ms[0]->flags & FLAG_CONF)) return fail(OCCD_ERR_UNSUPPORTED, w + ": the model was exported without confidence");
  if (probs && !(ms[0]->flags & FLAG_PROBS))
    return fail(OCCD_ERR_UNSUPPORTED, w + ": the model was exported without probabilities");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const occd_frame_ex fx{*f, OCCD_PIX_RGB, 0};
  for (int r = 0; r < world; ++r) ms[r]->last_n = 0;
  for (int r = 0; r < world; ++r) {
    int rc = stage(ms[r], &fx, 0, st);
    if (rc != OCCD_OK) return rc;
  }
  // rank 0 holds the group's graph; it is captured afresh when the group's models change
  occd_model* owner = ms[0];
  if (owner->graph_exec && owner->graph_ranks != std::vector<occd_model*>(ms, ms + world)) drop_graph(owner);
  const bool capture = !(f->flags & OCCD_FRAME_NO_GRAPH) && owner->graph_exec == nullptr;
  int rc = execute(owner, f->flags, st, [ms, world](cudaStream_t s) { return replay_lockstep(ms, world, s); });
  if (rc != OCCD_OK) return rc;
  if (capture && owner->graph_exec) owner->graph_ranks.assign(ms, ms + world);
  for (int r = 0; r < world; ++r) ms[r]->last_n = 1;
  return copy_out(owner, class_map, conf, 1, st, who, probs);
}

}  // namespace

extern "C" int occd_model_run_frame_group(occd_model* const* ms, int world, const occd_frame* f, uint16_t* class_map,
                                          void* conf, void* stream) {
  return run_frame_group("occd_model_run_frame_group", ms, world, f, class_map, conf, nullptr, stream);
}

extern "C" int occd_model_run_frame_group_probs(occd_model* const* ms, int world, const occd_frame* f,
                                                uint16_t* class_map, void* probs, void* stream) {
  if (!probs) return fail(OCCD_ERR_ARG, "occd_model_run_frame_group_probs: null argument");
  return run_frame_group("occd_model_run_frame_group_probs", ms, world, f, class_map, nullptr, probs, stream);
}

namespace {

// item b's fov_mask_1 (KITTI): vox2pix of its first view at the output resolution, centre pixel, into list_mask
int fov_mask_1(occd_model* m, uint32_t b, long long N, cudaStream_t st) {
  const occd_model::ViewCalib& c = m->view0[b];
  const double voxel = c.voxel / m->ps;
  int dims[3];
  for (int k = 0; k < 3; ++k) dims[k] = (int)ceil(((c.origin[k] + c.scene[k]) - c.origin[k]) / voxel);  // volume_dims
  if ((long long)dims[0] * dims[1] * dims[2] != N)
    return fail(OCCD_ERR_ARG, "occd_model_list_voxels: item " + std::to_string(b) + "'s geometry gives " +
                                  std::to_string((long long)dims[0] * dims[1] * dims[2]) +
                                  " voxels at the output resolution, the model predicts " + std::to_string(N));
  const float o32[3] = {(float)c.origin[0], (float)c.origin[1], (float)c.origin[2]};
  static const int centre[2] = {0, 0};  // the datasets' pattern 0
  return occd_vox2pix_fwd(c.f32 ? (const void*)c.Ef : (const void*)c.E, c.f32, c.k32, o32, voxel, dims[0], dims[1],
                          dims[2], (int)m->img_w, (int)m->img_h, centre, 1, nullptr, m->list_mask + (size_t)b * N,
                          nullptr, st);
}

}  // namespace

extern "C" int occd_model_list_voxels(occd_model* m, int n, const occd_voxel_out* out, void* stream) {
  OCCD_CHECK_ARG(m && out, "occd_model_list_voxels: null argument");
  OCCD_CHECK_ARG(out->count && out->hist && out->index && out->cls,
                 "occd_model_list_voxels: count, hist, index and cls are required");
  OCCD_CHECK_ARG(out->capacity >= 0, "occd_model_list_voxels: capacity must be >= 0");
  OCCD_CHECK_ARG(out->voxel_size >= 0.0, "occd_model_list_voxels: voxel_size must be >= 0 (0: the dataset's default)");
  if (m->rank != 0)
    return fail(OCCD_ERR_ARG, "occd_model_list_voxels: rank " + std::to_string(m->rank) + " of the X-slab partition "
                              "holds no map; rank 0 lists the whole map");
  if (m->last_n == 0)
    return fail(OCCD_ERR_ARG, "occd_model_list_voxels: no run yet (or the last run failed): nothing to list");
  if (n < 1 || n > m->last_n)
    return fail(OCCD_ERR_ARG, "occd_model_list_voxels: " + std::to_string(n) + " items, the last run ran 1 to " +
                                  std::to_string(m->last_n));
  const bool nyu = m->dataset == 1;
  const long long N = (long long)m->out[0] * m->out[1] * m->out[2];
  const long long work_len = OCCD_VOXEL_WORK_LEN((long long)m->batch, N);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  cudaError_t e;
  // the scratch of every later listing, on the current device (the model's, as for the runs): the work array of
  // `batch` items, and KITTI's masks
  if (!m->list_work) {
    if ((e = cudaMalloc(&m->list_work, (size_t)work_len * 4)) != cudaSuccess) {
      m->list_work = nullptr;
      return cuda_fail(e, "occd_model_list_voxels: cudaMalloc");
    }
    m->list_bytes += (size_t)work_len * 4;
  }
  if (!nyu && !m->list_mask) {
    if ((e = cudaMalloc(&m->list_mask, (size_t)m->batch * N)) != cudaSuccess) {
      m->list_mask = nullptr;
      return cuda_fail(e, "occd_model_list_voxels: cudaMalloc");
    }
    m->list_bytes += (size_t)m->batch * N;
  }
  if (!nyu)
    for (int b = 0; b < n; ++b) {
      if (m->mask_valid[b]) continue;
      int rc = fov_mask_1(m, (uint32_t)b, N, st);
      if (rc != OCCD_OK) return rc;
      m->mask_valid[b] = 1;
    }
  const double voxel = out->voxel_size > 0 ? out->voxel_size : nyu ? 0.08 : 0.2;
  return occd_occupied_voxels(static_cast<const uint16_t*>(m->dev(ROLE_CLASSES)), nyu ? nullptr : m->list_mask, n,
                              (int)m->out[0], (int)m->out[1], (int)m->out[2], 0, 0, 255, 64, out->capacity,
                              reinterpret_cast<uint32_t*>(out->count), reinterpret_cast<uint32_t*>(out->hist),
                              out->index, out->cls, out->xyz, voxel, out->origin, m->list_work, work_len, st);
}

extern "C" int occd_model_destroy(occd_model* m) {
  if (m) release(m);
  return OCCD_OK;
}
