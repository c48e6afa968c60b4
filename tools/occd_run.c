/*
 * occd_run -- run an exported OccDepth model (occdepth_b200.deploy.export) on camera frames, without Python.
 * Linked only against libocc_b200.so and the CUDA runtime; `python -m occdepth_b200._build` builds it next to
 * the library (occdepth_b200/lib/occd_run).
 *
 *   occd_run MODEL IMAGES CALIB N OUT_DIR [--raw H0 W0] [--format rgb|bgr|nv12] [--depth DEPTH] [--no-graph]
 *            [--voxels CAP] [--probs FILE] [--world W --rank R --nccl-id FILE [--nccl-lib LIBNCCL]]
 *
 * Inputs are raw little-endian files, one record per frame, frames back to back (no image decoder):
 *   IMAGES  N x V x H0 x W0 x 3 uint8, RGB, row-major (H0 x W0 default to the model's crop; --raw gives larger
 *           images, cropped to the top-left corner as the datasets do, or remapped by the file's rectification
 *           maps); --format bgr: the same with pixels B, G, R; --format nv12: N x V x (H0 * 3 / 2) x W0, each image
 *           OpenCV's NV12 layout (H0 luma rows, then H0 / 2 rows of interleaved U, V; H0 and W0 even)
 *   CALIB   N records of float64: KITTI  V x 9 cam_k, then V x 16 T_velo_2_cam (row-major)
 *                                  NYU    9 cam_k, 16 T_world_2_cam (the inverse of the camera pose), 3 vox_origin
 *   DEPTH   (NYU models with the virtual view) N x depth_h x depth_w uint16, the depth PNGs' values
 * Output: OUT_DIR/NNNNNN.label per frame, the uint16 class map (X x Y x Z, C order) as the KITTI submission writer
 * stores it; the labels are remapped when the model was exported with inv_map.  Prints ms per frame (device time
 * of occd_model_run_frames_ex, from CUDA events) and the mean over the frames after the first.
 *
 * --voxels CAP: after each run, occd_model_list_voxels lists the occupied voxels of every frame's map (CAP rows per
 * frame at most; coordinates at the dataset's output voxel size, in the grid's frame) and OUT_DIR/NNNNNN.voxels gets,
 * little-endian: int32 count[2] (occupied voxels inside / outside the FOV, the true counts), int32 hist[64] (per class
 * id), then the R = min(CAP, count[0] + count[1]) written rows as int32 index[R], uint16 cls[R], float32 xyz[R][3]
 * (in-FOV rows first, each group in ascending flat index).  The two counts are printed per frame.
 *
 * --probs FILE: a model exported with probabilities (deploy.export(..., probabilities=True)) runs through
 * occd_model_run_frames_probs, and FILE gets every frame's float16 class probabilities, C x X x Y x Z (C order), frame
 * after frame; the .label files are written as without it.
 *
 * A batched model file (deploy.export of a list of B frames) runs the frames in groups of B, the last group short;
 * the times are then per group, and the mean is per frame over the groups after the first.
 *
 * X-slab partition over W GPUs: one process per rank, each on its own device (e.g. CUDA_VISIBLE_DEVICES), MODEL the
 * rank's file (deploy.export(..., slab_output="root")) and the same inputs on every rank.  Rank 0 writes the NCCL id
 * to FILE, the other ranks wait for it; only rank 0 writes .label files.  LIBNCCL: where libnccl.so.2 is, when the
 * loader does not find it by name.
 */
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include "occdepth_b200_comm.h"

#define CK(x)                                                                          \
  do {                                                                                 \
    cudaError_t e_ = (x);                                                              \
    if (e_ != cudaSuccess) {                                                           \
      fprintf(stderr, "occd_run: %s: %s\n", #x, cudaGetErrorString(e_));              \
      return 1;                                                                        \
    }                                                                                  \
  } while (0)
#define OK(x)                                                                          \
  do {                                                                                 \
    if ((x) != OCCD_OK) {                                                              \
      fprintf(stderr, "occd_run: %s: %s\n", #x, occd_last_error());                    \
      return 1;                                                                        \
    }                                                                                  \
  } while (0)

static int read_exact(FILE* f, void* dst, size_t n, const char* what) {
  if (fread(dst, 1, n, f) != n) {
    fprintf(stderr, "occd_run: %s is shorter than the frames asked for\n", what);
    return 0;
  }
  return 1;
}

/* the NCCL id of a W-rank run: rank 0 makes it and writes FILE (whole, through a rename); the others wait for FILE */
static int share_id(const char* path, int rank, const char* nccl_lib, char* id) {
  if (rank == 0) {
    if (occd_comm_unique_id(nccl_lib, id) != OCCD_OK) {
      fprintf(stderr, "occd_run: occd_comm_unique_id: %s\n", occd_last_error());
      return 0;
    }
    char tmp[4096];
    snprintf(tmp, sizeof(tmp), "%s.tmp", path);
    FILE* f = fopen(tmp, "wb");
    if (!f || fwrite(id, 1, OCCD_COMM_ID_BYTES, f) != OCCD_COMM_ID_BYTES || fclose(f) != 0 || rename(tmp, path) != 0) {
      fprintf(stderr, "occd_run: cannot write %s\n", path);
      return 0;
    }
    return 1;
  }
  for (int t = 0; t < 6000; ++t) { /* 10 minutes */
    FILE* f = fopen(path, "rb");
    if (f) {
      size_t n = fread(id, 1, OCCD_COMM_ID_BYTES, f);
      fclose(f);
      if (n == OCCD_COMM_ID_BYTES) return 1;
    }
    usleep(100000);
  }
  fprintf(stderr, "occd_run: rank %d: no NCCL id in %s\n", rank, path);
  return 0;
}

/* OUT_DIR/NNNNNN.voxels of item i of a group of k listed frames: its counts and histogram from h (the group's k x 2
 * counts, then k x 64 bins), its written rows read back from the device lists */
static int write_voxels(const char* out_dir, int frame, int32_t* h, int k, int i, int cap, const int32_t* d_index,
                        const uint16_t* d_cls, const float* d_xyz) {
  const int32_t* count = h + 2 * i;
  const int32_t* hist = h + 2 * k + 64 * i;
  const long long total = (long long)count[0] + count[1];
  const size_t r = (size_t)(total < cap ? total : cap);
  char* rows = (char*)(h + 66 * k);  /* after the group's counts and bins */
  if (cudaMemcpy(rows, d_index + (size_t)i * cap, r * 4, cudaMemcpyDeviceToHost) != cudaSuccess ||
      cudaMemcpy(rows + r * 4, d_cls + (size_t)i * cap, r * 2, cudaMemcpyDeviceToHost) != cudaSuccess ||
      cudaMemcpy(rows + r * 6, d_xyz + (size_t)i * cap * 3, r * 12, cudaMemcpyDeviceToHost) != cudaSuccess) {
    fprintf(stderr, "occd_run: reading back the voxel rows failed\n");
    return 0;
  }
  char path[4096];
  snprintf(path, sizeof(path), "%s/%06d.voxels", out_dir, frame);
  FILE* fo = fopen(path, "wb");
  if (!fo || fwrite(count, 4, 2, fo) != 2 || fwrite(hist, 4, 64, fo) != 64 || fwrite(rows, 1, r * 18, fo) != r * 18) {
    fprintf(stderr, "occd_run: cannot write %s\n", path);
    return 0;
  }
  fclose(fo);
  printf("frame %d: %d voxels inside the FOV, %d outside\n", frame, count[0], count[1]);
  return 1;
}

int main(int argc, char** argv) {
  if (argc < 6) {
    fprintf(stderr, "usage: occd_run MODEL IMAGES CALIB N OUT_DIR [--raw H0 W0] [--format rgb|bgr|nv12] "
                    "[--depth DEPTH] [--no-graph] [--voxels CAP] [--probs FILE]\n");
    return 2;
  }
  const char *model_path = argv[1], *img_path = argv[2], *calib_path = argv[3], *out_dir = argv[5];
  const char *depth_path = NULL, *id_path = NULL, *nccl_lib = NULL, *probs_path = NULL;
  int n = atoi(argv[4]), H0 = 0, W0 = 0, flags = 0, world = 1, rank = 0, format = OCCD_PIX_RGB, cap = -1;
  for (int i = 6; i < argc; ++i) {
    if (!strcmp(argv[i], "--raw") && i + 2 < argc) {
      H0 = atoi(argv[++i]);
      W0 = atoi(argv[++i]);
    } else if (!strcmp(argv[i], "--format") && i + 1 < argc) {
      const char* f = argv[++i];
      format = !strcmp(f, "rgb") ? OCCD_PIX_RGB : !strcmp(f, "bgr") ? OCCD_PIX_BGR : !strcmp(f, "nv12") ? OCCD_PIX_NV12 : -1;
      if (format < 0) {
        fprintf(stderr, "occd_run: --format takes rgb, bgr or nv12\n");
        return 2;
      }
    } else if (!strcmp(argv[i], "--depth") && i + 1 < argc) {
      depth_path = argv[++i];
    } else if (!strcmp(argv[i], "--voxels") && i + 1 < argc) {
      cap = atoi(argv[++i]);
      if (cap < 0) {
        fprintf(stderr, "occd_run: --voxels takes a capacity >= 0\n");
        return 2;
      }
    } else if (!strcmp(argv[i], "--probs") && i + 1 < argc) {
      probs_path = argv[++i];
    } else if (!strcmp(argv[i], "--no-graph")) {
      flags |= OCCD_FRAME_NO_GRAPH;
    } else if (!strcmp(argv[i], "--world") && i + 1 < argc) {
      world = atoi(argv[++i]);
    } else if (!strcmp(argv[i], "--rank") && i + 1 < argc) {
      rank = atoi(argv[++i]);
    } else if (!strcmp(argv[i], "--nccl-id") && i + 1 < argc) {
      id_path = argv[++i];
    } else if (!strcmp(argv[i], "--nccl-lib") && i + 1 < argc) {
      nccl_lib = argv[++i];
    } else {
      fprintf(stderr, "occd_run: unknown option %s\n", argv[i]);
      return 2;
    }
  }
  if (world > 1 && (!id_path || rank < 0 || rank >= world)) {
    fprintf(stderr, "occd_run: --world W needs --rank R (0 <= R < W) and --nccl-id FILE\n");
    return 2;
  }
  occd_model* m = NULL;
  occd_comm* comm = NULL;
  if (world > 1) {
    char id[OCCD_COMM_ID_BYTES];
    if (!share_id(id_path, rank, nccl_lib, id)) return 1;
    OK(occd_comm_create(nccl_lib, id, rank, world, &comm));
    OK(occd_model_load_slab(model_path, comm, &m));
  } else {
    OK(occd_model_load(model_path, &m));
  }
  occd_model_geom g;
  OK(occd_model_info(m, &g));
  int B = 1;
  OK(occd_model_batch(m, &B));
  if (!H0) {
    H0 = g.img_h;
    W0 = g.img_w;
  }
  const int nyu = g.dataset == 1;
  // one image: 3 bytes a pixel, or NV12's 1.5
  const size_t one_img = format == OCCD_PIX_NV12 ? (size_t)H0 * W0 * 3 / 2 : (size_t)H0 * W0 * 3;
  const size_t img_bytes = (size_t)g.V * one_img;
  const size_t n_calib = nyu ? 9 + 16 + 3 : (size_t)g.V * 25;
  const size_t map_bytes = (size_t)g.X * g.Y * g.Z * 2;
  const size_t depth_bytes = (size_t)g.depth_h * g.depth_w * 2;
  if (g.has_depth && !depth_path) {
    fprintf(stderr, "occd_run: this model takes a depth map per frame (--depth)\n");
    return 2;
  }
  FILE* fi = fopen(img_path, "rb");
  FILE* fc = fopen(calib_path, "rb");
  FILE* fd = depth_path ? fopen(depth_path, "rb") : NULL;
  if (!fi || !fc || (depth_path && !fd)) {
    fprintf(stderr, "occd_run: cannot open the input files\n");
    return 1;
  }
  unsigned char* h_img = (unsigned char*)malloc(img_bytes * B);
  unsigned short* h_depth = (unsigned short*)malloc(depth_bytes ? depth_bytes * B : 1);
  unsigned short* h_map = (unsigned short*)malloc(map_bytes * B);
  /* --probs: C float16 planes of the map's size per frame */
  const size_t probs_bytes = probs_path ? map_bytes * g.n_classes : 0;
  void* d_probs = NULL;
  unsigned short* h_probs = probs_path ? (unsigned short*)malloc(probs_bytes * B) : NULL;
  FILE* fp = probs_path && rank == 0 ? fopen(probs_path, "wb") : NULL;
  if (probs_path && rank == 0 && !fp) {
    fprintf(stderr, "occd_run: cannot open %s\n", probs_path);
    return 1;
  }
  if (probs_path && rank == 0) CK(cudaMalloc(&d_probs, probs_bytes * B));
  double* calib = (double*)malloc(n_calib * sizeof(double) * B);
  occd_frame_ex* fs = (occd_frame_ex*)calloc(B, sizeof(occd_frame_ex));
  void *d_img, *d_depth = NULL, *d_map;
  cudaStream_t st;
  cudaEvent_t e0, e1;
  CK(cudaMalloc(&d_img, img_bytes * B));
  CK(cudaMalloc(&d_map, map_bytes * B));
  if (g.has_depth) CK(cudaMalloc(&d_depth, depth_bytes * B));
  /* --voxels: the lists of a group, and one frame's on the host */
  int32_t *d_count = NULL, *d_hist = NULL, *d_index = NULL, *h_vox = NULL;
  uint16_t* d_cls = NULL;
  float* d_xyz = NULL;
  const size_t row_bytes = 4 + 2 + 12;
  if (cap >= 0 && rank == 0) {
    CK(cudaMalloc((void**)&d_count, (size_t)B * 2 * 4));
    CK(cudaMalloc((void**)&d_hist, (size_t)B * 64 * 4));
    CK(cudaMalloc((void**)&d_index, (size_t)B * cap * 4 + 4));
    CK(cudaMalloc((void**)&d_cls, (size_t)B * cap * 2 + 2));
    CK(cudaMalloc((void**)&d_xyz, (size_t)B * cap * 12 + 12));
    h_vox = (int32_t*)malloc((size_t)B * 66 * 4 + (size_t)cap * row_bytes + 4);
  }
  CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  double total = 0;
  int groups = 0;
  for (int i0 = 0; i0 < n; i0 += B) {
    const int k = n - i0 < B ? n - i0 : B;
    for (int i = 0; i < k; ++i) {
      unsigned char* img = h_img + img_bytes * i;
      unsigned short* depth = h_depth + (depth_bytes / 2) * i;
      double* cal = calib + n_calib * i;
      if (!read_exact(fi, img, img_bytes, "IMAGES") || !read_exact(fc, cal, n_calib * 8, "CALIB") ||
          (fd && !read_exact(fd, depth, depth_bytes, "DEPTH")))
        return 1;
      CK(cudaMemcpyAsync((char*)d_img + img_bytes * i, img, img_bytes, cudaMemcpyHostToDevice, st));
      if (fd) CK(cudaMemcpyAsync((char*)d_depth + depth_bytes * i, depth, depth_bytes, cudaMemcpyHostToDevice, st));
      memset(&fs[i], 0, sizeof(fs[i]));
      fs[i].pixel_format = format;
      fs[i].uv_offset = (long long)H0 * W0;  /* NV12: the chroma rows follow the luma plane */
      occd_frame* f = &fs[i].frame;
      f->images = (char*)d_img + img_bytes * i;
      f->img_stride = (long long)one_img;
      f->row_stride = format == OCCD_PIX_NV12 ? (long long)W0 : (long long)W0 * 3;
      f->H0 = H0;
      f->W0 = W0;
      f->cam_k = cal;
      f->pose = nyu ? cal + 9 : cal + 9 * g.V;
      f->calib_f32 = 0;
      f->vox_origin = nyu ? cal + 25 : NULL;
      f->depth = d_depth ? (const uint16_t*)((char*)d_depth + depth_bytes * i) : NULL;
      f->depth_h = g.depth_h;
      f->depth_w = g.depth_w;
      f->flags = flags;
    }
    CK(cudaEventRecord(e0, st));
    if (probs_path)
      OK(occd_model_run_frames_probs(m, fs, k, rank == 0 ? (uint16_t*)d_map : NULL, d_probs, st));
    else
      OK(occd_model_run_frames_ex(m, fs, k, rank == 0 ? (uint16_t*)d_map : NULL, NULL, st));
    CK(cudaEventRecord(e1, st));
    if (rank == 0) CK(cudaMemcpyAsync(h_map, d_map, map_bytes * k, cudaMemcpyDeviceToHost, st));
    if (fp) CK(cudaMemcpyAsync(h_probs, d_probs, probs_bytes * k, cudaMemcpyDeviceToHost, st));
    if (h_vox) {
      occd_voxel_out vo;
      memset(&vo, 0, sizeof(vo));
      vo.capacity = cap;
      vo.count = d_count;
      vo.hist = d_hist;
      vo.index = d_index;
      vo.cls = d_cls;
      vo.xyz = d_xyz;
      OK(occd_model_list_voxels(m, k, &vo, st));
      CK(cudaMemcpyAsync(h_vox, d_count, (size_t)k * 2 * 4, cudaMemcpyDeviceToHost, st));
      CK(cudaMemcpyAsync(h_vox + (size_t)k * 2, d_hist, (size_t)k * 64 * 4, cudaMemcpyDeviceToHost, st));
    }
    CK(cudaStreamSynchronize(st));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    if (i0 > 0) {
      total += ms / k;
      ++groups;
    }
    if (rank != 0) continue;
    if (fp && fwrite(h_probs, 1, probs_bytes * k, fp) != probs_bytes * k) {
      fprintf(stderr, "occd_run: cannot write %s\n", probs_path);
      return 1;
    }
    for (int i = 0; i < k; ++i) {
      char path[4096];
      snprintf(path, sizeof(path), "%s/%06d.label", out_dir, i0 + i);
      FILE* fo = fopen(path, "wb");
      if (!fo || fwrite(h_map + (map_bytes / 2) * i, 1, map_bytes, fo) != map_bytes) {
        fprintf(stderr, "occd_run: cannot write %s\n", path);
        return 1;
      }
      fclose(fo);
      if (h_vox && !write_voxels(out_dir, i0 + i, h_vox, k, i, cap, d_index, d_cls, d_xyz)) return 1;
    }
    if (B == 1) printf("frame %d: %.3f ms\n", i0, ms);
    else printf("frames %d..%d: %.3f ms\n", i0, i0 + k - 1, ms);
  }
  if (groups > 0) {
    if (B == 1) printf("mean over frames 1..%d: %.3f ms per frame\n", n - 1, total / groups);
    else printf("mean over groups 1..%d: %.3f ms per frame\n", groups, total / groups);
  }
  OK(occd_model_destroy(m));
  if (comm) OK(occd_comm_destroy(comm));
  fclose(fi);
  fclose(fc);
  if (fd) fclose(fd);
  if (fp && fclose(fp) != 0) {
    fprintf(stderr, "occd_run: cannot write %s\n", probs_path);
    return 1;
  }
  free(h_probs);
  if (d_probs) cudaFree(d_probs);
  free(h_img);
  free(h_depth);
  free(h_map);
  free(calib);
  free(fs);
  free(h_vox);
  cudaFree(d_count);
  cudaFree(d_hist);
  cudaFree(d_index);
  cudaFree(d_cls);
  cudaFree(d_xyz);
  cudaFree(d_img);
  cudaFree(d_map);
  if (d_depth) cudaFree(d_depth);
  cudaStreamDestroy(st);
  return 0;
}
