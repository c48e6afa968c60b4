/*
 * occdepth_b200 -- communicators and model files under the X-slab partition (DESIGN.md section 9).
 *
 * One frame's voxel grid split along X over R ranks: every rank loads its own model file (deploy.export with
 * slab_output="root") and runs every frame; rank 0 receives the whole class map.  The collective launches the files
 * record (occd_comm_halo_exchange, occd_comm_all_gather, occd_comm_gather_root) are declared in occdepth_b200.h with
 * the other launches; this header holds the calls a host makes around them, none of which a model file records.
 *
 * Two kinds of communicator:
 *   NCCL  -- one rank per process and device.  libnccl.so.2 is loaded with dlopen from `nccl_lib` (NULL: the soname),
 *            so libocc_b200.so has no link-time NCCL dependency and single-GPU hosts need no NCCL; when it cannot be
 *            loaded the call returns OCCD_ERR_UNSUPPORTED without touching a device.  Rank 0 makes the 128-byte id
 *            with occd_comm_unique_id; the host ships it to the other ranks by its own means (a file, a socket, MPI).
 *   local -- `world` ranks in one process on the current device: the collectives are device copies between the
 *            ranks' buffers, and the ranks run through occd_model_run_frame_group in lock step.
 *
 * Deadlock rule: every rank calls occd_model_run_frame (or every rank _conf) with the same frames in the same order.
 * A rank that skips a frame, or fails before its collectives, leaves the others waiting inside NCCL.
 */
#ifndef OCCDEPTH_B200_COMM_H
#define OCCDEPTH_B200_COMM_H
#include "occdepth_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

#define OCCD_COMM_ID_BYTES 128

/* id: 128 bytes (host) that every rank passes to occd_comm_create */
int occd_comm_unique_id(const char* nccl_lib, void* id);
/* collective over the `world` ranks, on the current device (one device per rank) */
int occd_comm_create(const char* nccl_lib, const void* id, int rank, int world, occd_comm** comm);
/* `world` local ranks on the current device: rank r in comms[r] */
int occd_comm_create_local(int world, occd_comm** comms);
/* destroy every model that uses the communicator first */
int occd_comm_destroy(occd_comm* comm);

/* Loads the model file of the communicator's rank: the file's rank and world must be the communicator's.  The whole
 * file is validated before any CUDA call, as by occd_model_load, which refuses such files.  On rank 0
 * occd_model_run_frame / _conf write the whole map (and confidence); the other ranks pass class_map and conf NULL.
 * Models on a local communicator run only through occd_model_run_frame_group. */
int occd_model_load_slab(const char* path, occd_comm* comm, occd_model** m);
/* One frame through every rank of a local group: models[r] was loaded with comms[r] of one occd_comm_create_local.
 * The ranks' records run in lock step on `stream` -- each rank up to its next collective, then that collective for
 * all ranks -- and the first run captures the interleaved sequence into one CUDA graph (OCCD_FRAME_NO_GRAPH: never).
 * class_map and conf (NULL: the map only) as rank 0's of occd_model_run_frame / _conf. */
int occd_model_run_frame_group(occd_model* const* models, int world, const occd_frame* frame, uint16_t* class_map,
                               void* conf, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* OCCDEPTH_B200_COMM_H */
