// Communicators of the X-slab partition (include/occdepth_b200_comm.h): the fields the model runtime reads.
#pragma once
#include <cuda_runtime.h>

enum { OCCD_COMM_LOCAL = 0, OCCD_COMM_NCCL = 1 };

struct occd_comm;

// rank, world and kind of a communicator (no device is touched)
void occd_comm_describe(const occd_comm* c, int* rank, int* world, int* kind);
// the group a local communicator belongs to (nullptr for NCCL): equal for the ranks of one occd_comm_create_local
const void* occd_comm_group(const occd_comm* c);
// drops what a local group's ranks have posted towards a collective that will not complete (a failed lock-step run)
void occd_comm_reset(occd_comm* c);
