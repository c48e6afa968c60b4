// Communicators of the X-slab partition (include/occdepth_b200_comm.h) and the three collective launches a slab model
// file records (include/occdepth_b200.h).  They move exactly what parallel.HaloExchangeOp, AllGatherOp and
// GatherRootOp move over torch.distributed, but with no torch: NCCL loaded at run time, or -- for `world` ranks in one
// process -- device copies between the ranks' buffers (the C counterpart of parallel.SimSlabGroup).
#include "common.cuh"
#include "comm.cuh"
#include "../../include/occdepth_b200_comm.h"

#include <dlfcn.h>
#include <string.h>

#include <string>
#include <vector>

namespace {

// the NCCL entry points used here, with the ABI of nccl.h (ncclComm_t is a pointer, enums are int)
struct NcclId {
  char internal[OCCD_COMM_ID_BYTES];
};
const int kNcclInt8 = 0;
struct Nccl {
  int (*get_unique_id)(NcclId*);
  int (*comm_init_rank)(void**, int, NcclId, int);
  int (*comm_destroy)(void*);
  int (*group_start)();
  int (*group_end)();
  int (*send)(const void*, size_t, int, int, void*, cudaStream_t);
  int (*recv)(void*, size_t, int, int, void*, cudaStream_t);
  int (*all_gather)(const void*, void*, size_t, int, void*, cudaStream_t);
  const char* (*error_string)(int);
};

int fail(int code, const std::string& msg) {
  occd_set_last_error(msg.c_str());
  return code;
}

// the library stays loaded for the process (NCCL is not made to be unloaded)
int load_nccl(const char* path, Nccl* n) {
  const char* name = path ? path : "libnccl.so.2";
  void* h = dlopen(name, RTLD_NOW | RTLD_LOCAL);
  if (!h) {
    const char* why = dlerror();
    return fail(OCCD_ERR_UNSUPPORTED, std::string("occd_comm: cannot load NCCL from ") + name + ": " +
                                          (why ? why : "dlopen failed"));
  }
  struct {
    const char* sym;
    void** slot;
  } want[] = {{"ncclGetUniqueId", (void**)&n->get_unique_id}, {"ncclCommInitRank", (void**)&n->comm_init_rank},
              {"ncclCommDestroy", (void**)&n->comm_destroy},  {"ncclGroupStart", (void**)&n->group_start},
              {"ncclGroupEnd", (void**)&n->group_end},        {"ncclSend", (void**)&n->send},
              {"ncclRecv", (void**)&n->recv},                 {"ncclAllGather", (void**)&n->all_gather},
              {"ncclGetErrorString", (void**)&n->error_string}};
  for (auto& w : want) {
    *w.slot = dlsym(h, w.sym);
    if (!*w.slot)
      return fail(OCCD_ERR_UNSUPPORTED, std::string("occd_comm: ") + name + " has no " + w.sym);
  }
  return OCCD_OK;
}

enum Kind { HALO = 1, ALL_GATHER = 2, GATHER_ROOT = 3 };
const char* kKindNames[] = {"", "occd_comm_halo_exchange", "occd_comm_all_gather", "occd_comm_gather_root"};

// one rank's arguments of a collective, held until every local rank has posted its own
struct Post {
  int kind = 0;
  char* base = nullptr;       // halo: the activation; all-gather / gather-root: dst
  const char* src = nullptr;
  long long bytes = 0;        // halo / gather-root: plane bytes; all-gather: shard bytes
  int halo = 0, planes = 0;
  std::vector<int> bounds;
};

struct LocalGroup {
  int world = 0, live = 0;  // live: communicators not yet destroyed
  int posted = 0;
  std::vector<Post> posts;
};

}  // namespace

struct occd_comm {
  int kind, rank, world;
  LocalGroup* group = nullptr;  // local
  Nccl nccl;                    // NCCL
  void* nc = nullptr;
};

void occd_comm_describe(const occd_comm* c, int* rank, int* world, int* kind) {
  *rank = c->rank;
  *world = c->world;
  *kind = c->kind;
}

const void* occd_comm_group(const occd_comm* c) { return c->group; }

void occd_comm_reset(occd_comm* c) {
  if (!c->group) return;
  c->group->posted = 0;
  for (Post& p : c->group->posts) p = Post();
}

namespace {

int nccl_fail(const occd_comm* c, int r, const char* what) {
  return fail(OCCD_ERR_CUDA, std::string(what) + ": " + c->nccl.error_string(r));
}

int copy(void* dst, const void* src, long long n, cudaStream_t st) {
  if (n <= 0) return OCCD_OK;
  cudaError_t e = cudaMemcpyAsync(dst, src, (size_t)n, cudaMemcpyDeviceToDevice, st);
  return e == cudaSuccess ? OCCD_OK : fail(OCCD_ERR_CUDA, std::string("occd_comm: copy: ") + cudaGetErrorString(e));
}

// every local rank has posted: the copies of all ranks, on the stream of the last post
int run_local(LocalGroup* g, cudaStream_t st) {
  const int W = g->world;
  const Post& p0 = g->posts[0];
  for (int r = 1; r < W; ++r)
    if (g->posts[r].kind != p0.kind || g->posts[r].bytes != p0.bytes)
      return fail(OCCD_ERR_ARG, std::string(kKindNames[p0.kind]) + ": local rank " + std::to_string(r) +
                                    " posted another collective or size than rank 0 (the ranks are out of step)");
  int rc = OCCD_OK;
  const long long pb = p0.bytes;
  if (p0.kind == HALO) {
    for (int r = 0; r < W && rc == OCCD_OK; ++r) {
      const Post& p = g->posts[r];
      const int w = p.halo < p.planes ? p.halo : p.planes;
      if (r > 0) {
        const Post& q = g->posts[r - 1];
        if ((q.halo < q.planes ? q.halo : q.planes) != w)
          return fail(OCCD_ERR_ARG, "occd_comm_halo_exchange: neighbouring ranks move different plane counts");
        rc = copy(p.base + (long long)(p.halo - w) * pb, q.base + (long long)(q.halo + q.planes - w) * pb, w * pb, st);
      }
      if (rc == OCCD_OK && r < W - 1) {
        const Post& q = g->posts[r + 1];
        rc = copy(p.base + (long long)(p.halo + p.planes) * pb, q.base + (long long)q.halo * pb, w * pb, st);
      }
    }
  } else if (p0.kind == ALL_GATHER) {
    for (int r = 0; r < W && rc == OCCD_OK; ++r)
      for (int q = 0; q < W && rc == OCCD_OK; ++q) rc = copy(g->posts[r].base + q * pb, g->posts[q].src, pb, st);
  } else {
    for (int q = 0; q < W && rc == OCCD_OK; ++q) {
      const int lo = p0.bounds[2 * q], hi = p0.bounds[2 * q + 1];
      rc = copy(p0.base + (long long)lo * pb, g->posts[q].src, (long long)(hi - lo) * pb, st);
    }
  }
  return rc;
}

int post(occd_comm* c, Post p, cudaStream_t st) {
  LocalGroup* g = c->group;
  if (g->posts[c->rank].kind != 0)
    return fail(OCCD_ERR_ARG, std::string(kKindNames[p.kind]) + ": local rank " + std::to_string(c->rank) +
                                  " posted twice before the others (run local ranks through occd_model_run_frame_group)");
  g->posts[c->rank] = std::move(p);
  if (++g->posted < g->world) return OCCD_OK;
  int rc = run_local(g, st);
  occd_comm_reset(c);
  return rc;
}

}  // namespace

extern "C" int occd_comm_unique_id(const char* nccl_lib, void* id) {
  OCCD_CHECK_ARG(id, "occd_comm_unique_id: null id");
  Nccl n;
  int rc = load_nccl(nccl_lib, &n);
  if (rc != OCCD_OK) return rc;
  NcclId u;
  int r = n.get_unique_id(&u);
  if (r != 0) return fail(OCCD_ERR_CUDA, std::string("ncclGetUniqueId: ") + n.error_string(r));
  memcpy(id, &u, sizeof(u));
  return OCCD_OK;
}

extern "C" int occd_comm_create(const char* nccl_lib, const void* id, int rank, int world, occd_comm** comm) {
  OCCD_CHECK_ARG(id && comm, "occd_comm_create: null argument");
  *comm = nullptr;
  OCCD_CHECK_ARG(world >= 1 && rank >= 0 && rank < world, "occd_comm_create: rank outside [0, world)");
  occd_comm* c = new occd_comm();
  c->kind = OCCD_COMM_NCCL;
  c->rank = rank;
  c->world = world;
  int rc = load_nccl(nccl_lib, &c->nccl);
  if (rc == OCCD_OK) {
    NcclId u;
    memcpy(&u, id, sizeof(u));
    int r = c->nccl.comm_init_rank(&c->nc, world, u, rank);
    if (r != 0) rc = nccl_fail(c, r, "ncclCommInitRank");
  }
  if (rc != OCCD_OK) {
    delete c;
    return rc;
  }
  *comm = c;
  return OCCD_OK;
}

extern "C" int occd_comm_create_local(int world, occd_comm** comms) {
  OCCD_CHECK_ARG(comms && world >= 1 && world <= 64, "occd_comm_create_local: world must be 1..64 with comms");
  LocalGroup* g = new LocalGroup();
  g->world = g->live = world;
  g->posts.resize(world);
  for (int r = 0; r < world; ++r) {
    comms[r] = new occd_comm();
    comms[r]->kind = OCCD_COMM_LOCAL;
    comms[r]->rank = r;
    comms[r]->world = world;
    comms[r]->group = g;
  }
  return OCCD_OK;
}

extern "C" int occd_comm_destroy(occd_comm* c) {
  if (!c) return OCCD_OK;
  if (c->group && --c->group->live == 0) delete c->group;
  if (c->nc) c->nccl.comm_destroy(c->nc);
  delete c;
  return OCCD_OK;
}

// ---- the collective launches ------------------------------------------------------------------------------------------
// A NULL communicator passes the loader (a record with no communicator slot filled) and is refused here.
#define OCCD_CHECK_COMM(c, name) \
  OCCD_CHECK_ARG(c, name ": no communicator (a slab model file gets its communicator from occd_model_load_slab)")

extern "C" int occd_comm_halo_exchange(occd_comm* c, void* base, long long plane_bytes, int halo, int planes,
                                       void* stream) {
  OCCD_CHECK_COMM(c, "occd_comm_halo_exchange");
  OCCD_CHECK_ARG(base && plane_bytes > 0 && halo >= 0 && planes >= 1, "occd_comm_halo_exchange: bad arguments");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  char* b = static_cast<char*>(base);
  if (c->kind == OCCD_COMM_LOCAL) {
    Post p;
    p.kind = HALO;
    p.base = b;
    p.bytes = plane_bytes;
    p.halo = halo;
    p.planes = planes;
    return post(c, std::move(p), st);
  }
  const long long w = halo < planes ? halo : planes;
  const size_t n = (size_t)(w * plane_bytes);
  if (c->world == 1 || n == 0) return OCCD_OK;
  const Nccl& N = c->nccl;
  int r = N.group_start();
  if (r == 0 && c->rank > 0) {
    r = N.send(b + halo * plane_bytes, n, kNcclInt8, c->rank - 1, c->nc, st);
    if (r == 0) r = N.recv(b + (halo - w) * plane_bytes, n, kNcclInt8, c->rank - 1, c->nc, st);
  }
  if (r == 0 && c->rank < c->world - 1) {
    r = N.send(b + (halo + planes - w) * plane_bytes, n, kNcclInt8, c->rank + 1, c->nc, st);
    if (r == 0) r = N.recv(b + (halo + planes) * plane_bytes, n, kNcclInt8, c->rank + 1, c->nc, st);
  }
  const int r_end = N.group_end();
  if (r == 0) r = r_end;
  return r == 0 ? OCCD_OK : nccl_fail(c, r, "occd_comm_halo_exchange");
}

extern "C" int occd_comm_all_gather(occd_comm* c, const void* src, void* dst, long long bytes, void* stream) {
  OCCD_CHECK_COMM(c, "occd_comm_all_gather");
  OCCD_CHECK_ARG(src && dst && bytes > 0, "occd_comm_all_gather: bad arguments");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (c->kind == OCCD_COMM_LOCAL) {
    Post p;
    p.kind = ALL_GATHER;
    p.base = static_cast<char*>(dst);
    p.src = static_cast<const char*>(src);
    p.bytes = bytes;
    return post(c, std::move(p), st);
  }
  int r = c->nccl.all_gather(src, dst, (size_t)bytes, kNcclInt8, c->nc, st);
  return r == 0 ? OCCD_OK : nccl_fail(c, r, "occd_comm_all_gather");
}

extern "C" int occd_comm_gather_root(occd_comm* c, const void* src, void* dst, const int* bounds,
                                     long long plane_bytes, void* stream) {
  OCCD_CHECK_COMM(c, "occd_comm_gather_root");
  OCCD_CHECK_ARG(src && bounds && plane_bytes > 0 && (c->rank != 0 || dst), "occd_comm_gather_root: bad arguments");
  for (int r = 0; r < c->world; ++r)
    OCCD_CHECK_ARG(bounds[2 * r] == (r ? bounds[2 * r - 1] : 0) && bounds[2 * r + 1] > bounds[2 * r],
                   "occd_comm_gather_root: the bounds must tile the planes from 0, rank by rank");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (c->kind == OCCD_COMM_LOCAL) {
    Post p;
    p.kind = GATHER_ROOT;
    p.base = static_cast<char*>(dst);
    p.src = static_cast<const char*>(src);
    p.bytes = plane_bytes;
    p.bounds.assign(bounds, bounds + 2 * c->world);
    return post(c, std::move(p), st);
  }
  const Nccl& N = c->nccl;
  char* d = static_cast<char*>(dst);
  if (c->rank == 0) {
    cudaError_t e = cudaMemcpyAsync(d, src, (size_t)((bounds[1] - bounds[0]) * plane_bytes), cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) return fail(OCCD_ERR_CUDA, std::string("occd_comm_gather_root: ") + cudaGetErrorString(e));
    if (c->world == 1) return OCCD_OK;
  }
  int r = N.group_start();
  if (c->rank == 0) {
    for (int q = 1; q < c->world && r == 0; ++q)
      r = N.recv(d + bounds[2 * q] * plane_bytes, (size_t)((bounds[2 * q + 1] - bounds[2 * q]) * plane_bytes),
                 kNcclInt8, q, c->nc, st);
  } else if (r == 0) {
    r = N.send(src, (size_t)((bounds[2 * c->rank + 1] - bounds[2 * c->rank]) * plane_bytes), kNcclInt8, 0, c->nc, st);
  }
  const int r_end = N.group_end();
  if (r == 0) r = r_end;
  return r == 0 ? OCCD_OK : nccl_fail(c, r, "occd_comm_gather_root");
}
