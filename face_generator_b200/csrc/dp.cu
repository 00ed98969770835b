// Data parallelism: one process per GPU, one NCCL communicator, one in-place sum-allreduce of the
// flat gradient (+8 tail scalars) per optimizer step (SURVEY.md section 8e).  The reference has no
// multi-GPU path at all; this is new functionality behind the same train-step call.
//
// NCCL is bound at run time (dlopen) instead of DT_NEEDED so that loading libfg_b200.so never pins a
// libnccl.so.2 into a process that later imports another copy (e.g. the torch-bundled one used only
// for test/bench plumbing): an already-loaded libnccl.so.2 is reused, else the system one is opened.
#include <dlfcn.h>
#include <nccl.h>

#include <cstring>

#include "fg_internal.h"

namespace {
struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
} g_nccl;

int nccl_load() {
  if (g_nccl.handle) return FG_OK;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) {
    fg_set_error("cannot load libnccl.so.2: %s", dlerror());
    return FG_ERR_NCCL;
  }
#define SYM(field, name)                                                 \
  *(void**)(&g_nccl.field) = dlsym(h, name);                             \
  if (!g_nccl.field) {                                                   \
    fg_set_error("libnccl.so.2 lacks %s", name);                         \
    return FG_ERR_NCCL;                                                  \
  }
  SYM(GetUniqueId, "ncclGetUniqueId")
  SYM(CommInitRank, "ncclCommInitRank")
  SYM(CommDestroy, "ncclCommDestroy")
  SYM(AllReduce, "ncclAllReduce")
  SYM(Broadcast, "ncclBroadcast")
  SYM(GroupStart, "ncclGroupStart")
  SYM(GroupEnd, "ncclGroupEnd")
  SYM(GetErrorString, "ncclGetErrorString")
#undef SYM
  g_nccl.handle = h;
  return FG_OK;
}
}  // namespace

#define FG_NCCL(call)                                                                                 \
  do {                                                                                                \
    ncclResult_t r__ = (call);                                                                        \
    if (r__ != ncclSuccess) {                                                                         \
      fg_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, g_nccl.GetErrorString(r__));         \
      return FG_ERR_NCCL;                                                                             \
    }                                                                                                 \
  } while (0)

int net_allreduce(fg_ctx* c, float* buf, int64_t n) {
  if (c->world <= 1) return FG_OK;
  ScopedTimer t(c, "nccl.allreduce");
  FG_NCCL(g_nccl.AllReduce(buf, buf, (size_t)n, ncclFloat, ncclSum, (ncclComm_t)c->nccl_comm, c->stream));
  return FG_OK;
}

// rank 0's bytes -> every rank (on the ctx stream; callers group several and synchronise once)
int net_broadcast(fg_ctx* c, void* buf, size_t bytes) {
  if (c->world <= 1) return FG_OK;
  FG_NCCL(g_nccl.Broadcast(buf, buf, bytes, ncclChar, 0, (ncclComm_t)c->nccl_comm, c->stream));
  return FG_OK;
}
int net_group(bool start) {
  FG_NCCL(start ? g_nccl.GroupStart() : g_nccl.GroupEnd());
  return FG_OK;
}

extern "C" {
int fg_dp_unique_id(void* out128) {
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is expected to be 128 bytes");
  if (!out128) return FG_ERR_INVALID;
  FG_TRY(nccl_load());
  ncclUniqueId id;
  FG_NCCL(g_nccl.GetUniqueId(&id));
  memcpy(out128, &id, sizeof(id));
  return FG_OK;
}
int fg_dp_init(fg_ctx* c, const void* id128, int nranks, int rank) {
  if (!c || !id128 || nranks < 1 || rank < 0 || rank >= nranks) {
    fg_set_error("fg_dp_init: bad arguments");
    return FG_ERR_INVALID;
  }
  FG_CUDA(cudaSetDevice(c->device));
  pair_clear_graphs(net32_pair(c));  // captured steps reference the old communicator
  c->graph_epoch++;
  if (c->nccl_comm) {
    g_nccl.CommDestroy((ncclComm_t)c->nccl_comm);
    c->nccl_comm = nullptr;
  }
  c->world = 1;
  c->rank = 0;
  if (nranks == 1) return FG_OK;
  FG_TRY(nccl_load());
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  ncclComm_t comm;
  FG_NCCL(g_nccl.CommInitRank(&comm, nranks, id, rank));
  c->nccl_comm = comm;
  c->world = nranks;
  c->rank = rank;
  return FG_OK;
}
int fg_dp_broadcast_params(fg_ctx* c) {
  if (!c) return FG_ERR_INVALID;
  if (c->world <= 1) return FG_OK;
  FG_CUDA(cudaSetDevice(c->device));
  return pair_broadcast(c, net32_pair(c));
}
int fg_dp_world(fg_ctx* c) { return c ? c->world : 0; }
}
