// Multi-GPU exchange of the path: one 32-byte pose record per rank per step (SURVEY.md §8e).
//
// The path shards by independent tracks (one LaserTrack per GPU, reference
// laser_slam/src/incremental_estimator.cpp:22-26 creates n_laser_slam_workers of them); there is no data-path
// collective.  What every rank needs from the others each step is the 6-DoF pose delta its track produced (to
// feed the shared estimator): one ncclAllGather of 32 B/rank over NVLink -- latency bound, so it runs on the
// context's own stream right behind the registration and is synchronised once.
//
// NCCL is resolved at run time (dlopen "libnccl.so.2"): inside a torch process that is the NCCL torch already
// loaded, elsewhere the system one.  The library itself therefore has no link-time NCCL dependency.
#include <dlfcn.h>

#include <cstdio>
#include <cstring>
#include <string>

#include <cuda_runtime.h>

#include "../../include/ls_b200.h"
#include "ls_buffer.cuh"

namespace {

struct NcclUniqueId {
  char internal[128];
};
typedef void* NcclComm;
typedef int (*GetUniqueIdFn)(NcclUniqueId*);
typedef int (*CommInitRankFn)(NcclComm*, int, NcclUniqueId, int);
typedef int (*AllGatherFn)(const void*, void*, size_t, int /*ncclDataType_t*/, NcclComm, cudaStream_t);
typedef int (*CommDestroyFn)(NcclComm);
typedef const char* (*GetErrorStringFn)(int);

struct NcclApi {
  void* handle = nullptr;
  GetUniqueIdFn get_unique_id = nullptr;
  CommInitRankFn comm_init_rank = nullptr;
  AllGatherFn all_gather = nullptr;
  CommDestroyFn comm_destroy = nullptr;
  GetErrorStringFn get_error_string = nullptr;
  bool ok = false;
};

NcclApi& api() {
  static NcclApi a;
  if (!a.handle) {
    a.handle = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (a.handle) {
      a.get_unique_id = (GetUniqueIdFn)dlsym(a.handle, "ncclGetUniqueId");
      a.comm_init_rank = (CommInitRankFn)dlsym(a.handle, "ncclCommInitRank");
      a.all_gather = (AllGatherFn)dlsym(a.handle, "ncclAllGather");
      a.comm_destroy = (CommDestroyFn)dlsym(a.handle, "ncclCommDestroy");
      a.get_error_string = (GetErrorStringFn)dlsym(a.handle, "ncclGetErrorString");
      a.ok = a.get_unique_id && a.comm_init_rank && a.all_gather && a.comm_destroy;
    }
  }
  return a;
}

}  // namespace

struct ls_comm {
  int device = 0, rank = 0, nranks = 1;
  NcclComm comm = nullptr;
  cudaStream_t stream = nullptr;
  ls::Buffer<ls_pose_record> d_send;
  ls::Buffer<ls_pose_record> d_recv;
  ls::PinnedBuffer<ls_pose_record> h_pinned;  // [1 + nranks]
  bool pending = false;                // a begin() without its end()
  std::string err;
};

extern "C" {

int ls_comm_unique_id(void* id128) {
  if (!id128) return LS_ERR_ARG;
  NcclApi& a = api();
  if (!a.ok) return LS_ERR_NCCL;
  NcclUniqueId id;
  if (a.get_unique_id(&id) != 0) return LS_ERR_NCCL;
  std::memcpy(id128, &id, sizeof(id));
  return LS_OK;
}

int ls_comm_init(int device, int rank, int nranks, const void* id128, ls_comm** out) {
  if (!out || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return LS_ERR_ARG;
  *out = nullptr;
  NcclApi& a = api();
  if (!a.ok) return LS_ERR_NCCL;
  if (cudaSetDevice(device) != cudaSuccess) return LS_ERR_CUDA;
  ls_comm* c = new ls_comm();
  c->device = device;
  c->rank = rank;
  c->nranks = nranks;
  NcclUniqueId id;
  std::memcpy(&id, id128, sizeof(id));
  if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess ||
      c->d_send.reserve(1, 1) != cudaSuccess || c->d_recv.reserve((size_t)nranks, (size_t)nranks) != cudaSuccess ||
      c->h_pinned.reserve((size_t)nranks + 1, (size_t)nranks + 1) != cudaSuccess) {
    ls_comm_destroy(c);
    return LS_ERR_CUDA;
  }
  const int rc = a.comm_init_rank(&c->comm, nranks, id, rank);
  if (rc != 0) {
    ls_comm_destroy(c);
    return LS_ERR_NCCL;
  }
  *out = c;
  return LS_OK;
}

void ls_comm_destroy(ls_comm* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  if (c->comm && api().ok) api().comm_destroy(c->comm);
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;
}

const char* ls_comm_last_error(const ls_comm* c) { return c ? c->err.c_str() : "null communicator"; }

int ls_comm_allgather_pose_records_begin(ls_comm* c, const ls_pose_record* mine) {
  if (!c || !mine) return LS_ERR_ARG;
  if (c->pending) return LS_ERR_STATE;
  if (cudaSetDevice(c->device) != cudaSuccess) return LS_ERR_CUDA;
  c->h_pinned.get()[0] = *mine;
  if (cudaMemcpyAsync(c->d_send.get(), c->h_pinned.get(), sizeof(ls_pose_record), cudaMemcpyHostToDevice,
                      c->stream) != cudaSuccess)
    return LS_ERR_CUDA;
  const int rc = api().all_gather(c->d_send.get(), c->d_recv.get(), sizeof(ls_pose_record), 0 /* ncclInt8 */, c->comm, c->stream);
  if (rc != 0) {
    c->err = api().get_error_string ? api().get_error_string(rc) : "ncclAllGather failed";
    return LS_ERR_NCCL;
  }
  if (cudaMemcpyAsync(c->h_pinned.get() + 1, c->d_recv.get(), sizeof(ls_pose_record) * (size_t)c->nranks, cudaMemcpyDeviceToHost,
                      c->stream) !=
      cudaSuccess)
    return LS_ERR_CUDA;
  c->pending = true;
  return LS_OK;
}

int ls_comm_allgather_pose_records_end(ls_comm* c, ls_pose_record* all) {
  if (!c || !all) return LS_ERR_ARG;
  if (!c->pending) return LS_ERR_STATE;
  if (cudaSetDevice(c->device) != cudaSuccess) return LS_ERR_CUDA;
  c->pending = false;
  if (cudaStreamSynchronize(c->stream) != cudaSuccess) return LS_ERR_CUDA;
  std::memcpy(all, c->h_pinned.get() + 1, sizeof(ls_pose_record) * (size_t)c->nranks);
  return LS_OK;
}

int ls_comm_allgather_pose_records(ls_comm* c, const ls_pose_record* mine, ls_pose_record* all) {
  const int rc = ls_comm_allgather_pose_records_begin(c, mine);
  return rc != LS_OK ? rc : ls_comm_allgather_pose_records_end(c, all);
}

}  // extern "C"
