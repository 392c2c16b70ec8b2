// The multi-GPU C-ABI: hfb_comm_*, hfb_geom_broadcast and the sharded batch calls.
//
// One process (or thread) per GPU, one context per rank.  The path shards trivially -- pairs are independent -- so
// there are exactly two collectives: one broadcast of the geometry arena per scene and one all-gather of the result
// records per batch (SURVEY 8e).  NCCL is reached through dlopen: the library has no link-time dependency on it and
// shares whatever libnccl.so.2 the process has loaded already (torch's, when the caller is a torch.distributed job).
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "hfb_ctx.h"

struct ncclUniqueIdPOD {
  char internal[128];
};

namespace {
struct NcclApi {
  typedef int (*get_id_t)(void*);
  typedef int (*init_t)(void**, int, ncclUniqueIdPOD, int);
  typedef int (*destroy_t)(void*);
  typedef int (*bcast_t)(const void*, void*, size_t, int, int, void*, cudaStream_t);
  typedef int (*allgather_t)(const void*, void*, size_t, int, void*, cudaStream_t);
  typedef const char* (*errstr_t)(int);
  get_id_t get_id = nullptr;
  init_t init = nullptr;
  destroy_t destroy = nullptr;
  bcast_t bcast = nullptr;
  allgather_t allgather = nullptr;
  errstr_t errstr = nullptr;
  bool ok = false;
};
NcclApi& nccl() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return;
    api.get_id = (NcclApi::get_id_t)dlsym(h, "ncclGetUniqueId");
    api.init = (NcclApi::init_t)dlsym(h, "ncclCommInitRank");
    api.destroy = (NcclApi::destroy_t)dlsym(h, "ncclCommDestroy");
    api.bcast = (NcclApi::bcast_t)dlsym(h, "ncclBroadcast");
    api.allgather = (NcclApi::allgather_t)dlsym(h, "ncclAllGather");
    api.errstr = (NcclApi::errstr_t)dlsym(h, "ncclGetErrorString");
    api.ok = api.get_id && api.init && api.destroy && api.bcast && api.allgather && api.errstr;
  });
  return api;
}
int nccl_fail(hfb_ctx* c, int rc, const char* where) {
  return fail(c, HFB_ERR_CUDA, std::string(where) + ": NCCL: " + (nccl().errstr ? nccl().errstr(rc) : "?"));
}
#define NK(call)                                         \
  do {                                                   \
    const int _r = (call);                               \
    if (_r != 0) return nccl_fail(ctx, _r, #call);       \
  } while (0)
constexpr int kNcclChar = 0;  // ncclInt8 / ncclChar

// the host arena as one blob (what hfb_geom_broadcast sends)
template <class T>
void put_vec(std::vector<unsigned char>& b, const std::vector<T>& v) {
  const uint64_t n = v.size();
  const size_t at = b.size();
  b.resize(at + 8 + n * sizeof(T));
  std::memcpy(b.data() + at, &n, 8);
  if (n) std::memcpy(b.data() + at + 8, v.data(), n * sizeof(T));
}
template <class T>
bool get_vec(const unsigned char*& p, const unsigned char* end, std::vector<T>& v) {
  if (end - p < 8) return false;
  uint64_t n;
  std::memcpy(&n, p, 8);
  p += 8;
  if ((uint64_t)(end - p) < n * sizeof(T)) return false;
  v.resize(n);
  if (n) std::memcpy(v.data(), p, n * sizeof(T));
  p += n * sizeof(T);
  return true;
}
}  // namespace

extern "C" {

int hfb_comm_unique_id(hfb_comm_id* id) {
  if (!id) return HFB_ERR_INVALID_ARGUMENT;
  if (!nccl().ok) return HFB_ERR_NO_DEVICE;
  return nccl().get_id(id) == 0 ? HFB_OK : HFB_ERR_CUDA;
}

int hfb_comm_init(hfb_ctx* ctx, const hfb_comm_id* id, int rank, int nranks) {
  if (!ctx || !id || nranks < 1 || rank < 0 || rank >= nranks) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!nccl().ok) return fail(ctx, HFB_ERR_NO_DEVICE, "libnccl.so.2 not found");
  if (ctx->comm) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "communicator already initialised");
  CK(cudaSetDevice(ctx->device));
  ncclUniqueIdPOD u;
  std::memcpy(&u, id, sizeof(u));
  NK(nccl().init(&ctx->comm, nranks, u, rank));
  ctx->comm_rank = rank;
  ctx->comm_nranks = nranks;
  CK(cudaStreamCreateWithFlags(&ctx->comm_stream, cudaStreamNonBlocking));
  for (int k = 0; k < 2; ++k) {
    CK(cudaEventCreateWithFlags(&ctx->comm_computed[k], cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&ctx->comm_gathered[k], cudaEventDisableTiming));
  }
  return HFB_OK;
}

int hfb_comm_destroy(hfb_ctx* ctx) {
  if (!ctx) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->comm) return HFB_OK;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  nccl().destroy(ctx->comm);
  ctx->comm = nullptr;
  for (int k = 0; k < 2; ++k) {
    if (ctx->comm_computed[k]) cudaEventDestroy(ctx->comm_computed[k]);
    if (ctx->comm_gathered[k]) cudaEventDestroy(ctx->comm_gathered[k]);
    ctx->comm_computed[k] = ctx->comm_gathered[k] = nullptr;
    ctx->comm_all[k].release();
  }
  ctx->comm_blob.release();
  if (ctx->comm_stream) cudaStreamDestroy(ctx->comm_stream);
  ctx->comm_stream = nullptr;
  ctx->comm_nranks = 1;
  ctx->comm_rank = 0;
  return HFB_OK;
}

// the geometry registered on `root` replaces what this context holds, on every rank, and is committed: ONE broadcast
// of the arena (a second, 8-byte one carries its size)
int hfb_geom_broadcast(hfb_ctx* ctx, int root) {
  if (!ctx) return HFB_ERR_INVALID_ARGUMENT;
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!ctx->comm) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "no communicator (hfb_comm_init)");
    if (root < 0 || root >= ctx->comm_nranks) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "bad root");
    CK(cudaSetDevice(ctx->device));
    std::vector<unsigned char> blob;
    if (ctx->comm_rank == root) {
      const HostArena& A = ctx->arena;
      put_vec(blob, A.shapes);
      put_vec(blob, A.cvx);
      put_vec(blob, A.pool);
      put_vec(blob, A.bvh_nodes);
      put_vec(blob, A.bvh_verts);
      put_vec(blob, A.bvh_tris);
      put_vec(blob, A.bvh_desc);
      const int32_t flags[5] = {A.has_convex, A.has_tri, A.has_unknown, A.has_bvh, A.max_bvh_depth};
      const size_t at = blob.size();
      blob.resize(at + sizeof(flags));
      std::memcpy(blob.data() + at, flags, sizeof(flags));
    }
    unsigned long long size = blob.size();
    CK(ctx->comm_blob.reserve(8));
    CK(cudaMemcpy(ctx->comm_blob.p, &size, 8, cudaMemcpyHostToDevice));
    NK(nccl().bcast(ctx->comm_blob.p, ctx->comm_blob.p, 8, kNcclChar, root, ctx->comm, ctx->comm_stream));
    CK(cudaStreamSynchronize(ctx->comm_stream));
    CK(cudaMemcpy(&size, ctx->comm_blob.p, 8, cudaMemcpyDeviceToHost));
    CK(ctx->comm_blob.reserve(size + 8));
    if (ctx->comm_rank == root) CK(cudaMemcpy(ctx->comm_blob.p, blob.data(), size, cudaMemcpyHostToDevice));
    NK(nccl().bcast(ctx->comm_blob.p, ctx->comm_blob.p, size, kNcclChar, root, ctx->comm, ctx->comm_stream));
    CK(cudaStreamSynchronize(ctx->comm_stream));
    if (ctx->comm_rank != root) {
      blob.resize(size);
      CK(cudaMemcpy(blob.data(), ctx->comm_blob.p, size, cudaMemcpyDeviceToHost));
      HostArena A;
      const unsigned char* p = blob.data();
      const unsigned char* end = p + blob.size();
      int32_t flags[5];
      if (!get_vec(p, end, A.shapes) || !get_vec(p, end, A.cvx) || !get_vec(p, end, A.pool) || !get_vec(p, end, A.bvh_nodes) ||
          !get_vec(p, end, A.bvh_verts) || !get_vec(p, end, A.bvh_tris) || !get_vec(p, end, A.bvh_desc) ||
          (size_t)(end - p) != sizeof(flags))
        return fail(ctx, HFB_ERR_CUDA, "malformed arena blob");
      std::memcpy(flags, p, sizeof(flags));
      A.has_convex = flags[0] != 0;
      A.has_tri = flags[1] != 0;
      A.has_unknown = flags[2] != 0;
      A.has_bvh = flags[3] != 0;
      A.max_bvh_depth = flags[4];
      ctx->arena = std::move(A);
      ctx->committed = false;
    }
  }
  return hfb_geom_commit(ctx);
}

// this rank's n_local pairs (device rows) -> the records of ALL ranks' pairs, rank-major, on every rank: the batch
// runs on `stream` into this rank's slice of one of two context-owned buffers, the all-gather runs on the
// communicator's own stream and overlaps the NEXT call's kernels.  *d_all: the gathered buffer
// (nranks * n_local records), complete once `stream` has passed hfb_comm_wait.  Every rank passes the same n_local.
static int sharded_prologue(hfb_ctx* ctx, size_t n_local, size_t rec, int* b, unsigned char** mine) {
  if (!ctx->comm) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "no communicator (hfb_comm_init)");
  *b = (int)(ctx->comm_calls++ & 1u);
  CK(ctx->comm_all[*b].reserve(n_local * rec * (size_t)ctx->comm_nranks));
  *mine = static_cast<unsigned char*>(ctx->comm_all[*b].p) + (size_t)ctx->comm_rank * n_local * rec;
  return HFB_OK;
}
static int sharded_epilogue(hfb_ctx* ctx, int b, size_t n_local, size_t rec, cudaStream_t st, void** d_all) {
  CK(cudaEventRecord(ctx->comm_computed[b], st));
  CK(cudaStreamWaitEvent(ctx->comm_stream, ctx->comm_computed[b], 0));
  unsigned char* base = static_cast<unsigned char*>(ctx->comm_all[b].p);
  NK(nccl().allgather(base + (size_t)ctx->comm_rank * n_local * rec, base, n_local * rec, kNcclChar, ctx->comm, ctx->comm_stream));
  CK(cudaEventRecord(ctx->comm_gathered[b], ctx->comm_stream));
  if (d_all) *d_all = base;
  return HFB_OK;
}

int hfb_batch_distance_sharded_device(hfb_ctx* ctx, size_t n_local, const uint32_t* h1, const hfb_transform* tf1,
                                      const uint32_t* h2, const hfb_transform* tf2, const hfb_distance_request* req,
                                      hfb_distance_result** d_all, void* stream) {
  if (!ctx || !req) return HFB_ERR_INVALID_ARGUMENT;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int b;
  unsigned char* mine;
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (int rc = sharded_prologue(ctx, n_local, sizeof(hfb_distance_result), &b, &mine)) return rc;
    // the buffer's previous all-gather (two calls ago) has read it before this batch overwrites the slice
    CK(cudaStreamWaitEvent(st, ctx->comm_gathered[b], 0));
  }
  if (int rc = hfb_batch_distance_device(ctx, n_local, h1, tf1, h2, tf2, req, reinterpret_cast<hfb_distance_result*>(mine), nullptr, stream))
    return rc;
  std::lock_guard<std::mutex> lk(ctx->mu);
  return sharded_epilogue(ctx, b, n_local, sizeof(hfb_distance_result), st, reinterpret_cast<void**>(d_all));
}

int hfb_batch_collide_sharded_device(hfb_ctx* ctx, size_t n_local, const uint32_t* h1, const hfb_transform* tf1,
                                     const uint32_t* h2, const hfb_transform* tf2, const hfb_collision_request* req,
                                     hfb_contact** d_all, void* stream) {
  if (!ctx || !req) return HFB_ERR_INVALID_ARGUMENT;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int b;
  unsigned char* mine;
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (int rc = sharded_prologue(ctx, n_local, sizeof(hfb_contact), &b, &mine)) return rc;
    CK(cudaStreamWaitEvent(st, ctx->comm_gathered[b], 0));
  }
  if (int rc = hfb_batch_collide_device(ctx, n_local, h1, tf1, h2, tf2, req, reinterpret_cast<hfb_contact*>(mine), nullptr, stream))
    return rc;
  std::lock_guard<std::mutex> lk(ctx->mu);
  return sharded_epilogue(ctx, b, n_local, sizeof(hfb_contact), st, reinterpret_cast<void**>(d_all));
}

// `stream` waits for every all-gather this context has enqueued
int hfb_comm_wait(hfb_ctx* ctx, void* stream) {
  if (!ctx) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->comm) return HFB_OK;
  for (int k = 0; k < 2; ++k) CK(cudaStreamWaitEvent(static_cast<cudaStream_t>(stream), ctx->comm_gathered[k], 0));
  return HFB_OK;
}

}  // extern "C"
