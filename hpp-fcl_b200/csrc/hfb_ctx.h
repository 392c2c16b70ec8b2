// The host state the C-ABI's translation units share (hfb_kernels.cu, hfb_scene.cu, hfb_robot.cu, hfb_comm.cu): the
// context and its device buffers, the resident environment and the robot model, the error and CUDA-check helpers, and
// the narrow phase of the object-table calls that the scene and environment queries run.  Not part of the public ABI.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "hfb_batch.cuh"
#include "hfb_robot.h"

// lanes per pair: pairs touching ConvexBase/TriangleP (GC: 1, 2, 4, 8, 16, 32) and the EPA kernel
// (GE: 4, 8, 16, 32).  Small groups are the defaults (the scalar part of a GJK iteration is repeated by
// every lane of the group, so small groups win until divergence between the pairs of a warp takes over
// at 1); HFB_GC / HFB_GE override them per context.
#define HFB_GC_DEFAULT 2
#define HFB_GE_DEFAULT 8

// a device allocation that grows on demand; it is freed with its owner (move-only)
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) {
    o.p = nullptr;
    o.cap = 0;
  }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) {
      release();
      p = o.p;
      cap = o.cap;
      o.p = nullptr;
      o.cap = 0;
    }
    return *this;
  }
  ~DevBuf() { release(); }
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 4 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};

constexpr int kSlots = 4;
constexpr int kMaxParts = 8;  // phase-1 launches per batch that may each be followed by an EPA launch
struct Slot {
  cudaStream_t stream = nullptr;
  // EPA of the parts of a batch that are through phase 1 runs here, next to phase 1 of the later parts
  cudaStream_t epa_stream = nullptr;
  cudaEvent_t ev_part[kMaxParts] = {};
  cudaEvent_t ev_join = nullptr;
  // GJK passes, the hull / triangle kernel and EPA of a batch run here, at the device's highest stream priority, next
  // to the closed forms on the caller's stream: the block scheduler gives free SMs to the long GJK / EPA chains first
  // and the closed-form blocks fill the tails.  ev_fork / ev_work: the fork after the class sort and the join.
  cudaStream_t work_stream = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_work = nullptr;
  DevBuf cont;  // EpaCont records (k_epa tier 0 -> tier 1)
  DevBuf sup;   // k_epa tier 0: support points, one slot per resident lane group (a slot runs one tier-0 launch at a time)
  DevBuf h1, h2, tf1, tf2, out, gin, hin, gout, hout, queue, counters, lists, retry, bvh_ws, bvh_cnt, extra, ccnt, okeys, ohist, olist;
  DevBuf qprep, qstacks, qtl, qws, qsv;  // task-system mesh-shape walk (hfb_bvhq.cu)
  DevBuf hsort;                      // hfb_hullsort.cu scratch
  DevBuf gstate, glist, gcnt;        // GJK passes (hfb_gjkpass.cu): solver state, two lists of running pairs, counts
  DevBuf pi, pj, cmp;                // object-table batches: pair indices of the chunk; compact results
};

struct hfb_ctx {
  int device = 0;
  int num_sms = 0;
  HostArena arena;
  bool committed = false;
  DevBuf d_arena;
  ArenaView dview{};
  Slot slots[kSlots];
  Slot dev_slot;  // resources of the *_device entry points (caller's stream)
  // the *_device calls of a context share dev_slot's scratch: a call enqueued on another stream than the previous one
  // first waits for it (one device call of a context in flight at a time; calls on one stream are ordered anyway)
  cudaEvent_t dev_done = nullptr;
  cudaStream_t dev_last_stream = nullptr;
  bool dev_used = false;
  DevBuf sup_ids, sup_dirs, sup_idx, sup_out;
  DevBuf obj_h, obj_tf, cmp_flags, cmp_count, cmp_ids, cmp_recs;  // object table of the running call; compact collide results
  // host pipeline (host_batch_pipelined): the whole batch on the device, EPA fix-up rows, their pinned landing zone
  DevBuf big_h1, big_h2, big_tf1, big_tf2, big_out, big_pi, big_pj, big_min, fix_ids, fix_rows;
  void* pin_fix = nullptr;
  size_t pin_fix_cap = 0;
  std::vector<cudaEvent_t> pipe_events;
  int host_pipe = 1;  // HFB_HOST_PIPE=0: the rotating-slot pipeline of round 1 for every host call
  // share of EPA pairs in the last pipelined call: a batch whose EPA is throughput-bound (config 3: half of the pairs)
  // gains nothing from one EPA pass -- the rotating slots overlap the EPA of a chunk with phase 1 of the next -- so
  // such a context goes back to them, and looks again every 16th call
  double pipe_epa_frac = 0.0;
  unsigned pipe_skipped = 0;
  cudaEvent_t obj_ready = nullptr;
  hfb_stats stats{};
  int gc = HFB_GC_DEFAULT, ge = HFB_GE_DEFAULT, minb = 1, nsub = 0, bvh_minb = 4, refill = 0, iter_quorum = 8, stage = 0, chunk = 0;
  int bvh_quorum = HFB_BVH_INIT_QUORUM;  // HFB_BVH_QUORUM=1: a lane sets its next query up as soon as it is free
  int bvh_order = 0;  // HFB_BVH_ORDER=1: hand the (mesh, shape) queries out longest-expected first
  int bvhq = 1;        // HFB_BVHQ=0: mesh-shape distance queries through the lane-per-query kernel k_bvh instead of the task system k_bvhq
  // HFB_GJK_PASSES="10" (default) or e.g. "3,3,4": iterations of the first passes of the primitive-pair GJK (one more pass runs to
  // convergence); "0": the single kernel k_pairs<1, CAP_PRIM, MODE, PATH_GJKROUTE>
  // iterations of the first pass: 10 (a pass of few iterations leaves most pairs to the next; a long one idles the lanes
  // of the pairs that converged early)
  int gjk_steps[8] = {10, 0, 0, 0, 0, 0, 0, 0};
  int gjk_npass = 2;
  // HFB_EPA_OVERLAP=1: EPA of the pairs the first GJK pass finished starts on a side stream next to the remaining passes;
  // off by default: the two kernels take each other's SMs
  int epa_overlap = 0;
  int bvh_warps = 8;   // HFB_BVH_WARPS: 8 (255 registers per thread) or 16 (128) warps per block of k_bvhq
  int bvh_gens = 2;    // HFB_BVH_GENS: generations of BV items per cycle of k_bvhq
  int bvh_spec_big = 300;  // HFB_BVH_SPEC_BIG: items more before subtrees of up to 128 triangles are speculated
  int hull_sort = 1;      // HFB_HULL_SORT: second sort key (first operand's handle) inside the hull / triangle class
  int epa_resume = 8192;  // HFB_EPA_RESUME: retries per batch that continue from the state tier 0 reached (5 KB each)
  int bvh_chunk = 6;   // HFB_BVH_GJK_CHUNK: GJK iterations a leaf item runs before it parks its state
  int bvh_spec = 200;  // HFB_BVH_SPEC: items a query uses before it may speculate on subtrees (< 0: never)
  int bvh_bps = 4;  // k_bvh: blocks (of 2 warps) per SM the grid is capped at; HFB_BVH_BPS, see tests/tools/bvh_sched_model.py
  bool profiling = false;
  struct Ev { cudaEvent_t a, b; int kind; };
  std::vector<Ev> events;
  hfb_kernel_times ktimes{};
  // per-kernel launch configuration (dynamic shared-memory opt-in, blocks per SM): function attributes are per
  // DEVICE, so the cache belongs to the context (one device), not to the process; guarded by `mu`
  std::unordered_map<const void*, int> func_cfg;
  std::vector<double> local_aabbs;  // aabb_local per shape handle, as committed (host copy)
  // multi-GPU (hfb_comm_*): the communicator of this context's rank, its stream, and the two gathered result buffers
  void* comm = nullptr;
  int comm_rank = 0, comm_nranks = 1;
  cudaStream_t comm_stream = nullptr;
  cudaEvent_t comm_computed[2] = {nullptr, nullptr}, comm_gathered[2] = {nullptr, nullptr};
  DevBuf comm_all[2], comm_blob;
  unsigned comm_calls = 0;
  DevBuf bp_scratch;                // device broadphase
  DevBuf sc_bb, sc_pf, sc_ps, sc_cnt, sc_out, sc_f, sc_s, sc_rec;  // hfb_scene_collide
  DevBuf sc_flags;                                                 // hfb_env_collide
  DevBuf sc_tpl;                                                   // hfb_env_collide_configs: the self-pair template
  DevBuf sc_dist, sc_drec;  // hfb_env_distance: the per-A state (hfb::BpDistState), a round's distance() records
  DevBuf sc_cdist;          // hfb_env_distance_configs: the per-configuration state (hfb::BpConfigDist)
  DevBuf sc_moff, sc_mot;   // hfb_env_collide_motions: the motion offsets, the per-motion state (hfb::BpMotions)
  DevBuf sc_sweep, sc_side, sc_cpass;  // hfb_env_certify_motions: the sweep bounds (host form), the sides and widened
                                      // boxes of A, the per-sample pass flags (hfb::BpCertify)
  // hfb_env_validate_motions: the per-motion state and staged outputs, the open segments (two lists: this round's and
  // the next), the per-segment scans, the round's samples and runs, its counters, and CUB's scratch
  DevBuf sc_vmot, sc_vseg[2], sc_vscan, sc_vsmp, sc_vrun, sc_vcnt, sc_vcub;
  // resident environments: every hfb_geom_commit / hfb_geom_clear is counted, so that an env notices them
  std::vector<hfb_env*> envs;
  std::vector<hfb_robot*> robots;  // robot models (hfb_robot_create), checked against the same counters
  uint64_t commits = 0, clears = 0;
  std::string err;
  std::mutex mu;
};

// set B on the device (hfb_env_create): the object table with `head` free slots in front of B for A, so that a query's
// table [A; B] is contiguous without copying B; B's boxes and the persistent part of the cross grid over them
struct hfb_env {
  size_t n_b = 0, head = 0;
  DevBuf h, tf;  // (head + n_b) handles and poses, B from slot `head` on
  DevBuf bb;     // B's boxes
  DevBuf grid;   // hfb::bp_cross_grid_bytes(n_b)
  DevBuf reach;  // B's reach (hfb::bp_dist_reach_launch): 6 keys, for hfb_env_distance
  std::vector<uint32_t> handles;  // B's handles, checked again after a commit
  uint64_t commits = 0, clears = 0;  // the context's counters when B was last checked
};

// a robot model (hfb_robot_create): its joints, links and joint paths (hfb_kin.cuh) in one device buffer, the host
// copies that a commit's check and the links' reach need, and the staging buffers of the host form
struct hfb_robot {
  uint32_t J = 0, L = 0;
  std::vector<hfb::KinJoint> joints;
  std::vector<hfb::KinLink> links;
  std::vector<uint8_t> path_list;
  DevBuf model;  // joints, then links, then path_list
  size_t links_at = 0, path_at = 0;
  bool links_stale = false;  // links' reach changed on the host (a commit): uploaded in front of the next launch
  DevBuf off, q_in, tfs, handles, q_out, sweep;
  uint64_t commits = 0, clears = 0;  // the context's counters when the handles were last checked
};

// hfb_robot.cu: a robot of this context whose geometry is still valid (as env_ready; the links' reach is read again
// after a commit), and the robot's model arguments for a launch on stream s (links whose reach changed uploaded first)
int robot_ready(hfb_ctx* ctx, hfb_robot* r);
int robot_model_args(hfb_ctx* ctx, hfb_robot* r, cudaStream_t s, hfb::KinAtArgs* a);

inline int fail(hfb_ctx* c, int code, const std::string& msg) {
  if (c) c->err = msg;
  return code;
}
inline int cuda_fail(hfb_ctx* c, cudaError_t e, const char* where) {
  return fail(c, e == cudaErrorMemoryAllocation ? HFB_ERR_OUT_OF_MEMORY : HFB_ERR_CUDA,
              std::string(where) + ": " + cudaGetErrorString(e));
}
#define CK(call)                                                       \
  do {                                                                 \
    cudaError_t _e = (call);                                           \
    if (_e != cudaSuccess) return cuda_fail(ctx, _e, #call);           \
  } while (0)

// kernel timing hooks: kind 0 = GJK pairs, 1 = epa, 2 = other, 3 = closed-form pairs, 4 = convex pairs, 5 = bvh
struct KTimer {
  hfb_ctx* c;
  cudaStream_t s;
  hfb_ctx::Ev ev{};
  bool on;
  KTimer(hfb_ctx* c_, cudaStream_t s_, int kind) : c(c_), s(s_), on(c_->profiling) {
    if (!on) return;
    ev.kind = kind;
    cudaEventCreate(&ev.a);
    cudaEventCreate(&ev.b);
    cudaEventRecord(ev.a, s);
  }
  ~KTimer() {
    if (!on) return;
    cudaEventRecord(ev.b, s);
    c->events.push_back(ev);
  }
};

inline int check_ready(hfb_ctx* ctx) {
  if (!ctx) return HFB_ERR_INVALID_ARGUMENT;
  if (!ctx->committed) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "geometry not committed (hfb_geom_commit)");
  return HFB_OK;
}

// host-side handle validation (the reference dereferences caller pointers; here a
// bad handle is an invalid argument, never a device fault)
inline int check_handles(hfb_ctx* ctx, const uint32_t* h, size_t n) {
  const uint32_t ns = (uint32_t)ctx->arena.shapes.size();
  // (branch-free so that the host compiler vectorises it: this loop sits in front of every chunk's uploads)
  uint32_t bad = 0;
  for (size_t i = 0; i < n; ++i) bad |= (uint32_t)(h[i] >= ns);
  if (bad) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "shape handle out of range");
  return HFB_OK;
}

// the *_device calls may still be reading the shared scratch (dev_slot, the candidates, their records and counters of
// hfb_env_collide_device) or an env's table on another stream: a call on stream s that writes them waits for them first
inline int after_device_calls(hfb_ctx* ctx, cudaStream_t s) {
  if (!ctx->dev_done) CK(cudaEventCreateWithFlags(&ctx->dev_done, cudaEventDisableTiming));
  if (ctx->dev_used && ctx->dev_last_stream != s) CK(cudaStreamWaitEvent(s, ctx->dev_done, 0));
  return HFB_OK;
}
// the device call on s is the last one: the next call on another stream waits for what is still running here
inline int last_device_call(hfb_ctx* ctx, cudaStream_t s) {
  ctx->dev_used = true;
  ctx->dev_last_stream = s;
  CK(cudaEventRecord(ctx->dev_done, s));
  return HFB_OK;
}

// collide()'s checks of a request; *minus_inf: security_margin == -inf (no contacts)
inline int collide_prelude(hfb_ctx* ctx, const hfb_collision_request* req, bool* minus_inf) {
  if (int rc = validate_query(req->q)) return fail(ctx, rc, "invalid request");
  *minus_inf = req->security_margin == -INFINITY;
  if (!*minus_inf && req->num_max_contacts == 0)  // collision.cpp:82-85
    return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "Invalid number of max contacts (current value is 0).");
  return HFB_OK;
}

// device-resident object table: the pairs are expanded into the context's scratch rows, then the batch runs as
// hfb_batch_*_device does (hfb_kernels.cu: MODE 0 = distance() with an hfb_distance_request, MODE 1 = collide() with an
// hfb_collision_request)
template <int MODE, typename Req>
int objects_device(hfb_ctx* ctx, const hfb_object_pairs* sc, const Req* req, const SolverP& P, const CollideP& Cp,
                   const BvhReq& Bq, void* out, const hfb_guess_out* go, void* stream);
BvhReq bvh_req_of_distance(const hfb_distance_request* req);
BvhReq bvh_req_of_collision(const hfb_collision_request* req);
