// Robot models: the C-ABI (hfb_robot_*) and its kernel.  The kernel (hfb_robot_poses, hfb_robot_sample_motions): one
// thread per (configuration, link) walks the link's path from the root (hfb_kin.cuh), so the only state is one frame in
// registers and no thread waits on another.
#include <algorithm>
#include <memory>
#include <mutex>
#include <new>

#include "hfb_ctx.h"
#include "hfb_broadphase.cuh"
#include "hfb_robot.h"

namespace hfb {

namespace {

// the motion of configuration g: the largest m with off[m] <= g (off[0] = 0 <= g < off[n_motions] = n_configs, so
// off[m] <= g < off[m + 1] and empty motions are skipped)
__device__ __forceinline__ uint32_t motion_of(const uint32_t* off, uint32_t n_motions, uint32_t g) {
  uint32_t lo = 0, hi = n_motions;
  while (hi - lo > 1) {
    const uint32_t mid = lo + (hi - lo) / 2;
    if (__ldg(off + mid) <= g) lo = mid;
    else hi = mid;
  }
  return lo;
}

template <bool SAMPLE>
__global__ void __launch_bounds__(256) k_robot(const KinArgs a) {
  const size_t n = a.n_configs * a.L;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += stride) {
    const uint32_t g = (uint32_t)(t / a.L), i = (uint32_t)(t % a.L);
    const KinLink link = a.links[i];
    const uint32_t J = a.J;
    hfb_transform tf;
    if (SAMPLE) {
      const uint32_t m = motion_of(a.off, a.n_motions, g);
      const uint32_t o = __ldg(a.off + m);
      const uint32_t k = g - o, ns = __ldg(a.off + m + 1) - o;
      const double* from = a.q_from + (size_t)m * J;
      const double* to = a.q_to + (size_t)m * J;
      auto q0 = [&](uint32_t j) { return kin_sample(__ldg(from + j), __ldg(to + j), k, ns); };
      kin_link_pose(a.joints, link, a.path_list, q0, tf);
      if (a.sweep) {
        auto q1 = [&](uint32_t j) { return kin_sample(__ldg(from + j), __ldg(to + j), k + 1, ns); };
        a.sweep[t] = k + 1 < ns ? kin_link_sweep(a.joints, link, a.path_list, J, q0, q1) : 0.0;
      }
      if (a.q_out)
        for (uint32_t j = i; j < J; j += a.L) a.q_out[(size_t)g * J + j] = q0(j);
    } else {
      const double* q = a.q + (size_t)g * J;
      auto qg = [&](uint32_t j) { return __ldg(q + j); };
      kin_link_pose(a.joints, link, a.path_list, qg, tf);
    }
    a.tfs[t] = tf;
    if (a.handles) a.handles[t] = link.handle;
  }
}

// hfb_env_validate_motions' samples: one thread per (sample, link) as k_robot, at the sample's dyadic position
__global__ void __launch_bounds__(256) k_robot_at(const KinAtArgs a) {
  const size_t n = a.n_samples * a.L;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += stride) {
    const uint32_t g = (uint32_t)(t / a.L), i = (uint32_t)(t % a.L);
    const KinLink link = a.links[i];
    const uint32_t J = a.J, m = __ldg(a.m + g), k = __ldg(a.k + g);
    const double* from = a.q_from + (size_t)m * J;
    const double* to = a.q_to + (size_t)m * J;
    auto q0 = [&](uint32_t j) { return kin_sample(__ldg(from + j), __ldg(to + j), k, a.n_pos); };
    hfb_transform tf;
    kin_link_pose(a.joints, link, a.path_list, q0, tf);
    if (a.sweep) {
      auto q1 = [&](uint32_t j) { return kin_sample(__ldg(from + j), __ldg(to + j), k + a.len, a.n_pos); };
      a.sweep[t] = __ldg(a.seg + g) ? kin_link_sweep(a.joints, link, a.path_list, J, q0, q1) : 0.0;
    }
    a.tfs[t] = tf;
    a.handles[t] = link.handle;
  }
}

}  // namespace

int robot_at_launch(const KinAtArgs& a, int num_sms, cudaStream_t s) {
  const size_t n = a.n_samples * a.L;
  if (n == 0) return cudaSuccess;
  const size_t cap = (size_t)(num_sms > 0 ? num_sms : 1) * 8;
  const unsigned blocks = (unsigned)((n + 255) / 256 < cap ? (n + 255) / 256 : cap);
  k_robot_at<<<blocks, 256, 0, s>>>(a);
  return (int)cudaGetLastError();
}

int robot_launch(const KinArgs& a, bool sample, int num_sms, cudaStream_t s) {
  const size_t n = a.n_configs * a.L;
  if (n == 0) return cudaSuccess;
  // a grid-stride loop: no grid limit bounds n (8 blocks of 256 threads per SM keep every SM busy)
  const size_t cap = (size_t)(num_sms > 0 ? num_sms : 1) * 8;
  const unsigned blocks = (unsigned)((n + 255) / 256 < cap ? (n + 255) / 256 : cap);
  if (sample)
    k_robot<true><<<blocks, 256, 0, s>>>(a);
  else
    k_robot<false><<<blocks, 256, 0, s>>>(a);
  return (int)cudaGetLastError();
}

}  // namespace hfb

// ---- robot models (hfb_robot_*): forward kinematics, motion sampling and sweep bounds on the device ----------------
namespace {

// checks that need no context: the description's pointers, counts and model (hfb::kin_check, which allocates nothing)
int robot_desc_ok(const hfb_robot_desc* d) {
  if (!d || !d->parent || !d->type || !d->axis || !d->placement || !d->link_joint || !d->link_placement ||
      !d->link_handles)
    return HFB_ERR_INVALID_ARGUMENT;
  return hfb::kin_check(d) ? HFB_ERR_INVALID_ARGUMENT : HFB_OK;
}

// a link handle must name a committed shape that was not released
int robot_handles(hfb_ctx* ctx, const uint32_t* h, size_t n) {
  if (int rc = check_handles(ctx, h, n)) return rc;
  for (size_t i = 0; i < n; ++i)
    if (ctx->arena.shapes[h[i]].type == 0) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "a link's shape was released");
  return HFB_OK;
}

// the links' reach from the committed local boxes
void robot_reach(hfb_ctx* ctx, hfb_robot* r) {
  for (hfb::KinLink& k : r->links) k.reach = hfb::kin_link_reach(k, ctx->local_aabbs.data() + 6 * (size_t)k.handle);
}

}  // namespace

// a robot of this context whose geometry is still valid: as env_ready, plus the links' reach read again after a commit
int robot_ready(hfb_ctx* ctx, hfb_robot* r) {
  if (std::find(ctx->robots.begin(), ctx->robots.end(), r) == ctx->robots.end())
    return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "not a robot of this context");
  if (r->clears != ctx->clears)
    return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "the geometry was cleared since the robot was created (hfb_geom_clear)");
  if (int rc = check_ready(ctx)) return rc;
  if (r->commits != ctx->commits) {
    const size_t ns = ctx->arena.shapes.size();
    for (const hfb::KinLink& k : r->links) {
      if (k.handle >= ns) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "shape handle out of range");
      if (ctx->arena.shapes[k.handle].type == 0) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "a link's shape was released");
    }
    robot_reach(ctx, r);
    r->links_stale = true;
    r->commits = ctx->commits;
  }
  return HFB_OK;
}

int robot_model_args(hfb_ctx* ctx, hfb_robot* r, cudaStream_t s, hfb::KinAtArgs* a) {
  if (r->links_stale) {
    CK(cudaMemcpyAsync(static_cast<char*>(r->model.p) + r->links_at, r->links.data(), r->L * sizeof(hfb::KinLink),
                       cudaMemcpyHostToDevice, s));
    r->links_stale = false;
  }
  a->joints = static_cast<const hfb::KinJoint*>(r->model.p);
  a->links = reinterpret_cast<const hfb::KinLink*>(static_cast<char*>(r->model.p) + r->links_at);
  a->path_list = static_cast<const uint8_t*>(r->model.p) + r->path_at;
  a->J = r->J;
  a->L = r->L;
  return HFB_OK;
}

namespace {

// hfb_robot_poses and hfb_robot_sample_motions in both forms.  Sampling when `off` is not null: q and q_to are the
// motions' end points, n_configs = off[n_motions].  Host form (dev == false): every pointer is host memory, the call
// runs on the context's first stream and blocks; device form: device memory (the offsets excepted), ordered on `stream`.
int robot_call(hfb_ctx* ctx, hfb_robot* r, bool dev, void* stream, size_t n_configs, const double* q, const double* q_to,
               size_t n_motions, const uint32_t* off, hfb_transform* tfs, uint32_t* handles, double* q_out,
               double* sweep) {
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (int rc = robot_ready(ctx, r)) return rc;
  if (n_configs > 0xffffffffull / r->L) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "n_configs * num_links >= 2^32");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = dev ? static_cast<cudaStream_t>(stream) : ctx->slots[0].stream;
  if (int rc = after_device_calls(ctx, s)) return rc;
  if (r->links_stale) {
    CK(cudaMemcpyAsync(static_cast<char*>(r->model.p) + r->links_at, r->links.data(), r->L * sizeof(hfb::KinLink),
                       cudaMemcpyHostToDevice, s));
    r->links_stale = false;
  }
  const size_t n = n_configs * r->L, J = r->J;
  if (n) {
    const bool sample = off != nullptr;
    const size_t nq_in = sample ? n_motions * J : n_configs * J;
    hfb::KinArgs a{};
    a.joints = static_cast<const hfb::KinJoint*>(r->model.p);
    a.links = reinterpret_cast<const hfb::KinLink*>(static_cast<char*>(r->model.p) + r->links_at);
    a.path_list = static_cast<const uint8_t*>(r->model.p) + r->path_at;
    a.J = r->J;
    a.L = r->L;
    a.n_configs = n_configs;
    a.n_motions = (uint32_t)n_motions;
    if (sample) {
      CK(r->off.reserve((n_motions + 1) * 4));
      CK(cudaMemcpyAsync(r->off.p, off, (n_motions + 1) * 4, cudaMemcpyHostToDevice, s));
      a.off = static_cast<const uint32_t*>(r->off.p);
    }
    if (dev) {
      a.q = sample ? nullptr : q;
      a.q_from = sample ? q : nullptr;
      a.q_to = q_to;
      a.tfs = tfs;
      a.handles = handles;
      a.q_out = q_out;
      a.sweep = sweep;
    } else {
      CK(r->q_in.reserve(nq_in * (sample ? 2 : 1) * 8 + 8));
      double* d_q = static_cast<double*>(r->q_in.p);
      CK(cudaMemcpyAsync(d_q, q, nq_in * 8, cudaMemcpyHostToDevice, s));
      if (sample) CK(cudaMemcpyAsync(d_q + nq_in, q_to, nq_in * 8, cudaMemcpyHostToDevice, s));
      a.q = sample ? nullptr : d_q;
      a.q_from = sample ? d_q : nullptr;
      a.q_to = sample ? d_q + nq_in : nullptr;
      CK(r->tfs.reserve(n * sizeof(hfb_transform)));
      a.tfs = static_cast<hfb_transform*>(r->tfs.p);
      if (handles) {
        CK(r->handles.reserve(n * 4));
        a.handles = static_cast<uint32_t*>(r->handles.p);
      }
      if (q_out) {
        CK(r->q_out.reserve(n_configs * J * 8));
        a.q_out = static_cast<double*>(r->q_out.p);
      }
      if (sweep) {
        CK(r->sweep.reserve(n * 8));
        a.sweep = static_cast<double*>(r->sweep.p);
      }
    }
    {
      KTimer kt(ctx, s, 2);
      if (int e = hfb::robot_launch(a, sample, ctx->num_sms, s))
        return cuda_fail(ctx, static_cast<cudaError_t>(e), "k_robot launch");
    }
    ctx->stats.kernel_launches++;
    if (!dev) {
      CK(cudaMemcpyAsync(tfs, a.tfs, n * sizeof(hfb_transform), cudaMemcpyDeviceToHost, s));
      if (handles) CK(cudaMemcpyAsync(handles, a.handles, n * 4, cudaMemcpyDeviceToHost, s));
      if (q_out) CK(cudaMemcpyAsync(q_out, a.q_out, n_configs * J * 8, cudaMemcpyDeviceToHost, s));
      if (sweep) CK(cudaMemcpyAsync(sweep, a.sweep, n * 8, cudaMemcpyDeviceToHost, s));
    }
  }
  if (dev) return last_device_call(ctx, s);
  CK(cudaStreamSynchronize(s));
  return HFB_OK;
}

}  // namespace

extern "C" {

// Pinocchio's Model + GeometryModel for a tree of 1-DoF joints: forwardKinematics + updateGeometryPlacements on the
// device (include/hppfcl_b200.h states the model, the semantics and the sweep bounds)
int hfb_robot_create(hfb_ctx* ctx, const hfb_robot_desc* desc, hfb_robot** out) {
  if (!ctx || !out) return HFB_ERR_INVALID_ARGUMENT;
  if (int rc = robot_desc_ok(desc)) return rc;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (int rc = check_ready(ctx)) return rc;
  if (int rc = robot_handles(ctx, desc->link_handles, desc->num_links)) return rc;
  std::unique_ptr<hfb_robot> r(new hfb_robot);
  r->J = desc->num_joints;
  r->L = desc->num_links;
  try {  // (L * J <= UINT32_MAX links' worth of host copies: a large model may not fit)
    r->joints.resize(r->J);
    r->links.resize(r->L);
    r->path_list.resize((size_t)r->L * r->J);
  } catch (const std::bad_alloc&) {
    return fail(ctx, HFB_ERR_OUT_OF_MEMORY, "robot model: host memory");
  }
  hfb::kin_prepare(desc, nullptr, r->joints.data(), r->links.data(), r->path_list.data());
  robot_reach(ctx, r.get());
  r->commits = ctx->commits;
  r->clears = ctx->clears;
  r->links_at = r->J * sizeof(hfb::KinJoint);
  r->path_at = r->links_at + r->L * sizeof(hfb::KinLink);
  CK(cudaSetDevice(ctx->device));
  CK(r->model.reserve(r->path_at + r->path_list.size()));
  char* m = static_cast<char*>(r->model.p);
  CK(cudaMemcpy(m, r->joints.data(), r->links_at, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(m + r->links_at, r->links.data(), r->L * sizeof(hfb::KinLink), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(m + r->path_at, r->path_list.data(), r->path_list.size(), cudaMemcpyHostToDevice));
  ctx->robots.push_back(r.get());
  *out = r.release();
  return HFB_OK;
}

int hfb_robot_destroy(hfb_ctx* ctx, hfb_robot* robot) {
  if (!ctx || !robot) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  auto it = std::find(ctx->robots.begin(), ctx->robots.end(), robot);
  if (it == ctx->robots.end()) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "not a robot of this context");
  CK(cudaSetDevice(ctx->device));
  // what may still read its model: the last device call and the host calls' stream
  if (ctx->dev_used) CK(cudaEventSynchronize(ctx->dev_done));
  CK(cudaStreamSynchronize(ctx->slots[0].stream));
  ctx->robots.erase(it);
  delete robot;
  return HFB_OK;
}

int hfb_robot_poses(hfb_ctx* ctx, hfb_robot* robot, size_t n_configs, const double* q, hfb_transform* tfs,
                    uint32_t* handles) {
  if (!ctx || !robot || (n_configs && (!q || !tfs))) return HFB_ERR_INVALID_ARGUMENT;
  return robot_call(ctx, robot, false, nullptr, n_configs, q, nullptr, 0, nullptr, tfs, handles, nullptr, nullptr);
}

int hfb_robot_poses_device(hfb_ctx* ctx, hfb_robot* robot, size_t n_configs, const double* d_q, hfb_transform* d_tfs,
                           uint32_t* d_handles, void* stream) {
  if (!ctx || !robot || (n_configs && (!d_q || !d_tfs))) return HFB_ERR_INVALID_ARGUMENT;
  return robot_call(ctx, robot, true, stream, n_configs, d_q, nullptr, 0, nullptr, d_tfs, d_handles, nullptr, nullptr);
}

int hfb_robot_sample_motions(hfb_ctx* ctx, hfb_robot* robot, size_t n_motions, const double* q_from, const double* q_to,
                             const uint32_t* motion_offsets, const hfb_robot_samples_out* out) {
  if (!ctx || !robot || !out || (n_motions && (!q_from || !q_to))) return HFB_ERR_INVALID_ARGUMENT;
  if (!motion_offsets || motion_offsets_error(n_motions, motion_offsets)) return HFB_ERR_INVALID_ARGUMENT;
  const size_t n_configs = motion_offsets[n_motions];
  if (n_configs && (!out->tfs || !out->handles)) return HFB_ERR_INVALID_ARGUMENT;
  return robot_call(ctx, robot, false, nullptr, n_configs, q_from, q_to, n_motions, motion_offsets, out->tfs,
                    out->handles, out->q, out->sweep);
}

int hfb_robot_sample_motions_device(hfb_ctx* ctx, hfb_robot* robot, size_t n_motions, const double* d_q_from,
                                    const double* d_q_to, const uint32_t* motion_offsets,
                                    const hfb_robot_samples_out* d_out, void* stream) {
  if (!ctx || !robot || !d_out || (n_motions && (!d_q_from || !d_q_to))) return HFB_ERR_INVALID_ARGUMENT;
  if (!motion_offsets || motion_offsets_error(n_motions, motion_offsets)) return HFB_ERR_INVALID_ARGUMENT;
  const size_t n_configs = motion_offsets[n_motions];
  if (n_configs && (!d_out->tfs || !d_out->handles)) return HFB_ERR_INVALID_ARGUMENT;
  return robot_call(ctx, robot, true, stream, n_configs, d_q_from, d_q_to, n_motions, motion_offsets, d_out->tfs,
                    d_out->handles, d_out->q, d_out->sweep);
}

}  // extern "C"
