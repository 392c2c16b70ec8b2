// The robot-model kernel (hfb_robot_poses, hfb_robot_sample_motions): one thread per (configuration, link) walks the
// link's path from the root (hfb_kin.cuh), so the only state is one frame in registers and no thread waits on another.
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

}  // namespace

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
