// TEST HARNESS ONLY -- not part of the product and never loaded by it.
//
// The robot-model kinematics of hpp-fcl_b200/csrc/hfb_kin.cuh compiled with g++ (-ffp-contract=off), so that the
// exact arithmetic of the device kernel k_robot (hfb_robot.cu) can be checked against numpy without a GPU, and the
// device's outputs against these bit for bit on a GPU box.  Each call checks the model with hfb::kin_check and lays it
// out with hfb::kin_prepare, as hfb_robot_create does; `boxes` are the links' local boxes (6 doubles each), what
// hfb_geom_commit tabulates.
#include <cstdio>
#include <vector>

#include "../../hpp-fcl_b200/csrc/hfb_kin.cuh"

using namespace hfb;

namespace {

struct Model {
  std::vector<KinJoint> joints;
  std::vector<KinLink> links;
  std::vector<uint8_t> path;
  bool ok = false;
  Model(const hfb_robot_desc* d, const double* boxes) {
    if (kin_check(d)) return;
    joints.resize(d->num_joints);
    links.resize(d->num_links);
    path.resize((size_t)d->num_joints * d->num_links);
    kin_prepare(d, boxes, joints.data(), links.data(), path.data());
    ok = true;
  }
};

}  // namespace

extern "C" {

void kin_sincos(size_t n, const double* x, double* s, double* c) {
  for (size_t i = 0; i < n; ++i) hfb_sincos(x[i], s + i, c + i);
}

// hfb_robot_poses: n_configs x J joint values -> n_configs * L poses
int kin_poses(const hfb_robot_desc* d, const double* boxes, size_t n_configs, const double* q, hfb_transform* tfs) {
  Model m(d, boxes);
  if (!m.ok) return 1;
  const uint32_t J = d->num_joints, L = d->num_links;
  for (size_t g = 0; g < n_configs; ++g) {
    const double* qg = q + g * J;
    auto qf = [&](uint32_t j) { return qg[j]; };
    for (uint32_t i = 0; i < L; ++i) kin_link_pose(m.joints.data(), m.links[i], m.path.data(), qf, tfs[g * L + i]);
  }
  return 0;
}

// hfb_robot_sample_motions: the motions' samples -> poses, joint values and sweep bounds (q_out, sweep may be null)
int kin_sample_motions(const hfb_robot_desc* d, const double* boxes, size_t n_motions, const double* q_from,
                       const double* q_to, const uint32_t* off, hfb_transform* tfs, double* q_out, double* sweep) {
  Model m(d, boxes);
  if (!m.ok) return 1;
  const uint32_t J = d->num_joints, L = d->num_links;
  for (size_t mo = 0; mo < n_motions; ++mo) {
    const uint32_t ns = off[mo + 1] - off[mo];
    const double* from = q_from + mo * J;
    const double* to = q_to + mo * J;
    for (uint32_t k = 0; k < ns; ++k) {
      const size_t g = off[mo] + k;
      auto q0 = [&](uint32_t j) { return kin_sample(from[j], to[j], k, ns); };
      auto q1 = [&](uint32_t j) { return kin_sample(from[j], to[j], k + 1, ns); };
      if (q_out)
        for (uint32_t j = 0; j < J; ++j) q_out[g * J + j] = q0(j);
      for (uint32_t i = 0; i < L; ++i) {
        kin_link_pose(m.joints.data(), m.links[i], m.path.data(), q0, tfs[g * L + i]);
        if (sweep)
          sweep[g * L + i] = k + 1 < ns ? kin_link_sweep(m.joints.data(), m.links[i], m.path.data(), J, q0, q1) : 0.0;
      }
    }
  }
  return 0;
}

}  // extern "C"
