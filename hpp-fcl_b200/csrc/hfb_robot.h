// Host-side interface of the robot-model kernel (hfb_robot.cu; the arithmetic: hfb_kin.cuh).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "hfb_kin.cuh"

namespace hfb {

// One launch of k_robot: configurations [0, n_configs) of the model (joints, links, path_list in device memory).
// Poses (sample == false): q is n_configs x J.  Sampling: q_from / q_to are n_motions x J, off the n_motions + 1
// offsets in device memory.  tfs is written, handles, q_out and sweep when not null (sweep only when sampling).
struct KinArgs {
  const KinJoint* joints;
  const KinLink* links;
  const uint8_t* path_list;
  uint32_t J, L;
  size_t n_configs;
  const double* q;
  const double* q_from;
  const double* q_to;
  const uint32_t* off;
  uint32_t n_motions;
  hfb_transform* tfs;
  uint32_t* handles;
  double* q_out;
  double* sweep;
};
// returns a cudaError_t as int
int robot_launch(const KinArgs& a, bool sample, int num_sms, cudaStream_t s);

// One launch of k_robot_at (hfb_env_validate_motions): n_samples samples at dyadic positions of their motions.  Sample
// t is motion m[t] (q_from / q_to: its end points, J values per motion) at position k[t] of n_pos = 2^D + 1 (kin_sample's
// formula, so the depth-d samples are those of 2^d + 1 evenly spaced ones); its L link poses and handles go to
// tfs / handles[t * L ..].  When seg[t] is set, sweep[t * L ..] gets the links' sweep bounds over [k[t], k[t] + len];
// else 0 (a run's last sample).  sweep may be null.
struct KinAtArgs {
  const KinJoint* joints;
  const KinLink* links;
  const uint8_t* path_list;
  uint32_t J, L;
  size_t n_samples;
  const double* q_from;
  const double* q_to;
  const uint32_t* m;
  const uint32_t* k;
  const uint8_t* seg;
  uint32_t n_pos, len;
  hfb_transform* tfs;
  uint32_t* handles;
  double* sweep;
};
// returns a cudaError_t as int
int robot_at_launch(const KinAtArgs& a, int num_sms, cudaStream_t s);

}  // namespace hfb
