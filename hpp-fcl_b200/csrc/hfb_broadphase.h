// Host-side interface of the device broadphase (kernels in hfb_broadphase.cu; design: hfb_broadphase.cuh).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "../../include/hppfcl_b200.h"

namespace hfb {

// world-space boxes of n objects (6 doubles each) from the per-handle local boxes of the committed arena
int bp_scene_aabbs_launch(const double* d_local_aabbs, uint32_t nshapes, size_t n, const uint32_t* d_handles,
                          const hfb_transform* d_tfs, double* d_aabbs, cudaStream_t s);
// scratch the pair finder needs for n objects
size_t bp_scratch_bytes(size_t n);
// every pair i < j with overlapping boxes and i in [i_lo, i_hi) -> (d_first, d_second), at most `capacity` stored,
// all counted in *d_n_pairs; `scratch`: bp_scratch_bytes(n) bytes.  Returns a cudaError_t as int; *launches += kernels
// launched.
int bp_pairs_launch(size_t n, const double* d_aabbs, size_t i_lo, size_t i_hi, uint32_t* d_first, uint32_t* d_second,
                    size_t capacity, unsigned* d_n_pairs, void* scratch, int num_sms, cudaStream_t s, int* launches);
// scratch the cross pair finder needs for n_a objects in A and n_b in B
size_t bp_cross_scratch_bytes(size_t n_a, size_t n_b);
// every (i, j), i in A with i in [a_lo, a_hi), j in B, with overlapping boxes -> (i, second_base + j), at most
// `capacity` stored, all counted in *d_n_pairs (grid over B only: hfb_broadphase.cuh, broadphase_cross_pairs_host);
// `scratch`: bp_cross_scratch_bytes(n_a, n_b) bytes.  Returns a cudaError_t as int; *launches += kernels launched.
int bp_cross_pairs_launch(size_t n_a, const double* d_aabbs_a, size_t a_lo, size_t a_hi, size_t n_b, const double* d_aabbs_b,
                          uint32_t* d_first, uint32_t* d_second, uint32_t second_base, size_t capacity, unsigned* d_n_pairs,
                          void* scratch, int num_sms, cudaStream_t s, int* launches);

// bp_cross_pairs_launch in its two halves, for a grid over B that outlives the call (hfb_env): the grid's persistent
// part -- cell size and dims, B's oversize count, `order`, `start` -- lives in bp_cross_grid_bytes(n_b) bytes of the
// caller's; the build-only buffers and A's brute list come from `scratch` (bp_cross_scratch_bytes(n_a, n_b) bytes).
struct BpCrossGrid {
  void* grid;          // cell size and dims (256 bytes)
  unsigned* counters;  // [0]: B's oversize + unbounded objects; [2], [3]: a query's (bp_cross_query_reset)
  unsigned* order;     // n_b
  unsigned* start;     // cells + 1
};
size_t bp_cross_grid_bytes(size_t n_b);
BpCrossGrid bp_cross_grid_carve(void* p, size_t n_b);
// the grid over B's boxes; run again after B's boxes change
int bp_cross_build_launch(size_t n_b, const double* d_aabbs_b, const BpCrossGrid& g, void* scratch, cudaStream_t s,
                          int* launches);
// clears *d_n_pairs and A's brute list (not B's oversize count) in front of a query against a built grid
int bp_cross_query_reset(const BpCrossGrid& g, unsigned* d_n_pairs, cudaStream_t s);
// the query: k_cross_sweep and k_cross_brute as in bp_cross_pairs_launch, B's oversize list by k_cross_oversize
int bp_cross_query_launch(size_t n_a, const double* d_aabbs_a, size_t a_lo, size_t a_hi, size_t n_b, const double* d_aabbs_b,
                          const BpCrossGrid& g, uint32_t* d_first, uint32_t* d_second, uint32_t second_base, size_t capacity,
                          unsigned* d_n_pairs, void* scratch, int num_sms, cudaStream_t s, int* launches);
// the self pairs of configurations [g0, g0 + num_configs) of L = `links` objects each (config_pair of
// hfb_broadphase.cuh; d_tpl: n_tpl pairs of link indices, validated) -> (d_first, d_second), APPENDED after the pairs
// *d_n_pairs already counts; at most `capacity` stored in all.  Returns a cudaError_t as int; *launches += kernels
// launched.  d_entry (may be null): each pair's template entry, stored at its position in the list.
int bp_config_pairs_launch(const double* d_aabbs, size_t links, const uint32_t* d_tpl, size_t n_tpl, size_t g0,
                           size_t num_configs, uint32_t* d_first, uint32_t* d_second, size_t capacity, unsigned* d_n_pairs,
                           int num_sms, cudaStream_t s, int* launches, uint32_t* d_entry = nullptr);
// ---- hfb_env_distance: each A object's nearest B object, found in rounds of growing radius (DESIGN.md §3) ----------
// Round k runs distance() on the pairs whose B box overlaps the A box inflated by rho_k = min(cell * 8^k, max_distance)
// (outward rounding) and did not overlap the round before's; an A object is settled once its best eligible distance is
// <= rho_k, rho_k == max_distance, or its inflated box overlaps every box of B.  A pair a round skips has a box gap,
// and so a distance, above rho_k.  Per-A state (n_a each, bp_dist_state_bytes(n_a) bytes of the caller's):
struct BpDistState {
  unsigned long long* key;   // order-preserving key of the best eligible distance so far; ~0: none
  unsigned long long* prev;  // key at the start of the round
  int32_t* nearest;          // index in B of the best pair; -1: none
  uint32_t* jround;          // the lowest index in B among this round's pairs at `key`
  uint8_t* state;            // 0: settled or outside the range, 1: open, 2: open for round 0 against all of B
  hfb_distance_result* rec;  // the record of `nearest` (a fresh DistanceResult while there is none)
  const unsigned long long* reach;  // B's reach (bp_dist_reach_launch), kept with the env's grid
};
size_t bp_dist_state_bytes(size_t n_a);
BpDistState bp_dist_state_carve(void* p, size_t n_a, const unsigned long long* reach);
// B's reach from B's boxes, 6 keys: per axis the smallest box maximum and the largest box minimum (an A box widened
// past both overlaps every box of B); run again after B's boxes change
int bp_dist_reach_launch(size_t n_b, const double* d_bb, unsigned long long* d_reach, int num_sms, cudaStream_t s,
                         int* launches);
// state of all n_a objects from A's boxes d_ba, [a_lo, a_hi) open (a_lo <= a_hi <= n_a)
int bp_dist_init_launch(size_t n_a, const double* d_ba, size_t a_lo, size_t a_hi, const BpDistState& st, cudaStream_t s,
                        int* launches);
// round `round`'s start: objects settled by the round before, then the query boxes d_bq of the open ones (the empty
// box for the others); *d_n_open = the number of open ones
int bp_dist_boxes_launch(const double* d_ba, size_t a_lo, size_t a_hi, const BpCrossGrid& g, double max_distance, int round,
                         const BpDistState& st, double* d_bq, unsigned* d_n_open, cudaStream_t s, int* launches);
// the first min(*d_n_raw, capacity) candidates (d_first, d_second = second_base + index in B) less the pairs the round
// before already ran -> (d_kept_first, d_kept_second), counted in *d_n_kept
int bp_dist_filter_launch(const uint32_t* d_first, const uint32_t* d_second, const unsigned* d_n_raw, size_t capacity,
                          const double* d_ba, const double* d_bb, uint32_t second_base, const BpCrossGrid& g,
                          double max_distance, int round, uint32_t* d_kept_first, uint32_t* d_kept_second,
                          unsigned* d_n_kept, int num_sms, cudaStream_t s, int* launches);
// the round's n distance() records into the per-A best (smallest eligible distance, then lowest index in B); the
// candidates that came back HFB_PATH_UNSUPPORTED are added to *d_n_unsupported
int bp_dist_reduce_launch(const hfb_distance_result* d_recs, const uint32_t* d_first, const uint32_t* d_second, size_t n,
                          uint32_t second_base, double max_distance, const BpDistState& st, unsigned* d_n_unsupported,
                          cudaStream_t s, int* launches);
// ---- hfb_env_distance_configs: each configuration's nearest pair, environment or self (DESIGN.md §3) ---------------
// After the rounds above over the range's links, the self pairs config_dist_pair runs go through distance(); the best
// per configuration is then taken over the links' winners (ordinal: link index i) and the self records (ordinal L + k,
// k the template entry), smallest key first, then lowest ordinal.  Per-configuration state, n_configs each
// (bp_config_dist_bytes(n_configs) bytes of the caller's):
struct BpConfigDist {
  unsigned long long* key;  // order-preserving key of the best eligible distance; ~0: none
  unsigned long long* ord;  // the lowest ordinal at `key`
  uint32_t* first;          // the winner's index in A; UINT32_MAX: none
  uint32_t* second;         // its index in B (kind 0) or in A (kind 1); UINT32_MAX: none
  int8_t* kind;             // 0: environment pair, 1: self pair, -1: none
  hfb_distance_result* rec; // the winner's record (a fresh DistanceResult while there is none)
};
size_t bp_config_dist_bytes(size_t n_configs);
BpConfigDist bp_config_dist_carve(void* p, size_t n_configs);
// every configuration without a winner
int bp_config_dist_init_launch(size_t n_configs, const BpConfigDist& cs, cudaStream_t s, int* launches);
// the self pairs of configurations [g0, g0 + num_configs) that config_dist_pair runs -> (d_first, d_second, d_entry: the
// template entry), at most `capacity` stored, all counted in *d_n_pairs (cleared first)
int bp_config_dist_pairs_launch(const double* d_aabbs, size_t links, const uint32_t* d_tpl, size_t n_tpl, size_t g0,
                                size_t num_configs, double max_distance, uint32_t* d_first, uint32_t* d_second,
                                uint32_t* d_entry, size_t capacity, unsigned* d_n_pairs, int num_sms, cudaStream_t s,
                                int* launches);
// the winners of the configurations that links [a_lo, a_hi) make up (whole configurations), from the links' state st
// and the n_self records of their self pairs (d_first, d_second, d_entry as bp_config_dist_pairs_launch stored them);
// the self records that came back HFB_PATH_UNSUPPORTED are added to *d_n_unsupported
int bp_config_dist_reduce_launch(const BpDistState& st, size_t a_lo, size_t a_hi, size_t links,
                                 const hfb_distance_result* d_recs, const uint32_t* d_first, const uint32_t* d_second,
                                 const uint32_t* d_entry, size_t n_self, double max_distance, const BpConfigDist& cs,
                                 unsigned* d_n_unsupported, cudaStream_t s, int* launches);
// ---- hfb_env_collide_motions: each motion's first colliding sample and its first colliding pair (DESIGN.md §3) ----
// Over the collide() records of hfb_env_collide_configs' candidate list (environment pairs before `split`, self pairs
// from there on), three passes touch the colliding ones: the smallest sample per motion, then the lowest pair ordinal
// at that sample (environment: link * n_b + index in B; self: L * n_b + template entry), then the gather of the
// winner.  Per-motion state, n_motions each (bp_motions_bytes(n_motions) bytes of the caller's; `staged` adds room for
// the outputs, which the host form downloads from there):
struct BpMotions {
  const uint32_t* off;          // the motion offsets, n_motions + 1 (device copy)
  unsigned m0, m1;              // the motions checked
  unsigned* sample;             // the smallest colliding sample; UINT32_MAX: none
  unsigned long long* ord;      // the lowest ordinal among the colliding pairs at `sample`
  int32_t* first_invalid;       // outputs, each may be null
  int8_t* kind;
  uint32_t* first;
  uint32_t* second;
  hfb_contact* rec;
};
size_t bp_motions_bytes(size_t n_motions, bool staged);
BpMotions bp_motions_carve(void* p, size_t n_motions, bool staged);
// every motion without a witness: the state (when ms.sample is set) and the outputs that are set
int bp_motions_init_launch(size_t n_motions, const BpMotions& ms, cudaStream_t s, int* launches);
// the n records d_recs of the candidates (d_first, d_second, d_entry: the self pairs' template entries) into the
// per-motion state and, when `witness`, the outputs kind, first, second and rec (second_base taken off the environment
// pairs' second index); the colliding candidates before / from `split` on are added to d_n_colliding[0] / [1]
int bp_motions_reduce_launch(const hfb_contact* d_recs, const uint32_t* d_first, const uint32_t* d_second,
                             const uint32_t* d_entry, size_t n, size_t split, size_t links, size_t n_b,
                             uint32_t second_base, bool witness, const BpMotions& ms, unsigned* d_n_colliding,
                             cudaStream_t s, int* launches);
// first_invalid of the motions checked from the state (-1: none)
int bp_motions_final_launch(const BpMotions& ms, cudaStream_t s, int* launches);
// ---- hfb_env_certify_motions: motions certified between their samples from lower bounds and sweeps (DESIGN.md §3) --
// The sides of each A object (sweep_sides of hfb_broadphase.cuh) widen its box for the environment candidates and its
// self pairs' boxes for the self candidates; the collide() records of the candidates then clear per-sample pass flags
// (a pair passes a side when it has no contact, is supported and 2 * distance_lower_bound exceeds the side's
// threshold), and the unwidened overlaps among them give the first colliding sample as hfb_env_collide_motions does.
struct BpCertify {
  const uint32_t* off;  // the motion offsets, n_motions + 1 (device copy)
  unsigned m0, m1;      // the motions checked
  unsigned links, g0, ng;  // their configurations: [g0, g0 + ng)
  double* sides;        // 2 per A object: right side, left side (NaN: none)
  uint8_t* pass;        // 2 per configuration of the range (index g - g0): every pair passes the right / left side
  unsigned* sample;     // per motion: the smallest colliding sample, UINT32_MAX: none
  unsigned* unc;        // per motion: the smallest uncertified segment, UINT32_MAX: none
  int32_t* first_invalid;      // outputs, n_motions each (may be null)
  int32_t* first_uncertified;
  uint8_t* certified;   // per configuration of the range, index g - g0 (may be null)
};
// bytes of the per-motion state (sample, unc, and with `staged` the two per-motion outputs) and its carving
size_t bp_certify_bytes(size_t n_motions, bool staged);
BpCertify bp_certify_carve(void* p, size_t n_motions, bool staged);
// the sides of A objects [a_lo, a_hi) (c.sides) from the caller's sweep bounds d_sweep, and their boxes d_bb widened
// by their reach, rounded outward, into d_wbb (boxes without a box are copied)
int bp_sweep_sides_launch(const double* d_bb, const double* d_sweep, size_t a_lo, size_t a_hi, const BpCertify& c,
                          double* d_wbb, cudaStream_t s, int* launches);
// the self candidates of the range's configurations (sweep_pair), APPENDED as bp_config_pairs_launch appends
int bp_sweep_pairs_launch(const double* d_bb, const BpCertify& c, const uint32_t* d_tpl, size_t n_tpl, uint32_t* d_first,
                          uint32_t* d_second, size_t capacity, unsigned* d_n_pairs, int num_sms, cudaStream_t s,
                          int* launches);
// the certification of the range from the n records d_recs of the candidates (environment pairs (i, second_base + j)
// before `split`, self pairs from there on; n = 0: no records, every pair passes), d_ba / d_bb_b the unwidened boxes
// of A and B: the per-sample flags and the per-motion state, then the outputs of c (first_invalid, first_uncertified:
// motions [m0, m1) only; certified).  d_counts[0] += the records HFB_PATH_UNSUPPORTED, d_counts[1] += the range's
// segments not certified.
int bp_certify_launch(const hfb_contact* d_recs, const uint32_t* d_first, const uint32_t* d_second, size_t n, size_t split,
                      uint32_t second_base, const double* d_ba, const double* d_bb_b, const BpCertify& c,
                      unsigned* d_counts, cudaStream_t s, int* launches);
// hfb_env_update: d_tfs[d_idx[k]] = d_tfs_new[k] and the box of object d_idx[k] recomputed, k < m
int bp_env_update_launch(const double* d_local_aabbs, uint32_t nshapes, size_t m, const uint32_t* d_idx,
                         const hfb_transform* d_tfs_new, const uint32_t* d_handles, hfb_transform* d_tfs, double* d_aabbs,
                         cudaStream_t s);

}  // namespace hfb
