// The round bookkeeping of hfb_env_validate_motions (include/hppfcl_b200.h states the rules), as HFB_HD functions that the
// kernels (hfb_scene.cu, k_val_*) use and a host build can check.
//
// Positions: a sample of a motion sits at an integer position k in [0, 2^D]; a segment [a, a + len] of depth d has
// len = 2^(D - d).  Every open segment of a round has the round's depth, so one len serves the round.  Positions and
// counts fit in 32 bits: D <= 30, and a round's sample count is capped at 2^29, so a round's list (at most twice the
// samples of the round before) holds fewer than 2^30 segments and the inclusive scan of their costs stays below 2^31.
#pragma once
#include <stdint.h>

#include "hfb_math.cuh"

namespace hfb {

constexpr uint32_t kValNone = 0xffffffffu;  // no colliding sample, no stuck segment, no uncertified segment

enum ValRule : uint8_t { VAL_CERTIFIED = 0, VAL_DROPPED = 1, VAL_STUCK = 2, VAL_SPLIT = 3 };

// Runs.  In the round's list of open segments, sorted by (motion, start), segment i (motion m, start a) starts a new
// run unless the segment before it belongs to the same motion and ends at a.
HFB_HD bool val_new_run(bool first_in_list, uint32_t prev_m, uint32_t prev_a, uint32_t m, uint32_t a, uint32_t len) {
  return first_in_list || prev_m != m || prev_a + len != a;
}
// A segment adds one sample (its end) to the round, two when it starts a run.
HFB_HD uint32_t val_cost(bool new_run) { return new_run ? 2u : 1u; }
// Admission: the segments whose inclusive prefix sum of val_cost stays within the cap.  The costs are positive, so the
// admitted segments are a prefix of the list.  Segment i's start and end samples are the round's samples scan - 2 and
// scan - 1 (a segment that continues a run shares its start with the end of the segment before it).
HFB_HD bool val_admitted(uint32_t cost_scan, uint32_t cap) { return cost_scan <= cap; }
HFB_HD uint32_t val_start_sample(uint32_t cost_scan) { return cost_scan - 2u; }

// The segment rules, the first that applies: certified -> closed; starting at or after the motion's earliest colliding
// sample c -> dropped; not admitted, at the deepest depth or with a non-finite sweep for some link -> stuck; else split.
HFB_HD ValRule val_rule(bool admitted, bool certified, uint32_t a, uint32_t c, bool deepest, bool finite_sweep) {
  if (admitted && certified) return VAL_CERTIFIED;
  if (a >= c) return VAL_DROPPED;
  if (!admitted || deepest || !finite_sweep) return VAL_STUCK;
  return VAL_SPLIT;
}
// The frontier: after the rules, a half of a split segment stays open when it starts before f, the start of the
// motion's earliest stuck segment (kValNone: none).
HFB_HD bool val_keep(uint32_t start, uint32_t f) { return start < f; }

// Round 0 without its list: each motion of the range is one run of `per` = 2^d0 segments (per + 1 samples), so the
// admitted prefix is n_full whole motions and the first `partial` segments of the next one.  adm: motion w's admitted
// segments; its first segment that is not admitted is stuck.
HFB_HD void val_round0(uint64_t n_range, uint32_t per, uint32_t cap, uint64_t* n_full, uint32_t* partial) {
  const uint64_t whole = (uint64_t)cap / ((uint64_t)per + 1u);
  *n_full = whole < n_range ? whole : n_range;
  const uint64_t rem = (uint64_t)cap - *n_full * ((uint64_t)per + 1u);
  *partial = (*n_full < n_range && rem >= 2) ? (uint32_t)(rem - 1) : 0u;  // (rem <= per: partial < per)
}
HFB_HD uint32_t val_round0_admitted(uint64_t w, uint64_t n_full, uint32_t partial, uint32_t per) {
  return w < n_full ? per : w == n_full ? partial : 0u;
}

// A motion's outputs from its earliest colliding sample c and the start u of its earliest segment closed without a
// certificate (stuck or dropped), kValNone for none: status 1 (collides) when c exists, else 0 (valid) when every
// segment is certified, else 2 (unresolved); t_valid = u * 2^-D (1 without u); t_collide = c * 2^-D, -1 without c.
HFB_HD void val_result(uint32_t c, uint32_t u, uint32_t D, int8_t* status, double* t_valid, double* t_collide) {
  const double scale = 1.0 / (double)(1u << D);  // exact: a power of two
  *status = c != kValNone ? (int8_t)1 : u == kValNone ? (int8_t)0 : (int8_t)2;
  *t_valid = u == kValNone ? 1.0 : (double)u * scale;
  *t_collide = c == kValNone ? -1.0 : (double)c * scale;
}

}  // namespace hfb
