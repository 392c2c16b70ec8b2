// What the batch kernels share: the launch arguments of one (sub)batch, the EPA queue items, and the
// per-pair load / store helpers.
#pragma once
#include "hfb_arena.cuh"
#include "hfb_bvh.cuh"
#include "hfb_request.cuh"

using namespace hfb;

#define CAPS_ALL (CAP_PRIM | CAP_CONVEX | CAP_TRI)
#define CAPS_ALLP (CAPS_ALL | CAP_PLANE)  // phase 1 of the hull / triangle class, which also takes their plane pairs
#define CAPS_BVH (CAPS_ALL | CAP_INLINE_PRIM)

// ---------------------------------------------------------------- EPA queue --
struct EpaItem {
  uint32_t pair;
  int32_t rank;
  int32_t hint0, hint1;
  uint32_t gjk_iterations;
  uint32_t _pad;
  double w0[12];
  double w1[12];
};

// k_epa, tier 0 -> tier 1: a run that filled the reduced-size workspace at the top of an iteration leaves its state
// here (slot = its position in the retry list) and tier 1 carries on from it in the full-size workspace instead of
// starting the pair over: the run state, the polytope, and the support points of its vertices (EpaSupArray)
struct EpaCont {
  EpaResume rs;
  EpaPolySmall ws;
  double sp[6 * EpaPolySmall::MAXV];
};

struct BatchArgs {
  ArenaView A;
  const uint32_t* h1;
  const hfb_transform* tf1;
  const uint32_t* h2;
  const hfb_transform* tf2;
  const double* guess_in;     // n x 3 or null
  const int32_t* hint_in;     // n x 2 or null
  double* guess_out;          // n x 3 or null
  int32_t* hint_out;          // n x 2 or null
  void* out;                  // hfb_distance_result* or hfb_contact*
  EpaItem* queue;
  unsigned* queue_count;      // [0] = items pushed this batch, [1] = running total
  const unsigned* epa_lo;     // k_epa: device pointers to the [lo, hi) slice of the queue this launch owns
  const unsigned* epa_hi;
  unsigned* epa_head;         // k_epa: work counter of this launch (items are handed out one by one)
  uint32_t* retry;            // queue indices of the items that outgrew the reduced-size EPA workspace
  unsigned* retry_count;
  EpaCont* cont;              // continuation records of the first cont_cap retry positions (null: every retry starts over)
  unsigned cont_cap;
  double* epa_sup;            // k_epa tier 0: the support points of the polytopes, 6 * EpaPolySmall::MAXV doubles per
  unsigned epa_sup_groups;    // resident lane group (slot blockIdx.x * GPB + group), for this many groups
  unsigned pair_base;         // added to the pair index of an EPA queue item: the host pipeline runs phase 1 chunk by chunk
                              // (pointers offset to the chunk) and EPA once, over the whole batch (base pointers)
  unsigned sub_idx, sub_cnt;  // k_pairs: this launch takes the sub_idx-th of sub_cnt equal parts of [lo, hi)
  unsigned* gjk_work;         // k_gjk_refill: work counter of this launch
  unsigned iter_quorum;       // k_gjk_refill: lanes that must be mid-GJK for an iteration round to run
  unsigned stage;             // lane-group k_pairs: TMA-stage the hulls' vertex blocks into shared memory
  const uint32_t* index_list; // optional indirection: pair ids sorted by class (k_bin_scatter)
  const unsigned* range_lo;   // device pointers to the [lo, hi) slice of index_list to process
  const unsigned* range_hi;
  SolverP P;
  CollideP C;
  BvhReq B;                   // traversal request fields (BVH pairs)
  EpaWs* bvh_ws;              // one EPA workspace per thread of k_bvh (global memory)
  unsigned long long* bvh_counters;  // [0] bv tests, [1] leaf tests (running totals)
  unsigned* bvh_work;         // k_bvh: work counter of this launch
  unsigned n;
  // hfb_batch_collide_contacts (null / 0 otherwise): contacts[1..] of mesh pairs, extra_cap records per pair, and
  // the number of contacts of every mesh pair
  hfb_contact* extra;
  uint32_t* counts;
  unsigned extra_cap;
};
__device__ __forceinline__ BvhContactSink contact_sink(const BatchArgs& a, unsigned i) {
  BvhContactSink s;
  s.extra = a.extra ? a.extra + (size_t)i * a.extra_cap : nullptr;
  s.cap = a.extra ? a.extra_cap : 0u;
  s.count = a.counts ? a.counts + i : nullptr;
  return s;
}

template <int CAPS>
__device__ __forceinline__ PairIn load_pair_in(const BatchArgs& a, unsigned i) {
  PairIn in;
  in.s1 = load_shape<CAPS>(a.A, a.h1[i]);
  in.s2 = load_shape<CAPS>(a.A, a.h2[i]);
  in.tf1 = load_xf(a.tf1[i].R);
  in.tf2 = load_xf(a.tf2[i].R);
  in.cached_guess = mk(1, 0, 0);
  in.hint0 = in.hint1 = 0;
  if (a.P.initial_guess == HFB_GUESS_CACHED) {
    if (a.guess_in) in.cached_guess = mk(a.guess_in[3 * i], a.guess_in[3 * i + 1], a.guess_in[3 * i + 2]);
    if (a.hint_in) {
      in.hint0 = a.hint_in[2 * i];
      in.hint1 = a.hint_in[2 * i + 1];
    }
  }
  return in;
}

template <int MODE>
__device__ __forceinline__ void store_result(const BatchArgs& a, unsigned i, const PairOut& o) {
  if (MODE == 0) write_distance(o, reinterpret_cast<hfb_distance_result*>(a.out) + i);
  else write_contact(o, a.C, reinterpret_cast<hfb_contact*>(a.out) + i);
  if (a.guess_out) {
    a.guess_out[3 * i] = o.cached_guess.x;
    a.guess_out[3 * i + 1] = o.cached_guess.y;
    a.guess_out[3 * i + 2] = o.cached_guess.z;
  }
  if (a.hint_out) {
    a.hint_out[2 * i] = o.hint0;
    a.hint_out[2 * i + 1] = o.hint1;
  }
}

__device__ __forceinline__ void st3(double* p, v3 v) {
  p[0] = v.x;
  p[1] = v.y;
  p[2] = v.z;
}
__device__ __forceinline__ v3 ld3(const double* p) { return mk(p[0], p[1], p[2]); }

template <class V>
__device__ __forceinline__ EpaItem* new_epa_item(const BatchArgs& a, unsigned i, const GjkStateT<V>& g) {
  const unsigned slot = atomicAdd(a.queue_count, 1u);
  atomicAdd(a.queue_count + 1, 1u);
  EpaItem* it = a.queue + slot;
  it->pair = i + a.pair_base;
  it->rank = g.rank;
  it->hint0 = g.hint0;
  it->hint1 = g.hint1;
  it->gjk_iterations = g.iterations;
  return it;
}
// the item of a simplex whose support points sit in a store of the caller's (the GJK passes' SlotStore); the
// vertices at and above `rank` are written as zeros
template <class Store>
__device__ __forceinline__ void push_epa_item(const BatchArgs& a, unsigned i, const GjkStateT<typename Store::V>& g,
                                              const Store& st) {
  EpaItem* it = new_epa_item(a, i, g);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    v3 w0 = mk(0, 0, 0), w1 = mk(0, 0, 0);
    if (j < g.rank) st.support_points(pick(g, j), w0, w1);
    st3(it->w0 + 3 * j, w0);
    st3(it->w1 + 3 * j, w1);
  }
}
__device__ __forceinline__ void push_epa_item(const BatchArgs& a, unsigned i, const GjkState& g) {
  EpaItem* it = new_epa_item(a, i, g);
  st3(it->w0 + 0, g.s0.w0);
  st3(it->w1 + 0, g.s0.w1);
  st3(it->w0 + 3, g.s1.w0);
  st3(it->w1 + 3, g.s1.w1);
  st3(it->w0 + 6, g.s2.w0);
  st3(it->w1 + 6, g.s2.w1);
  st3(it->w0 + 9, g.s3.w0);
  st3(it->w1 + 9, g.s3.w1);
}
