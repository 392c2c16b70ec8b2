// GJK for the primitive pairs of a batch in PASSES (replaces the single kernel k_pairs<1, CAP_PRIM, MODE,
// PATH_GJKROUTE> on the GJK-routed classes; same per-pair operations: pair_gjk_begin / gjk_step / pair_gjk_end of
// hfb_pair.cuh, i.e. GJK::evaluate src/narrowphase/gjk.cpp:188-370 and the extractors narrowphase.h:589-656).
//
// Why.  In the single kernel few lanes of a warp are active per instruction and the warps stall on instruction
// fetch.  A pair needs 3 to 26 iterations, so
// a warp that keeps its 32 pairs until the last one has converged idles most of its lanes; and set-up, iteration
// and witness extraction together are ~13 000 instructions against an instruction cache of 2 000 (32 KB L1.5 per
// SM), with the warps of an SM spread all over them.  Here:
//   k_gjk_first<MODE>   set-up + the first K1 iterations of every pair; the loop state of the pairs still running to
//                       HBM, and the pairs appended to a list
//   k_gjk_more<MODE>    K2, K3, ... more iterations of the pairs still running, which each pass compacts into a list
//                       (the last pass runs to convergence)
// A pair whose iterations end is finished by the kernel that ran them: status machine + witness points (pair_gjk_end),
// result record or EPA queue item.  Every kernel is small, and the later passes run full warps of the long pairs.
//
// The loop state of a running pair is stored field-major (one row per scalar field, one column per slot in the list
// of running pairs), so that the lanes of a warp, which hold consecutive slots, move consecutive words: 56 B plus 48 B
// per live simplex vertex (plus 52 B for the Polyak and Nesterov variants), where the next pass reads it densely.
//
// Inside k_gjk_first and k_gjk_more a simplex vertex is w and a slot id (SVSlot): the support points w0 / w1, which
// the iterations never read, wait in a per-thread store in shared memory (SlotStore) until the pair's loop state is
// saved, its witness points are summed (their weights come from w) or its EPA item is written.  What the iterations
// read but never write (the relative pose, the shapes' parameters, the radii) waits there as well, and is read again
// where it is needed.  That leaves registers for 4 blocks of 128 threads per SM in the first pass instead of 3.
#include "hfb_gjkpass.h"

namespace {

// k_gjk_first / k_gjk_more: block size, resident blocks per SM.  4 for the first pass of the default variant, which
// every pair goes through and which gains from the extra warps.  3 for the later passes: they run the long pairs, a
// few per SM, where the length of one iteration's dependent chain counts more than the warps that hide it, so they
// keep the pose in registers rather than read it from shared memory in every iteration.  3 for the Polyak and
// Nesterov variants as well: they carry L.w and L.dir from one iteration to the next, which does not fit the registers
// of 4 blocks without spilling in the loop.
enum { PASS_THREADS = 128, PASS_BLOCKS_PER_SM_FIRST = 4, PASS_BLOCKS_PER_SM = 3 };
constexpr int pass_blocks_per_sm(bool first, bool momentum) {
  return first && !momentum ? PASS_BLOCKS_PER_SM_FIRST : PASS_BLOCKS_PER_SM;
}

// w0 / w1 of the simplex vertices of the passes: 4 slots per thread, laid out [slot][component][thread] so that the
// lanes of a warp touch consecutive doubles (24 KB per block).  gjk_step appends a support point in the lowest slot no
// live vertex uses: at most 3 vertices are live when it appends, so one is always free.
// Next to them, what a pair reads but never writes while it iterates: the two radii (finishing reads them) and, with
// POSE, the relative pose oR1 / ot1 of its Minkowski difference, the parameters p0..p2 of both shapes (the support
// calls read them) and the early-stop bound (check B reads it), laid out [row][thread] (2 or 21 KB per block).
// Without POSE (the passes that run 3 blocks per SM) the support calls read the pose and the parameters, and check B
// the bound, from registers.
enum { RADII_ROWS = 2, POSE_ROWS = 21 };  // ssr0, ssr1; then oR1 row-major (9), ot1 (3), p0..p2 of each shape, bound
template <bool POSE>
struct SlotStore {
  using V = SVSlot;
  static constexpr bool inline_projections = true;
  static constexpr int rows = POSE ? POSE_ROWS : RADII_ROWS;
  double* col;   // this thread's column: component c of slot j at col[(6 * j + c) * PASS_THREADS]
  double* pose;  // this thread's column of the `rows` rows: row c at pose[c * PASS_THREADS]

  // L: the loop state gjk_begin or load_running set up for the pair (its upper_bound)
  __device__ __forceinline__ void set_pose(const GjkSetup& S, const GjkLoop& L) const {
    const MinkD& md = S.md;
    const double v[POSE_ROWS] = {md.ssr0,     md.ssr1,     md.oR1.r0.x, md.oR1.r0.y, md.oR1.r0.z,
                                 md.oR1.r1.x, md.oR1.r1.y, md.oR1.r1.z, md.oR1.r2.x, md.oR1.r2.y,
                                 md.oR1.r2.z, md.ot1.x,    md.ot1.y,    md.ot1.z,    S.a.p0,
                                 S.a.p1,      S.a.p2,      S.b.p0,      S.b.p1,      S.b.p2,
                                 L.upper_bound};
#pragma unroll
    for (int c = 0; c < rows; ++c) pose[c * PASS_THREADS] = v[c];
  }
  // row c (read through a volatile pointer: otherwise the compiler forwards what set_pose stored and keeps it in
  // registers across the iterations)
  __device__ __forceinline__ double pr(int c) const {
    return static_cast<const volatile double*>(pose)[c * PASS_THREADS];
  }
  __device__ __forceinline__ double ssr0() const { return pr(0); }
  __device__ __forceinline__ double ssr1() const { return pr(1); }
  __device__ __forceinline__ m3 oR1() const {
    m3 R;
    R.r0 = mk(pr(2), pr(3), pr(4));
    R.r1 = mk(pr(5), pr(6), pr(7));
    R.r2 = mk(pr(8), pr(9), pr(10));
    return R;
  }
  __device__ __forceinline__ v3 ot1() const { return mk(pr(11), pr(12), pr(13)); }
  // what gjk_begin puts in L.ssr and L.upper_bound, with POSE read from the rows rather than kept in registers (the
  // sum of the radii, which only a pair's last step reads, computed again by the same operation)
  __device__ __forceinline__ double ssr(const GjkLoop& L) const {
    if constexpr (POSE) return ssr0() + ssr1();
    else return L.ssr;
  }
  __device__ __forceinline__ double upper_bound(const GjkLoop& L, const GjkParams&) const {
    if constexpr (POSE) return pr(20);
    else return L.upper_bound;
  }
  __device__ __forceinline__ ShapeD shape_at(const ShapeD& s, int c) const {
    ShapeD r = s;
    r.p0 = pr(c);
    r.p1 = pr(c + 1);
    r.p2 = pr(c + 2);
    return r;
  }
  __device__ __forceinline__ ShapeD shape0(const ShapeD& s) const { return shape_at(s, 14); }
  __device__ __forceinline__ ShapeD shape1(const ShapeD& s) const { return shape_at(s, 17); }
  template <int G, int CAPS>
  __device__ __forceinline__ SV support(const ShapeD& a, const ShapeD& b, const MinkD& md, v3 d, int& h0,
                                        int& h1) const {
    if constexpr (POSE) return gjk_support<G, CAPS>(a, b, md, d, h0, h1, *this);
    else return gjk_support<G, CAPS>(a, b, md, d, h0, h1);
  }

  __device__ __forceinline__ void st(int j, v3 w0, v3 w1) const {
    double* p = col + 6 * j * PASS_THREADS;
    p[0] = w0.x;
    p[PASS_THREADS] = w0.y;
    p[2 * PASS_THREADS] = w0.z;
    p[3 * PASS_THREADS] = w1.x;
    p[4 * PASS_THREADS] = w1.y;
    p[5 * PASS_THREADS] = w1.z;
  }
  __device__ __forceinline__ void ld(int j, v3& w0, v3& w1) const {
    const double* p = col + 6 * j * PASS_THREADS;
    w0 = mk(p[0], p[PASS_THREADS], p[2 * PASS_THREADS]);
    w1 = mk(p[3 * PASS_THREADS], p[4 * PASS_THREADS], p[5 * PASS_THREADS]);
  }
  __device__ __forceinline__ v3 append(GjkStateT<SVSlot>& g, const SV& nv) const {
    unsigned used = 0;
    if (g.rank > 0) used |= 1u << g.s0.slot;
    if (g.rank > 1) used |= 1u << g.s1.slot;
    if (g.rank > 2) used |= 1u << g.s2.slot;
    SVSlot v;
    v.w = nv.w;
    v.slot = __ffs(~used) - 1;
    st(v.slot, nv.w0, nv.w1);
    put(g, g.rank, v);
    return nv.w;
  }
  __device__ __forceinline__ void support_points(const SVSlot& v, v3& w0, v3& w1) const { ld(v.slot, w0, w1); }
};

// rows of the loop state of a running pair (by slot in the running list).  A pair that goes on into the next pass
// has at most 3 live vertices: a rank-4 simplex either encloses the origin, which ends GJK, or is projected onto
// one of its faces, edges or vertices.
enum { RUN_SLOTS = 3 };
enum { RD_RAY = 0, RD_ALPHA = 3, RD_RL = 4, RD_W = 5, RD_LW = RD_W + RUN_SLOTS * 6, RD_DIR = RD_LW + 3, RD_ROWS = RD_DIR + 3 };
enum { RI_RANK = 0, RI_ITER, RI_HINT0, RI_HINT1, RI_VARIANT, RI_ROWS };

struct Rows {  // entry `at` of row r: d[r * stride + at] / i[r * stride + at]
  double* d;
  int* i;
};
struct PassState {
  Rows run[2];    // running pairs, two buffers, ping-ponged like the lists
  size_t stride;  // positions of the range (rows of every buffer have this length)
};

struct PassArgs {
  PassState st;
  const uint32_t* in_list;   // positions still running (null: the whole range)
  const unsigned* in_count;
  uint32_t* out_list;        // positions still running after this pass (null: last pass)
  unsigned* out_count;
  Rows rin, rout;            // loop state of the pairs of in_list / out_list (entries of st.run)
  int steps;
};

__device__ __forceinline__ void st3r(double* d, size_t stride, int row, unsigned at, v3 v) {
  d[row * stride + at] = v.x;
  d[(row + 1) * stride + at] = v.y;
  d[(row + 2) * stride + at] = v.z;
}
__device__ __forceinline__ v3 ld3r(const double* d, size_t stride, int row, unsigned at) {
  return mk(d[row * stride + at], d[(row + 1) * stride + at], d[(row + 2) * stride + at]);
}

// the loop state of a pair that goes on into the next pass.  L.w and L.dir are only carried from one iteration to
// the next by the Polyak and Nesterov variants (gjk_step overwrites both before it reads them otherwise).
template <class Store>
__device__ __forceinline__ void save_running(const Rows& r, size_t m, unsigned q, const GjkStateT<SVSlot>& g,
                                             const GjkLoop& L, bool momentum, const Store& ss) {
  r.i[RI_RANK * m + q] = g.rank;
  r.i[RI_ITER * m + q] = (int)g.iterations;
  r.i[RI_HINT0 * m + q] = g.hint0;
  r.i[RI_HINT1 * m + q] = g.hint1;
  st3r(r.d, m, RD_RAY, q, g.ray);
  r.d[RD_ALPHA * m + q] = L.alpha;
  r.d[RD_RL * m + q] = L.rl;
#pragma unroll
  for (int j = 0; j < RUN_SLOTS; ++j) {
    if (j < g.rank) {
      v3 w0, w1;
      ss.ld(pick(g, j).slot, w0, w1);
      st3r(r.d, m, RD_W + 6 * j, q, w0);
      st3r(r.d, m, RD_W + 6 * j + 3, q, w1);
    }
  }
  if (momentum) {
    r.i[RI_VARIANT * m + q] = L.variant;
    st3r(r.d, m, RD_LW, q, L.w);
    st3r(r.d, m, RD_DIR, q, L.dir);
  }
}
// the inverse of save_running; status and distance are those of gjk_begin (a running pair has no result yet), ssr
// and upper_bound are recomputed as gjk_begin computes them.  Vertex j's support points go to store slot j; the
// vertices at and above `rank` are left unset (the next support point is written there before anything reads them).
template <bool MOM, class Store>
__device__ __forceinline__ void load_running(const Rows& r, size_t m, unsigned q, const MinkD& md, const GjkParams& P,
                                             GjkStateT<SVSlot>& g, GjkLoop& L, const Store& ss) {
  g.status = HFB_GJK_NO_COLLISION;
  g.distance = 0.0;
  g.rank = r.i[RI_RANK * m + q];
  g.iterations = (unsigned)r.i[RI_ITER * m + q];
  g.hint0 = r.i[RI_HINT0 * m + q];
  g.hint1 = r.i[RI_HINT1 * m + q];
  g.ray = ld3r(r.d, m, RD_RAY, q);
  L.alpha = r.d[RD_ALPHA * m + q];
  L.rl = r.d[RD_RL * m + q];
  L.ssr = md.ssr0 + md.ssr1;
  L.upper_bound = P.distance_upper_bound + L.ssr;
#pragma unroll
  for (int j = 0; j < RUN_SLOTS; ++j) {
    if (j < g.rank) {
      const v3 w0 = ld3r(r.d, m, RD_W + 6 * j, q);
      const v3 w1 = ld3r(r.d, m, RD_W + 6 * j + 3, q);
      ss.st(j, w0, w1);
      SVSlot v;
      v.w = w0 - w1;
      v.slot = j;
      put(g, j, v);
    }
  }
  if (MOM) {
    L.variant = r.i[RI_VARIANT * m + q];
    L.w = ld3r(r.d, m, RD_LW, q);
    L.dir = ld3r(r.d, m, RD_DIR, q);
  } else {
    L.variant = HFB_GJK_DEFAULT;
    L.w = L.dir = g.ray;
  }
}

// what load_pair_in and pair_gjk_begin leave in `o` for the extractors, read again when they run rather than kept
// in registers across the iterations
__device__ __forceinline__ PairOut begin_out(const BatchArgs& a, unsigned i) {
  PairOut o;
  o.cached_guess = mk(1, 0, 0);
  o.hint0 = o.hint1 = 0;
  o.iterations = 0;
  if (a.P.initial_guess == HFB_GUESS_CACHED) {
    if (a.guess_in) o.cached_guess = mk(a.guess_in[3 * i], a.guess_in[3 * i + 1], a.guess_in[3 * i + 2]);
    if (a.hint_in) {
      o.hint0 = a.hint_in[2 * i];
      o.hint1 = a.hint_in[2 * i + 1];
    }
  }
  return o;
}

// pair_gjk_end of a pair whose iterations ended: its EPA queue item, or its result record.  Of what make_setup<CAP_PRIM>
// builds, the extractors read the first pose, `swapped` (false) and the two radii.  The radii are kept from the set-up
// in the store (reading them again costs two dependent loads, handle then shape record, on the pair's last step); the
// first pose, which the iterations do not need, is read again here.
template <int MODE, class Store>
__device__ __forceinline__ void finish_pair(const BatchArgs& a, unsigned i, GjkStateT<SVSlot>& g, const Store& ss) {
  if (g.status == HFB_GJK_COLLISION && a.P.compute_penetration) {  // the EPA case of pair_gjk_end
    push_epa_item(a, i, g, ss);
    return;
  }
  GjkSetup S;
  S.tfa = load_xf(a.tf1[i].R);
  S.swapped = false;
  S.md.ssr0 = ss.ssr0();
  S.md.ssr1 = ss.ssr1();
  PairOut o = begin_out(a, i);
  pair_gjk_end<true>(a.P, S, g, o, ss);
  store_result<MODE>(a, i, o);
}

// appends `pos` to the running list if `more`; returns its slot there
__device__ __forceinline__ unsigned append_running(const PassArgs& p, bool more, unsigned pos) {
  const unsigned m = __ballot_sync(0xffffffffu, more);
  if (!m) return 0;
  const unsigned lane = threadIdx.x & 31u;
  unsigned base = 0;
  if (lane == (unsigned)(__ffs(m) - 1)) base = atomicAdd(p.out_count, (unsigned)__popc(m));
  base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
  const unsigned q = base + (unsigned)__popc(m & ((1u << lane) - 1u));
  if (more) p.out_list[q] = pos;
  return q;
}

// MOM: the batch runs the Polyak or Nesterov variant (false: the default one, L.variant never changes)
template <int MODE, bool MOM>
__global__ void __launch_bounds__(PASS_THREADS, pass_blocks_per_sm(true, MOM))
    k_gjk_first(const BatchArgs a, const PassArgs p) {
  using Store = SlotStore<!MOM>;  // the pose in shared memory where the pass runs 4 blocks per SM
  __shared__ double store_rows[4 * 6 * PASS_THREADS];
  __shared__ double pose_rows[Store::rows * PASS_THREADS];
  const Store ss{store_rows + threadIdx.x, pose_rows + threadIdx.x};
  const unsigned lo = *a.range_lo, hi = *a.range_hi;
  const unsigned stride = gridDim.x * blockDim.x;
  for (unsigned k0 = lo + blockIdx.x * blockDim.x; k0 < hi; k0 += stride) {  // (warp-uniform trip count)
    const unsigned k = k0 + threadIdx.x;
    bool more = false, fin = false;
    unsigned i = 0;
    GjkStateT<SVSlot> g;
    GjkLoop L;
    if (k < hi) {
      i = a.index_list[k];
      const PairIn in = load_pair_in<CAP_PRIM>(a, i);
      if (!type_known(in.s1.type) || !type_known(in.s2.type)) {
        PairOut o = begin_out(a, i);
        set_unsupported(o);
        store_result<MODE>(a, i, o);
      } else {
        GjkSetup S;
        PairOut o;
        pair_gjk_begin<CAP_PRIM>(in, a.P, S, L, g, o);
        ss.set_pose(S, L);
        more = true;
        for (int s = 0; s < p.steps && more; ++s) more = gjk_step<1, CAP_PRIM, Store, MOM>(S.a, S.b, S.md, a.P.gjk, g, L, ss);
        fin = !more;
      }
    }
    // the pairs that ended are finished after the others are saved: the loop state is dead by then
    if (p.out_list) {
      const unsigned q = append_running(p, more, k - lo);
      if (more) save_running(p.rout, p.st.stride, q, g, L, MOM, ss);
    }
    if (fin) finish_pair<MODE>(a, i, g, ss);
  }
}

template <int MODE, bool MOM>
__global__ void __launch_bounds__(PASS_THREADS, pass_blocks_per_sm(false, MOM))
    k_gjk_more(const BatchArgs a, const PassArgs p) {
  using Store = SlotStore<false>;
  __shared__ double store_rows[4 * 6 * PASS_THREADS];
  __shared__ double pose_rows[Store::rows * PASS_THREADS];
  const Store ss{store_rows + threadIdx.x, pose_rows + threadIdx.x};
  const unsigned lo = *a.range_lo;
  const unsigned n = *p.in_count;
  const unsigned stride = gridDim.x * blockDim.x;
  for (unsigned q0 = blockIdx.x * blockDim.x; q0 < n; q0 += stride) {
    const unsigned q = q0 + threadIdx.x;
    bool more = false;
    unsigned pos = 0, i = 0;
    GjkStateT<SVSlot> g;
    GjkLoop L;
    if (q < n) {
      pos = p.in_list[q];
      i = a.index_list[lo + pos];
      const PairIn in = load_pair_in<CAP_PRIM>(a, i);
      GjkSetup S;
      make_setup<CAP_PRIM>(in, S);
      load_running<MOM>(p.rin, p.st.stride, q, S.md, a.P.gjk, g, L, ss);
      ss.set_pose(S, L);
      more = true;
      for (int s = 0; s < p.steps && more; ++s) more = gjk_step<1, CAP_PRIM, Store, MOM>(S.a, S.b, S.md, a.P.gjk, g, L, ss);
    }
    if (p.out_list) {
      const unsigned qo = append_running(p, more, pos);
      if (more) save_running(p.rout, p.st.stride, qo, g, L, MOM, ss);
    }
    if (q < n && !more) finish_pair<MODE>(a, i, g, ss);
  }
}

// the buffers of the pass state, carved from `base` (null: only the size is wanted); returns the bytes used
size_t carve(void* base, size_t n, PassState& st) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    void* q = reinterpret_cast<void*>(reinterpret_cast<uintptr_t>(base) + off);
    off += (bytes + 255) & ~(size_t)255;
    return q;
  };
  st.stride = n;
  for (Rows& r : st.run) {
    r.d = static_cast<double*>(take(RD_ROWS * n * sizeof(double)));
    r.i = static_cast<int*>(take(RI_ROWS * n * sizeof(int)));
  }
  return off;
}

}  // namespace

size_t gjk_pass_state_bytes(size_t n) {
  PassState st;
  return carve(nullptr, n, st);
}

// one block per PASS_THREADS pairs, at most 16 waves of resident blocks (the kernels stride over the rest)
static unsigned pass_blocks(unsigned n, int num_sms, bool first, bool mom) {
  unsigned blocks = (n + PASS_THREADS - 1) / PASS_THREADS;
  const unsigned cap = (unsigned)num_sms * pass_blocks_per_sm(first, mom) * 16u;
  if (blocks > cap) blocks = cap;
  return blocks ? blocks : 1u;
}

// the first pass (the result records and EPA items of the pairs it finished are written when it ends, so that the
// caller can start EPA on a side stream next to the remaining passes)
int gjk_passes_first(const BatchArgs& a, int mode, unsigned n, void* state, uint32_t* list_a, unsigned* counts,
                     const int* steps, int npass, int num_sms, cudaStream_t s, int* launches) {
  if (npass < 1) return (int)cudaErrorInvalidValue;
  cudaError_t e = cudaMemsetAsync(counts, 0, (size_t)npass * sizeof(unsigned), s);
  if (e != cudaSuccess) return (int)e;
  const bool mom = a.P.gjk.variant != HFB_GJK_DEFAULT;
  const unsigned blocks = pass_blocks(n, num_sms, true, mom);
  PassArgs p;
  carve(state, n, p.st);
  p.in_list = nullptr;
  p.in_count = nullptr;
  p.out_list = npass > 1 ? list_a : nullptr;
  p.out_count = counts;
  p.rout = p.st.run[0];
  p.steps = npass > 1 ? steps[0] : 0x7fffffff;
  if (mode == 0) (mom ? k_gjk_first<0, true> : k_gjk_first<0, false>)<<<blocks, PASS_THREADS, 0, s>>>(a, p);
  else (mom ? k_gjk_first<1, true> : k_gjk_first<1, false>)<<<blocks, PASS_THREADS, 0, s>>>(a, p);
  *launches += 1;
  return (int)cudaGetLastError();
}

// the remaining passes
int gjk_passes_rest(const BatchArgs& a, int mode, unsigned n, void* state, uint32_t* list_a, uint32_t* list_b,
                    unsigned* counts, const int* steps, int npass, int num_sms, cudaStream_t s, int* launches) {
  if (npass < 2) return 0;
  const bool mom = a.P.gjk.variant != HFB_GJK_DEFAULT;
  const unsigned blocks = pass_blocks(n, num_sms, false, mom);
  PassArgs p;
  carve(state, n, p.st);
  for (int k = 1; k < npass; ++k) {
    const bool last = k + 1 == npass;
    // list_a goes with run[0], list_b with run[1]
    p.in_list = (k & 1) ? list_a : list_b;
    p.rin = p.st.run[(k & 1) ? 0 : 1];
    p.in_count = counts + (k - 1);
    p.out_list = last ? nullptr : ((k & 1) ? list_b : list_a);
    p.rout = p.st.run[(k & 1) ? 1 : 0];
    p.out_count = counts + k;
    p.steps = last ? 0x7fffffff : steps[k];
    // the number of running pairs is only known on the device: the grid is sized for the typical survival rate of
    // a pass and strides over whatever there is, but never fills less than one wave of resident blocks
    const unsigned wave = (unsigned)num_sms * pass_blocks_per_sm(false, mom);
    unsigned b = blocks >> (k < 3 ? k : 3);
    if (b < wave) b = wave < blocks ? wave : blocks;
    if (mode == 0) (mom ? k_gjk_more<0, true> : k_gjk_more<0, false>)<<<b, PASS_THREADS, 0, s>>>(a, p);
    else (mom ? k_gjk_more<1, true> : k_gjk_more<1, false>)<<<b, PASS_THREADS, 0, s>>>(a, p);
    ++*launches;
  }
  return (int)cudaGetLastError();
}
