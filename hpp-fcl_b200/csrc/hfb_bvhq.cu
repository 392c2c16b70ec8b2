// k_bvhq_prep / k_bvhq: mesh-shape distance queries as a per-block task system (design: hfb_bvhq.cuh).
//
// One persistent block of 8 warps per SM.  Shared memory holds the block's HFB_Q_NSLOTS queries in flight
// (QSlot: poses, the shape's RSS, result so far, counters), two item queues (rings of 32-bit items) and a
// free mask of the treelet buffers; the traversal stacks and the treelet value caches live in global memory
// (L1/L2-resident, written and read by the same SM).  The block alternates between two phases: in the
// bounding-volume phase every warp takes BV items until their queue is empty, then -- after a block barrier -- every
// warp takes leaf items; the lane that completes a query's last outstanding item continues that query's walk
// (q_advance), which pushes the next item(s) or retires the query and starts another.
// Why phases and not "any warp takes any item" (the first version): the kernel is ~18 000
// instructions, the SM's instruction cache holds 2 000 (L1.5: 32 KB) -- with its eight warps in eight different
// places of that code the warps stall on instruction fetch.  In a phase the eight warps run the same two thousand
// instructions at the same time.
#include <cfloat>
#include <type_traits>

#include "hfb_bvhq_launch.h"

namespace hfb {

#define CAPS_BVHQ (CAP_PRIM | CAP_CONVEX | CAP_TRI | CAP_INLINE_PRIM)

struct QSched {
  int lhead, ltail, bhead, btail, ehead, etail;
  int active;          // queries in flight in this block
  unsigned tl_free;    // free treelet buffers
  int abort_;
  int lsnap;           // leaf phase: items queued before this ring position belong to the phase
  int do_epa, stop;    // decisions of the cycle, taken by thread 0 between two barriers
  int bn0;             // BV items of the generation that is starting
  unsigned leafq[HFB_Q_QCAP];
  unsigned bvq[HFB_Q_QCAP];
  unsigned epaq[HFB_Q_QCAP];
};

__device__ __forceinline__ int vload(const int* p) { return *reinterpret_cast<const volatile int*>(p); }

struct DevSink {
  QSched* sc;
  // the lanes of the warp that push to this ring at the same instruction share one bump of its tail (the tail is one
  // shared-memory word all eight warps hammer: a bump per lane serialised them)
  __device__ __forceinline__ void push(unsigned* buf, int* tail, unsigned item) {
    __threadfence_block();  // the slot / stack / treelet writes of this item's producer come first
    const unsigned act = __activemask();
    const unsigned lane = threadIdx.x & 31u;
    const int leader = __ffs(act) - 1;
    int base = 0;
    if ((int)lane == leader) base = atomicAdd(tail, __popc(act));
    base = __shfl_sync(act, base, leader);
    const int pos = (base + __popc(act & ((1u << lane) - 1u))) & (HFB_Q_QCAP - 1);
    volatile unsigned* q = buf;
    // the ring is larger than the number of items that can exist: the previous occupant was taken long ago
    for (unsigned spins = 0; q[pos] != 0u; ++spins)
      if (spins > (1u << 26)) {  // cannot happen; never hang the GPU over it
        atomicExch(&sc->abort_, 1);
        break;
      }
    q[pos] = item | HFB_Q_ITEM_VALID;
  }
  // `count` speculated BV items of one slot (pairs 0, 2, 4, ... of its subtree): one bump, then plain stores
  __device__ __forceinline__ void push_bv_pairs(unsigned slot_id, int count) {
    __threadfence_block();
    const int base = atomicAdd(&sc->btail, count);
    volatile unsigned* q = sc->bvq;
    for (int p = 0; p < count; ++p) {
      const int pos = (base + p) & (HFB_Q_QCAP - 1);
      for (unsigned spins = 0; q[pos] != 0u; ++spins)
        if (spins > (1u << 26)) {
          atomicExch(&sc->abort_, 1);
          break;
        }
      q[pos] = slot_id | ((unsigned)(2 * p) << 12) | HFB_Q_ITEM_SPEC | HFB_Q_ITEM_VALID;
    }
  }
  __device__ __forceinline__ void push_leaf(unsigned it) { push(sc->leafq, &sc->ltail, it); }
  __device__ __forceinline__ void push_bv(unsigned it) { push(sc->bvq, &sc->btail, it); }
  __device__ __forceinline__ void push_epa(unsigned it) { push(sc->epaq, &sc->etail, it); }
  __device__ __forceinline__ int treelet_acquire() {
    unsigned m = *reinterpret_cast<volatile unsigned*>(&sc->tl_free);
    while (m) {
      const int b = __ffs(m) - 1;
      const unsigned old = atomicAnd(&sc->tl_free, ~(1u << b));
      if (old & (1u << b)) return b;
      m = old & ~(1u << b);
    }
    return -1;
  }
  __device__ __forceinline__ void treelet_release(int id) { atomicOr(&sc->tl_free, 1u << id); }
  __device__ __forceinline__ int dec_pending(QSlot& s) {
    __threadfence_block();
    const int old = atomicSub(&s.pending, 1);
    __threadfence_block();
    return old;
  }
};

// waits for the producer of a reserved ring entry (it stores right after reserving)
__device__ __forceinline__ unsigned q_take(volatile unsigned* q, int pos, QSched* sc) {
  unsigned item;
  for (unsigned spins = 0; ((item = q[pos]) & HFB_Q_ITEM_VALID) == 0u; ++spins)
    if (spins > (1u << 26)) {  // cannot happen; never hang the GPU over it
      atomicExch(&sc->abort_, 1);
      break;
    }
  return item;
}

// next query of the slice into slot `sl` (+ its seed leaf item); false when the slice is exhausted
__device__ __noinline__ bool q_fetch(const BvhqLaunch& L, unsigned lo, unsigned hi, QSlot& s, QStackEnt* stk, unsigned sl,
                        DevSink& sink) {
  for (;;) {
    const unsigned k = atomicAdd(L.work, 1u);
    if (k >= hi - lo) return false;
    const QPrep& pr = L.prep[k];
    if (!pr.ok) continue;  // unsupported pair: k_bvhq_prep wrote its record
    const unsigned i = L.index_list[lo + k];
    const xf t1 = load_xf(L.tf1[i].R), t2 = load_xf(L.tf2[i].R);
    v3 guess = mk(1, 0, 0);
    int h0 = 0, h1 = 0;
    if (L.P.initial_guess == HFB_GUESS_CACHED) {
      if (L.guess_in) guess = mk(L.guess_in[3 * i], L.guess_in[3 * i + 1], L.guess_in[3 * i + 2]);
      if (L.hint_in) {
        h0 = L.hint_in[2 * i];
        h1 = L.hint_in[2 * i + 1];
      }
    }
    BvhQuery q;
    bool swapped;
    bvh_make_query<CAPS_BVHQ>(L.A, L.h1[i], t1, L.h2[i], t2, q, swapped);
    q_start(s, stk, q, pr, i, guess, h0, h1);
    sink.push_leaf(sl);
    return true;
  }
}

// the walk of slot `sl` continues on this lane; a finished query is written out and the slot refilled.  One copy of
// this code for every call site (instruction-cache footprint).
struct QBlock {
  QSlot* slots;
  QStackEnt* stacks;
  QTreelet* tls;
  QTreeletHot* hot;
  QSched* sc;
  unsigned lo, hi;
};
__device__ __noinline__ void q_continue(const BvhqLaunch& L, const QBlock& B, const QCtx& c, unsigned sl,
                                        unsigned long long& bv_total, unsigned long long& leaf_total, bool have,
                                        QStackEnt near) {
  DevSink sink{B.sc};
  QSlot& s = B.slots[sl];
  QStackEnt* stk = B.stacks + (size_t)sl * L.stack_cap;
  if (q_advance(s, sl, stk, B.tls, B.hot, c, sink, have, near) != Q_DONE) return;
  q_write_result(s, L.out + s.pair);
  bv_total += (unsigned)s.bv_tests;
  leaf_total += (unsigned)s.leaf_tests;
  if (!q_fetch(L, B.lo, B.hi, s, stk, sl, sink)) atomicSub(&B.sc->active, 1);
}

// The RSS distances of the two children `pair[0]`, `pair[1]` of a node by a group of G = 2 * LC lanes of the warp
// (lanes gbase .. gbase + G - 1): the first LC lanes take child 0, the others child 1; lane u of a child evaluates
// the edge-pair cases u, LC + u, 2 LC + u, ... of rectDistance in turn until one of the child's lanes has a passing
// case; the lowest passing case index is the reference's first return (RSS.cpp:121-713), its lane computes the
// distance.  LC = 1 (16 items per warp, no divergence between the lanes of a case) when the queue is long, LC = 4
// (4 items per warp, a quarter of the dependent chain) when it is not.
template <int LC>
__device__ __forceinline__ void q_bv_group(bool active, const QSlot& s, const hfb_bvh_node* pair, unsigned gbase,
                                           unsigned sub, double& d1, double& d2, int& f1, int& f2) {
  // every lane of the warp comes here (votes and shuffles are warp-wide: a vote over part of a warp is executed
  // once per distinct mask, which cost a fifth of the kernel's instructions in the first version); lanes of a group
  // without an item are passengers
  constexpr unsigned FULL = 0xffffffffu;
  const unsigned child = sub / LC, u = sub % LC;
  // (passenger lanes run the same arithmetic on the first group's item -- valid memory, values unused)
  const hfb_bvh_node& nd = pair[child];
  m3 R;
  v3 T;
  double b0, b1, rad;
  q_rss_operands(s, nd, R, T, b0, b1, rad);
  const int fc = nd.first_child;
  RectPre p;
  rect_prelude(R, T, s.sbv[12], s.sbv[13], b0, b1, p);
  int kmine = 16;
  bool sub_found = false;
  const unsigned cmask = (1u << LC) - 1u;
#pragma unroll 1
  for (int t = 0; t < 16 / LC; ++t) {
    if (active && !sub_found && rect_case(p, LC * t + (int)u)) kmine = LC * t + (int)u;
    const unsigned b = __ballot_sync(FULL, kmine < 16) >> gbase;
    sub_found = ((b >> (LC * child)) & cmask) != 0u;
    const bool group_done = !active || ((b & cmask) != 0u && ((b >> LC) & cmask) != 0u);  // both children have their case
    if (__all_sync(FULL, group_done)) break;
  }
  int kwin = kmine;
#pragma unroll
  for (int off = 1; off < LC; off <<= 1) kwin = min(kwin, __shfl_xor_sync(FULL, kwin, off));
  double dist = 0;
  if (kwin < 16 ? (kmine == kwin) : (u == 0u)) {
    dist = rect_finish(p, kwin < 16 ? kwin : -1);
    dist -= rad;
    dist = (dist < 0.0) ? 0.0 : dist;
  }
  const unsigned src0 = gbase + (kwin < 16 ? (unsigned)(kwin % LC) : 0u);
  // every lane of a child asks its own child's winner; then the group leader collects both
  const double dc = __shfl_sync(FULL, dist, (int)(src0 + LC * child));
  d1 = __shfl_sync(FULL, dc, (int)gbase);
  d2 = __shfl_sync(FULL, dc, (int)gbase + LC);
  f1 = __shfl_sync(FULL, fc, (int)gbase);
  f2 = __shfl_sync(FULL, fc, (int)gbase + LC);
}

__global__ void __launch_bounds__(128) k_bvhq_prep(const BvhqLaunch L) {
  const unsigned lo = *L.range_lo, hi = *L.range_hi;
  for (unsigned k = blockIdx.x * blockDim.x + threadIdx.x; k < hi - lo; k += gridDim.x * blockDim.x) {
    const unsigned i = L.index_list[lo + k];
    const xf t1 = load_xf(L.tf1[i].R), t2 = load_xf(L.tf2[i].R);
    BvhJob job;
    QPrep& pr = L.prep[k];
    if (!bvh_make_job<CAPS_BVHQ, 0>(L.A, L.h1[i], t1, L.h2[i], t2, L.B, mk(1, 0, 0), 0, 0, L.out + i, job)) {
      pr.ok = 0;
      continue;
    }
    q_make_prep(job.q, job.swapped, pr);
  }
}

template <int THREADS>
__global__ void __launch_bounds__(THREADS, 1) k_bvhq(const BvhqLaunch L) {
  extern __shared__ __align__(16) unsigned char q_smem[];
  QSlot* slots = reinterpret_cast<QSlot*>(q_smem);
  QTreeletHot* hot = reinterpret_cast<QTreeletHot*>(q_smem + HFB_Q_NSLOTS * sizeof(QSlot));
  QSched* sc = reinterpret_cast<QSched*>(q_smem + HFB_Q_NSLOTS * sizeof(QSlot) + HFB_Q_NTREELETS * sizeof(QTreeletHot));
  const unsigned lo = *L.range_lo, hi = *L.range_hi;
  const unsigned lane = threadIdx.x & 31u;
  if (threadIdx.x == 0) {
    sc->lhead = sc->ltail = sc->bhead = sc->btail = sc->ehead = sc->etail = 0;
    sc->lsnap = sc->do_epa = sc->stop = 0;
    sc->active = 0;
    sc->tl_free = (1u << HFB_Q_NTREELETS) - 1u;
    sc->abort_ = 0;
  }
  for (unsigned k = threadIdx.x; k < HFB_Q_QCAP; k += blockDim.x) {
    sc->leafq[k] = 0u;
    sc->bvq[k] = 0u;
    sc->epaq[k] = 0u;
  }
  __syncthreads();
  QStackEnt* stacks = L.stacks + (size_t)blockIdx.x * HFB_Q_NSLOTS * (size_t)L.stack_cap;
  QTreelet* tls = L.treelets + (size_t)blockIdx.x * HFB_Q_NTREELETS;
  EpaWs* ws = L.ws + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  QLeafSave* saves = L.saves + (size_t)blockIdx.x * (HFB_Q_NSLOTS + 2 * HFB_Q_TREELET_MAX * HFB_Q_NTREELETS);
  DevSink sink{sc};
  QCtx c;
  c.P = L.P;
  c.rel_err = L.B.rel_err;
  c.abs_err = L.B.abs_err;
  c.spec_after = (L.P.initial_guess == HFB_GUESS_CACHED) ? -1 : L.spec_after;
  c.spec_big_after = L.spec_big_after;
  unsigned long long bv_total = 0, leaf_total = 0;
  {  // thread t fills slot t
    const unsigned sl = threadIdx.x;
    if (sl < HFB_Q_NSLOTS && q_fetch(L, lo, hi, slots[sl], stacks + (size_t)sl * L.stack_cap, sl, sink))
      atomicAdd(&sc->active, 1);
  }
  __syncthreads();
  const QBlock B{slots, stacks, tls, hot, sc, lo, hi};
  // up to `want` items of one queue for this warp; 0 when the queue is empty
  auto pop = [&](int* head, int* tail, int want, int& base, const int* limit = nullptr) -> int {
    int cnt = 0;
    if (lane == 0) {
      for (;;) {
        const int h = vload(head);
        int avail = vload(tail) - h;
        if (limit && vload(limit) - h < avail) avail = vload(limit) - h;
        if (avail <= 0) break;
        cnt = avail < want ? avail : want;
        if (atomicCAS(head, h, h + cnt) == h) {
          base = h;
          break;
        }
        cnt = 0;
      }
    }
    cnt = __shfl_sync(0xffffffffu, cnt, 0);
    base = __shfl_sync(0xffffffffu, base, 0);
    return cnt;
  };
  // one task of G-lane groups over `cnt` BV items starting at ring position `base`
  auto bv_task = [&](auto lc_tag, int cnt, int base) {
    constexpr int LC = decltype(lc_tag)::value, G = 2 * LC;
    const unsigned g = lane / G, sub = lane % G, gbase = g * G;
    const bool mine = (int)g < cnt;
    volatile unsigned* q = sc->bvq;
    const int pos = (base + (int)g) & (HFB_Q_QCAP - 1);
    unsigned item = 0;
    if (mine && sub == 0u) {
      item = q_take(q, pos, sc);
      q[pos] = 0u;
    }
    item = __shfl_sync(0xffffffffu, item, (int)gbase);
    __threadfence_block();
    const bool active = mine && (item & HFB_Q_ITEM_VALID) != 0u;
    item &= ~HFB_Q_ITEM_VALID;
    // passenger lanes (groups without an item) run the arithmetic of group 0's item: valid memory, results unused
    const unsigned item0 = __shfl_sync(0xffffffffu, item, 0);  // (every lane takes part in the shuffle)
    const unsigned item_x = active ? item : item0;
    const unsigned sl = item_x & HFB_Q_SLOT_MASK;
    QSlot& s = slots[sl];
    const hfb_bvh_node* nodes = static_cast<const hfb_bvh_node*>(s.ptr[0]);
    double d1, d2;
    int f1, f2;
    q_bv_group<LC>(active, s, nodes + q_bv_base(s, item_x), gbase, sub, d1, d2, f1, f2);
    bool have;
    QStackEnt near;
    if (active && sub == 0u && q_bv_store(s, item, stacks + (size_t)sl * L.stack_cap, hot, sink, d1, d2, f1, f2, have, near))
      q_continue(L, B, c, sl, bv_total, leaf_total, have, near);
    __syncwarp();
  };
  long long t_prev = clock64(), t_bv = 0, t_leaf = 0, t_epa = 0, n_cycles = 0, n_epa = 0;
  auto lap = [&](long long& acc) {
    const long long t = clock64();
    acc += t - t_prev;
    t_prev = t;
  };
  for (;;) {
    // ---- bounding-volume phase: bv_gens generations of items.  A generation is what was queued when it started;
    // the items it pushes (a walk going down a level) are the next generation.  Running "until the queue is empty"
    // instead made every cycle wait for its deepest descent with a handful of lanes busy
    // (BV phases of several times the length of the leaf phases). ----
    for (int gen = 0; gen < L.bv_gens; ++gen) {
      if (gen > 0) __syncthreads();
      if (threadIdx.x == 0) {
        sc->lsnap = vload(&sc->btail);
        sc->bn0 = sc->lsnap - vload(&sc->bhead);
      }
      __syncthreads();
      const int nb0 = vload(&sc->bn0);
      if (nb0 <= 0) break;  // (uniform: written by thread 0 before the barrier, by nobody after it)
      const int ipw = (nb0 + (THREADS / 32) - 1) / (THREADS / 32);  // items per warp
      int base = 0, cnt;
      // lanes per child: the fewer items, the more lanes share one (shorter dependent chain per task)
      if (ipw > 8) {
        while ((cnt = pop(&sc->bhead, &sc->btail, 16, base, &sc->lsnap)) > 0) bv_task(std::integral_constant<int, 1>(), cnt, base);
      } else if (ipw > 4) {
        while ((cnt = pop(&sc->bhead, &sc->btail, 8, base, &sc->lsnap)) > 0) bv_task(std::integral_constant<int, 2>(), cnt, base);
      } else {
        while ((cnt = pop(&sc->bhead, &sc->btail, 4, base, &sc->lsnap)) > 0) bv_task(std::integral_constant<int, 4>(), cnt, base);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      lap(t_bv);
      const int nl = vload(&sc->ltail) - vload(&sc->lhead), ne = vload(&sc->etail) - vload(&sc->ehead);
      sc->lsnap = vload(&sc->ltail);
      // EPA items are rare and long: they wait until there are enough of them to fill lanes, or nothing else is left
      sc->do_epa = (ne >= 32 || (ne > 0 && nl == 0)) ? 1 : 0;
    }
    __syncthreads();
    // ---- leaf phase: the items queued before it started; each runs at most gjk_chunk GJK iterations ----
    {
      const int nl0 = vload(&sc->lsnap) - vload(&sc->lhead);
      int want = (nl0 + (THREADS / 32) - 1) / (THREADS / 32);  // spread over the warps: a task is as long as its longest item
      want = want < 1 ? 1 : (want > 32 ? 32 : want);
      int base = 0, cnt;
      while ((cnt = pop(&sc->lhead, &sc->ltail, want, base, &sc->lsnap)) > 0) {
        if ((int)lane < cnt) {
          volatile unsigned* q = sc->leafq;
          const int pos = (base + (int)lane) & (HFB_Q_QCAP - 1);
          unsigned item = q_take(q, pos, sc);
          q[pos] = 0u;
          __threadfence_block();
          const bool valid = (item & HFB_Q_ITEM_VALID) != 0u;
          item &= ~HFB_Q_ITEM_VALID;
          const unsigned sl = item & HFB_Q_SLOT_MASK;
          QSlot& s = slots[sl];
          const bool spec = (item & HFB_Q_ITEM_SPEC) != 0u;
          if (valid) {
            QLeafRes r;
            QLeafSave& sv = saves[q_save_index(s, item, HFB_Q_NSLOTS)];
            const int st = q_leaf_gjk<CAPS_BVHQ>(s, q_leaf_prim(s, hot, item), L.P, !spec, (item & HFB_Q_ITEM_RESUME) != 0u,
                                                 L.gjk_chunk, sv, r);
            if (st == QL_SUSPENDED) sink.push_leaf(item | HFB_Q_ITEM_RESUME);
            else if (st == QL_NEED_EPA) sink.push_epa(item & ~HFB_Q_ITEM_RESUME);
            else if (q_leaf_store(s, item, tls, hot, sink, r)) q_continue(L, B, c, sl, bv_total, leaf_total, false, QStackEnt());
          }
        }
        __syncwarp();
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) lap(t_leaf);
    // ---- EPA phase (some cycles only) ----
    if (vload(&sc->do_epa)) {
      const int ne0 = vload(&sc->etail) - vload(&sc->ehead);
      int want = (ne0 + (THREADS / 32) - 1) / (THREADS / 32);
      want = want < 1 ? 1 : (want > 32 ? 32 : want);
      int base = 0, cnt;
      while ((cnt = pop(&sc->ehead, &sc->etail, want, base)) > 0) {
        if ((int)lane < cnt) {
          volatile unsigned* q = sc->epaq;
          const int pos = (base + (int)lane) & (HFB_Q_QCAP - 1);
          unsigned item = q_take(q, pos, sc);
          q[pos] = 0u;
          __threadfence_block();
          const bool valid = (item & HFB_Q_ITEM_VALID) != 0u;
          item &= ~HFB_Q_ITEM_VALID;
          const unsigned sl = item & HFB_Q_SLOT_MASK;
          QSlot& s = slots[sl];
          const bool spec = (item & HFB_Q_ITEM_SPEC) != 0u;
          if (valid) {
            QLeafRes r;
            q_leaf_epa<CAPS_BVHQ>(s, q_leaf_prim(s, hot, item), L.P, !spec, ws, saves[q_save_index(s, item, HFB_Q_NSLOTS)], r);
            if (q_leaf_store(s, item, tls, hot, sink, r)) q_continue(L, B, c, sl, bv_total, leaf_total, false, QStackEnt());
          }
        }
        __syncwarp();
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        lap(t_epa);
        ++n_epa;
      }
    }
    if (threadIdx.x == 0) {
      ++n_cycles;
      sc->stop = (vload(&sc->active) <= 0 || vload(&sc->abort_)) ? 1 : 0;
    }
    __syncthreads();  // nobody retires a query (changes `active`) between thread 0's read and this barrier
    if (vload(&sc->stop)) break;
  }
  if (bv_total) atomicAdd(L.counters, bv_total);
  if (leaf_total) atomicAdd(L.counters + 1, leaf_total);
  __syncthreads();
  if (threadIdx.x == 0 && sc->abort_ && sc->active > 0) atomicAdd(L.counters + 2, 1ull);
  if (threadIdx.x == 0) {  // phase profile (clock cycles summed over the blocks; hfb_debug_bvh_profile)
    atomicAdd(L.counters + 3, (unsigned long long)t_bv);
    atomicAdd(L.counters + 4, (unsigned long long)t_leaf);
    atomicAdd(L.counters + 5, (unsigned long long)t_epa);
    atomicAdd(L.counters + 6, (unsigned long long)n_cycles);
    atomicAdd(L.counters + 7, (unsigned long long)n_epa);
  }
}

static size_t bvhq_smem_bytes() { return HFB_Q_NSLOTS * sizeof(QSlot) + HFB_Q_NTREELETS * sizeof(QTreeletHot) + sizeof(QSched); }

unsigned bvhq_blocks(int num_sms, size_t n) {
  // a block is worth launching for every 64 queries; never more than one per SM (persistent)
  size_t b = (n + 63) / 64;
  if (b > (size_t)num_sms) b = (size_t)num_sms;
  return b ? (unsigned)b : 1u;
}

BvhqSizes bvhq_sizes(unsigned blocks, size_t n, int stack_cap) {
  BvhqSizes z;
  z.prep = n * sizeof(QPrep);
  z.stacks = (size_t)blocks * HFB_Q_NSLOTS * (size_t)stack_cap * sizeof(QStackEnt);
  z.treelets = (size_t)blocks * HFB_Q_NTREELETS * sizeof(QTreelet);
  z.ws = (size_t)blocks * HFB_Q_MAX_THREADS * sizeof(EpaWs);
  z.saves = (size_t)blocks * (HFB_Q_NSLOTS + 2 * HFB_Q_TREELET_MAX * HFB_Q_NTREELETS) * sizeof(QLeafSave);
  return z;
}

int bvhq_launch(const BvhqLaunch& L, unsigned blocks, size_t n, cudaStream_t s) {
  static_assert(HFB_Q_NSLOTS <= 256, "thread t fills slot t");
  static_assert(HFB_Q_NSLOTS + HFB_Q_TREELET_MAX * HFB_Q_NTREELETS <= HFB_Q_QCAP, "each ring holds every item of its kind that can exist");
  static_assert(sizeof(QSlot) % 16 == 8, "odd stride in 8-byte words: lanes reading one field of 32 slots spread over the banks");
  const size_t smem = bvhq_smem_bytes();
  const int threads = L.warps >= 16 ? 512 : (L.warps >= 12 ? 384 : 256);
  cudaError_t e = threads == 512   ? cudaFuncSetAttribute(k_bvhq<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                  : threads == 384 ? cudaFuncSetAttribute(k_bvhq<384>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                                   : cudaFuncSetAttribute(k_bvhq<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  unsigned pb = (unsigned)((n + 127) / 128);
  if (pb > blocks * 16u) pb = blocks * 16u;
  if (pb == 0) pb = 1;
  k_bvhq_prep<<<pb, 128, 0, s>>>(L);
  if (threads == 512) k_bvhq<512><<<blocks, 512, smem, s>>>(L);
  else if (threads == 384) k_bvhq<384><<<blocks, 384, smem, s>>>(L);
  else k_bvhq<256><<<blocks, 256, smem, s>>>(L);
  return (int)cudaGetLastError();
}

}  // namespace hfb
