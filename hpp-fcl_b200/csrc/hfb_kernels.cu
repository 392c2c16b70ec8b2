// CUDA kernels (sm_90a) of the narrow phase and the C-ABI of include/hppfcl_b200.h for the context, the geometry and the
// batch calls.  The rest of the C-ABI:
//   hfb_scene.cu   broadphase feed, hfb_scene_collide(_sets) and the resident environment (hfb_env_*), with the four
//                  small kernels only they launch
//   hfb_robot.cu   robot models (hfb_robot_*) next to k_robot
//   hfb_comm.cu    multi-GPU (hfb_comm_*, hfb_geom_broadcast and the sharded batch calls)
//   hfb_ctx.h      what these files share: the context and its buffers, error and CUDA checks, objects_device
//
// Kernel inventory (DESIGN.md section 3 has the measurements)
//   k_bin_hist/scan/scatter  device-side counting sort of the batch by pair class (closed-form combos |
//                          GJK-routed primitive combos | touches ConvexBase/TriangleP | mesh-shape |
//                          mesh-mesh): every warp of the kernels below meets one class
//   k_pairs<G,CAPS,MODE,PATHS,MINB,STAGE>  phase 1, a lane group of G threads per pair: closed form, or GJK +
//                          witness extraction; pairs that need EPA are appended to a device queue.
//                          Instantiated per class family (PATHS) to keep each kernel's code small;
//                          STAGE adds cp.async.bulk staging of the hulls' vertex blocks
//   k_gjk_refill<MODE>     optional (HFB_REFILL=1): phase 1 for primitive pairs with lane refill
//   k_epa<G,CAPS,MODE,TIER>  phase 2 over the EPA queue, polytope in shared memory; tier 0 in a
//                          reduced-size workspace, tier 1 retries the pairs that outgrew it
//   k_bvh<MODE,KINDS,MINB> OBBRSS tree walks: mesh-shape (warp-scheduled, exact DFS order) and mesh-mesh
//   k_convex_support       batched ConvexBase support argmax (warp per query, coalesced streaming of the
//                          vertex block: HBM-bound over a 1.2 GB pool)
// MODE 0 = distance() epilogue, MODE 1 = collide() epilogue.
#include <cuda_runtime.h>

#include <chrono>

#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "hfb_ctx.h"
#include "hfb_bvh_build.cuh"
#include "hfb_bvhq_launch.h"
#include "hfb_gjkpass.h"
#include "hfb_hullsort.h"
#include "hfb_broadphase.cuh"

// lanes per pair of the EPA kernel's second tier (k_epa<G,CAPS,MODE,1>), whatever HFB_GE asks for the first
#define HFB_GE_TIER1 32
// lane groups per SM the global-memory support-point store of tier 0 is sized for (k_epa; the largest first-tier shape)
#define HFB_EPA_SUP_GROUPS_PER_SM 64

// pair classes of the device-side counting sort (k_bin_*): bins [0,9) closed-form
// combos (bin 8: a plane or halfspace against a primitive or another plane), [9,45) GJK-routed
// primitive combos, bin 45: unknown node types (reported as unsupported), bin 46: pairs touching
// ConvexBase / TriangleP
#define HFB_NBINS 49
#define HFB_BIN_PLANE 8
#define HFB_BIN_GJK0 9
#define HFB_BIN_UNKNOWN 45
#define HFB_BIN_CONVEX 46
#define HFB_BIN_BVH 47   // one operand is a BVHModel<OBBRSS>
#define HFB_BIN_BVH2 48  // both are

// ------------------------------------------------------------------ phase 1 --
// ---- TMA staging of ConvexBase vertex blocks (lane-group kernels) -------------------------------
// A group's two hulls are copied once per pair from the arena into the group's shared-memory slots by
// the copy engine (cp.async.bulk, completion on an mbarrier); the GJK loop's support argmax then reads
// shared memory.  One SoA block x[vpad] y[vpad] z[vpad] is contiguous and 16-byte aligned in the pool
// (hfb_arena.cuh), i.e. one bulk copy per hull.  Hulls above HFB_STAGE_MAXV vertices stay in global memory.
#define HFB_STAGE_MAXV 64
#define HFB_STAGE_SLOT_BYTES (3 * HFB_STAGE_MAXV * 8)
struct __align__(16) StageGroup {  // double-buffered: the next pair's hulls land while this pair computes
  double slot[2][2][3 * HFB_STAGE_MAXV];  // [buffer][operand]
  unsigned long long mbar[2];
};
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* m, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(m)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* m, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(m)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* m) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(m))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* m, unsigned parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "HFB_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra HFB_DONE;\n\t"
      "bra HFB_WAIT;\n\t"
      "HFB_DONE:\n\t"
      "}" ::"r"(smem_u32(m)),
      "r"(parity)
      : "memory");
}
// vertex block of shape handle h if it is a ConvexBase that fits a slot: pointer + bytes (else 0 bytes)
__device__ __forceinline__ unsigned stage_block(const ArenaView& A, uint32_t h, const double*& src) {
  const hfb_shape& r = A.shapes[h];
  if (r.type != HFB_GEOM_CONVEX) return 0u;
  const ConvexDesc& d = A.cvx[r.data];
  const unsigned b = d.vpad * 24u;  // 3 arrays of vpad doubles
  src = A.pool + d.off;
  return b <= HFB_STAGE_SLOT_BYTES ? b : 0u;
}
// lane 0 of a group: start the copies of pair i's hulls into buffer `buf`
__device__ __forceinline__ void stage_issue(const BatchArgs& a, unsigned i, StageGroup* sg, int buf) {
  const double *p1 = nullptr, *p2 = nullptr;
  const unsigned b1 = stage_block(a.A, a.h1[i], p1), b2 = stage_block(a.A, a.h2[i], p2);
  if (b1 | b2) {
    // the buffer was last read through the generic proxy (two pairs ago, ordered by the group sync at the
    // end of the loop body); the copy engine writes through the async proxy
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    mbar_expect_tx(&sg->mbar[buf], b1 + b2);
    if (b1) bulk_g2s(sg->slot[buf][0], p1, b1, &sg->mbar[buf]);
    if (b2) bulk_g2s(sg->slot[buf][1], p2, b2, &sg->mbar[buf]);
  }
}
__device__ __forceinline__ unsigned stage_bytes(const ShapeD& s) {
  if (s.type != HFB_GEOM_CONVEX) return 0u;
  const unsigned b = (unsigned)(s.cy - s.cx) * 24u;
  return b <= HFB_STAGE_SLOT_BYTES ? b : 0u;
}

// ------------------------------------------------------------------ phase 1 --
template <int G, int CAPS, int MODE, int PATHS, int MINB, bool STAGE_>
__global__ void __launch_bounds__(128, MINB) k_pairs(const BatchArgs a) {
  constexpr bool STAGE = STAGE_ && (G > 1) && (CAPS & CAP_CONVEX);
  extern __shared__ __align__(16) unsigned char dyn_smem[];
  StageGroup* sg = nullptr;
  unsigned parity0 = 0, parity1 = 0;
  int buf = 0;
  if (STAGE) {
    sg = reinterpret_cast<StageGroup*>(dyn_smem) + threadIdx.x / G;
    if (Coop<G>::lane() == 0) {
      mbar_init(&sg->mbar[0], 1);
      mbar_init(&sg->mbar[1], 1);
    }
    Coop<G>::sync();
  }
  const unsigned ngroups = (gridDim.x * blockDim.x) / G;
  const unsigned gid = (blockIdx.x * blockDim.x + threadIdx.x) / G;
  unsigned lo = a.index_list ? *a.range_lo : 0u;
  unsigned hi = a.index_list ? *a.range_hi : a.n;
  if (a.sub_cnt > 1) {
    const unsigned long long len = hi - lo;
    const unsigned l2 = lo + (unsigned)(len * a.sub_idx / a.sub_cnt);
    hi = lo + (unsigned)(len * (a.sub_idx + 1) / a.sub_cnt);
    lo = l2;
  }
  if (STAGE && lo + gid < hi && Coop<G>::lane() == 0)
    stage_issue(a, a.index_list ? a.index_list[lo + gid] : lo + gid, sg, 0);
  for (unsigned k = lo + gid; k < hi; k += ngroups) {
    const unsigned i = a.index_list ? a.index_list[k] : k;
    PairIn in = load_pair_in<CAPS>(a, i);
    if (STAGE) {
      // next pair's hulls into the other buffer (its readers finished before the sync that ended the
      // previous iteration)
      if (k + ngroups < hi && Coop<G>::lane() == 0)
        stage_issue(a, a.index_list ? a.index_list[k + ngroups] : k + ngroups, sg, buf ^ 1);
      const unsigned b1 = stage_bytes(in.s1), b2 = stage_bytes(in.s2);
      if (b1 | b2) {
        mbar_wait(&sg->mbar[buf], buf ? parity1 : parity0);
        if (buf) parity1 ^= 1u;
        else parity0 ^= 1u;
        if (b1) {
          const unsigned vpad = (unsigned)(in.s1.cy - in.s1.cx);
          in.s1.cx = sg->slot[buf][0];
          in.s1.cy = sg->slot[buf][0] + vpad;
          in.s1.cz = sg->slot[buf][0] + 2 * vpad;
        }
        if (b2) {
          const unsigned vpad = (unsigned)(in.s2.cy - in.s2.cx);
          in.s2.cx = sg->slot[buf][1];
          in.s2.cy = sg->slot[buf][1] + vpad;
          in.s2.cz = sg->slot[buf][1] + 2 * vpad;
        }
      }
      buf ^= 1;
    }
    PairOut o;
    GjkState g;
    const bool need_epa = pair_phase1<G, CAPS, PATHS>(in, a.P, o, g);
    if (Coop<G>::lane() == 0) {
      if (need_epa) {
        const unsigned slot = atomicAdd(a.queue_count, 1u);
        atomicAdd(a.queue_count + 1, 1u);
        EpaItem* it = a.queue + slot;
        it->pair = i + a.pair_base;
        it->rank = g.rank;
        it->hint0 = g.hint0;
        it->hint1 = g.hint1;
        it->gjk_iterations = g.iterations;
        st3(it->w0 + 0, g.s0.w0);
        st3(it->w1 + 0, g.s0.w1);
        st3(it->w0 + 3, g.s1.w0);
        st3(it->w1 + 3, g.s1.w1);
        st3(it->w0 + 6, g.s2.w0);
        st3(it->w1 + 6, g.s2.w1);
        st3(it->w0 + 9, g.s3.w0);
        st3(it->w1 + 9, g.s3.w1);
      } else {
        store_result<MODE>(a, i, o);
      }
    }
    if (STAGE) Coop<G>::sync();  // every lane is done with the slots before the next pair's copy lands
  }
}

// Phase 1 for the GJK-routed primitive classes with lane refill.  GJK takes 3 to 26 iterations inside
// one class; with a pair per lane for the whole kernel a warp runs at the pace of its slowest pair
// (few lanes active per instruction).  Here a lane is in one of three states -- needs a pair,
// iterating, needs its result extracted -- and the warp alternates between an iteration round (every
// iterating lane does one GJK iteration) and a service round (finished lanes extract + store or queue
// for EPA, then every free lane takes the next pair and sets it up).  Results do not depend on the
// schedule: every pair runs gjk_begin / gjk_step* / pair_gjk_end exactly as in pair_phase1.
enum { GR_FETCH = 0, GR_ITER = 1, GR_FINISH = 2, GR_EXIT = 3 };
template <int MODE>
__global__ void __launch_bounds__(128, 1) k_gjk_refill(const BatchArgs a) {
  unsigned lo = *a.range_lo, hi = *a.range_hi;
  if (a.sub_cnt > 1) {
    const unsigned long long len = hi - lo;
    const unsigned l2 = lo + (unsigned)(len * a.sub_idx / a.sub_cnt);
    hi = lo + (unsigned)(len * (a.sub_idx + 1) / a.sub_cnt);
    lo = l2;
  }
  const unsigned lane = threadIdx.x & 31u;
  const unsigned lt_mask = (1u << lane) - 1u;
  int state = GR_FETCH;
  unsigned i = 0;
  GjkSetup S;
  GjkLoop L;
  GjkState g;
  PairOut o;
  for (;;) {
    const unsigned m_iter = __ballot_sync(0xffffffffu, state == GR_ITER);
    const unsigned m_serv = __ballot_sync(0xffffffffu, state == GR_FETCH || state == GR_FINISH);
    if (!(m_iter | m_serv)) break;
    if (m_serv == 0 || __popc(m_iter) >= (int)a.iter_quorum) {
      if (state == GR_ITER) {
        if (!gjk_step<1, CAP_PRIM>(S.a, S.b, S.md, a.P.gjk, g, L)) state = GR_FINISH;
      }
    } else {
      if (state == GR_FINISH) {
        o.iterations = 0;
        if (pair_gjk_end(a.P, S, g, o)) push_epa_item(a, i, g);
        else store_result<MODE>(a, i, o);
        state = GR_FETCH;
      }
      // every free lane takes the next pair: one counter bump per warp
      const unsigned m_fetch = __ballot_sync(0xffffffffu, state == GR_FETCH);
      unsigned base = 0;
      if (lane == (unsigned)(__ffs(m_fetch) - 1)) base = atomicAdd(a.gjk_work, (unsigned)__popc(m_fetch));
      base = __shfl_sync(0xffffffffu, base, __ffs(m_fetch) - 1);
      if (state == GR_FETCH) {
        const unsigned k = lo + base + (unsigned)__popc(m_fetch & lt_mask);
        if (k < hi) {
          i = a.index_list[k];
          const PairIn in = load_pair_in<CAP_PRIM>(a, i);
          pair_gjk_begin<CAP_PRIM>(in, a.P, S, L, g, o);
          state = GR_ITER;
        } else {
          state = GR_EXIT;
        }
      }
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------ phase 2 --
// EPA runs in two tiers.  Tier 0 gives every pair a reduced-size workspace (EpaPolySmall), so that 64 lane groups fit in
// one SM (4 blocks x 16 groups at 8 lanes per pair) instead of 20: the kernel is bound by the latency of one pair's
// dependent FP64 chain, and throughput is the number of pairs in flight.  A pair whose polytope outgrows it is appended
// to the retry list and run again by tier 1 in the full-size workspace.
// Tier 0 keeps only the polytope in shared memory.  The support points w0 / w1 of its vertices, which the loop writes
// and never reads, go to global memory (EpaSupArray), one slot per resident lane group: blockIdx.x * GPB + group.
template <int G, int TIER>
struct EpaCfg {
  typedef EpaWs WS;
  static constexpr int GPB = (G == 32) ? 4 : 10;  // two blocks per SM (G <= 16); registers bound G = 32
  static constexpr int THREADS = GPB * G;
  static constexpr int MINB = 1;
};
template <int G>
struct EpaCfg<G, 0> {
  typedef EpaPolySmall WS;
  static constexpr int GPB = (G == 4) ? 24 : ((G == 8) ? 16 : (G == 16 ? 16 : 8));
  static constexpr int THREADS = GPB * G;
  // G = 8: 4 blocks x 16 groups per SM at 128 registers (16 warps: 4 per SM sub-partition of 16 K registers); G = 4:
  // 2 blocks x 24 groups
  static constexpr int MINB = (G == 8) ? 4 : (G == 4 ? 2 : 1);
};
template <int G, int TIER, class WS>
__device__ __forceinline__ auto epa_side(const BatchArgs& a, WS* ws, unsigned lg) {
  if constexpr (TIER == 0) {
    return EpaSupArray{a.epa_sup + (size_t)(blockIdx.x * EpaCfg<G, 0>::GPB + lg) * (6 * WS::MAXV)};
  } else {
    return EpaSideWs<WS>{ws};
  }
}
template <int G, int CAPS, int MODE, int TIER>
__global__ void __launch_bounds__(EpaCfg<G, TIER>::THREADS, EpaCfg<G, TIER>::MINB) k_epa(const BatchArgs a) {
  typedef typename EpaCfg<G, TIER>::WS WS;
  extern __shared__ __align__(16) unsigned char smem[];
  const unsigned lg = threadIdx.x / G;  // group within block
  WS* ws = reinterpret_cast<WS*>(smem) + lg;
  const auto sd = epa_side<G, TIER>(a, ws, lg);
  const unsigned lo = TIER == 0 ? *a.epa_lo : 0u, hi = TIER == 0 ? *a.epa_hi : *a.retry_count;
  for (;;) {
    unsigned k = 0;
    if (Coop<G>::lane() == 0) k = lo + atomicAdd(a.epa_head, 1u);
    k = __shfl_sync(Coop<G>::mask(), k, (threadIdx.x & 31u) & ~(unsigned)(G - 1));
    if (k >= hi) break;
    const unsigned k_pos = k;  // (tier 1: position in the retry list = slot of the continuation record)
    // tier 0 hands the queue out from its end: the first GJK pass fills it in pair-class order, with the cylinder
    // classes last, and the later passes append the pairs whose GJK ran longer.  Their runs are the longest, so starting
    // them first shortens the end of the launch
    if (TIER == 0) k = lo + hi - 1 - k;
    if (TIER == 1) k = a.retry[k];
    const EpaItem* it = a.queue + k;
    const unsigned i = it->pair;
    // the loop needs the two shapes and the Minkowski set-up only; the pose the witness points are mapped back with
    // is read again when the run is over instead of being kept in registers across the loop
    GjkSetup S;
    make_setup<CAPS>(load_pair_in<CAPS>(a, i), S);
    GjkState g;
    g.rank = it->rank;
    g.hint0 = it->hint0;
    g.hint1 = it->hint1;
    g.iterations = it->gjk_iterations;
    g.status = HFB_GJK_COLLISION;
    g.distance = 0;
    g.ray = mk(0, 0, 0);
    g.s0.w0 = ld3(it->w0 + 0);
    g.s0.w1 = ld3(it->w1 + 0);
    g.s1.w0 = ld3(it->w0 + 3);
    g.s1.w1 = ld3(it->w1 + 3);
    g.s2.w0 = ld3(it->w0 + 6);
    g.s2.w1 = ld3(it->w1 + 6);
    g.s3.w0 = ld3(it->w0 + 9);
    g.s3.w1 = ld3(it->w1 + 9);
    g.s0.w = g.s0.w0 - g.s0.w1;
    g.s1.w = g.s1.w0 - g.s1.w1;
    g.s2.w = g.s2.w0 - g.s2.w1;
    g.s3.w = g.s3.w0 - g.s3.w1;
    Coop<G>::sync();
    EpaResume rs;
    bool done;
    if (TIER == 0) {
      done = pair_epa<G, CAPS>(S, a.P, g, ws, sd, rs);
      if (!done) {
        unsigned r = 0;
        if (Coop<G>::lane() == 0) {
          r = atomicAdd(a.retry_count, 1u);
          a.retry[r] = k;
        }
        r = __shfl_sync(Coop<G>::mask(), r, (threadIdx.x & 31u) & ~(unsigned)(G - 1));
        if (a.cont && r < a.cont_cap) {  // (the group's lanes hold the same rs)
          EpaCont* c = a.cont + r;
          if (rs.L.resumable) {
            Coop<G>::sync();  // the support points the other lanes stored
            epa_ws_grow<G>(ws, sd, &c->ws, EpaSupArray{c->sp}, rs.E);
          }
          if (Coop<G>::lane() == 0) c->rs = rs;
        }
      }
    } else {
      const unsigned kk = k_pos;
      if (a.cont && kk < a.cont_cap && a.cont[kk].rs.L.resumable) {
        rs = a.cont[kk].rs;
        epa_ws_grow<G>(&a.cont[kk].ws, EpaSupArray{a.cont[kk].sp}, ws, sd, rs.E);
        done = pair_epa_resume<G, CAPS>(S, a.P, ws, sd, rs);
      } else {
        done = pair_epa<G, CAPS>(S, a.P, g, ws, sd, rs);
      }
    }
    if (done) {
      // make_setup's tfa: the first pose, or the second one when the operands were swapped (a triangle first)
      S.tfa = load_xf((S.swapped ? a.tf2 : a.tf1)[i].R);
      if constexpr (TIER == 0) Coop<G>::sync();  // the support points the other lanes stored
      PairOut o;
      pair_epa_result(S, g.iterations, rs, ws, sd, o);
      if (Coop<G>::lane() == 0) store_result<MODE>(a, i, o);
    }
    Coop<G>::sync();
  }
}

// ----------------------------------------------------------------- BVH pairs ---
// One thread per (mesh, shape) query: per-query shape BV, depth-first traversal with a
// per-thread stack (RSS distance bounds / OBB SAT per node, loaded from the 256-B node
// records), triangle-shape GJK(+EPA) at the leaves.
// (mesh, shape) and (mesh, mesh) pairs.  Work is handed out one pair at a time from a counter: the
// walks differ tenfold in length, a fixed assignment would leave most lanes of a warp waiting.
__device__ __forceinline__ void bvh_load_pair(const BatchArgs& a, unsigned i, xf& t1, xf& t2, v3& guess, int& h0,
                                              int& h1) {
  t1 = load_xf(a.tf1[i].R);
  t2 = load_xf(a.tf2[i].R);
  guess = mk(1, 0, 0);
  h0 = h1 = 0;
  if (a.P.initial_guess == HFB_GUESS_CACHED) {
    if (a.guess_in) guess = mk(a.guess_in[3 * i], a.guess_in[3 * i + 1], a.guess_in[3 * i + 2]);
    if (a.hint_in) {
      h0 = a.hint_in[2 * i];
      h1 = a.hint_in[2 * i + 1];
    }
  }
}
__device__ __forceinline__ void bvh_set_sink(BvhJob&, const BatchArgs&, unsigned) {}
__device__ __forceinline__ void bvh_set_sink(BvhColJob& j, const BatchArgs& a, unsigned i) {
  j.sink = contact_sink(a, i);
  if (j.sink.count) *j.sink.count = 0;  // stays 0 for a pair that is not walked
}
template <int MODE>
struct BvhDeviceSrc {
  const BatchArgs& a;
  unsigned lo, hi;
  template <class Job>
  __device__ bool next(Job& j) {
    for (;;) {
      const unsigned k = lo + atomicAdd(a.bvh_work, 1u);
      if (k >= hi) return false;
      const unsigned i = a.index_list[k];
      xf t1, t2;
      v3 guess;
      int h0, h1;
      bvh_load_pair(a, i, t1, t2, guess, h0, h1);
      void* rec = MODE == 0 ? static_cast<void*>(reinterpret_cast<hfb_distance_result*>(a.out) + i)
                            : static_cast<void*>(reinterpret_cast<hfb_contact*>(a.out) + i);
      bvh_set_sink(j, a, i);
      if (bvh_make_job<CAPS_BVH, MODE>(a.A, a.h1[i], t1, a.h2[i], t2, a.B, guess, h0, h1, rec, j)) return true;
    }
  }
};
template <int MODE, int KINDS, int MINB, int QUORUM = HFB_BVH_INIT_QUORUM>
__global__ void __launch_bounds__(64, MINB) k_bvh(const BatchArgs a) {
  const unsigned tid = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned lo = *a.range_lo, hi = *a.range_hi;
  EpaWs* ws = a.bvh_ws + tid;
  unsigned long long bv_total = 0, leaf_total = 0;
  if (KINDS == BVK_SHAPE) {
    BvhDeviceSrc<MODE> src{a, lo, hi};
    if (MODE == 0)
      bvh_shape_distance_stream<CAPS_BVH, BvhDeviceSrc<MODE>, QUORUM>(src, a.P, a.B.rel_err, a.B.abs_err, ws, bv_total,
                                                                      leaf_total);
    else
      bvh_shape_collide_stream<CAPS_BVH, BvhDeviceSrc<MODE>, QUORUM>(src, a.P, a.B.security_margin, a.B.break_distance,
                                         a.B.collision_distance_threshold, a.B.num_max_contacts, ws, bv_total,
                                         leaf_total);
  } else {
    for (;;) {
      const unsigned k = lo + atomicAdd(a.bvh_work, 1u);
      if (k >= hi) break;
      const unsigned i = a.index_list[k];
      xf t1, t2;
      v3 guess;
      int h0, h1;
      bvh_load_pair(a, i, t1, t2, guess, h0, h1);
      unsigned bt, lt;
      if (MODE == 0)
        bvh_mesh_pair_distance(a.A, a.h1[i], t1, a.h2[i], t2, a.B, reinterpret_cast<hfb_distance_result*>(a.out) + i,
                               bt, lt);
      else
        bvh_mesh_pair_collide<CAPS_BVH>(a.A, a.h1[i], t1, a.h2[i], t2, a.P, a.B, guess, h0, h1, ws,
                                        reinterpret_cast<hfb_contact*>(a.out) + i, bt, lt, contact_sink(a, i));
      bv_total += bt;
      leaf_total += lt;
    }
  }
  if (bv_total) atomicAdd(a.bvh_counters, bv_total);
  if (leaf_total) atomicAdd(a.bvh_counters + 1, leaf_total);
}

// ---- hand-out order of the (mesh, shape) queries (HFB_BVH_ORDER=1; tests/tools/bvh_sched_model.py) ------------
// k_bvh is bound by its tail at BASELINE sizes: the longest walks should start first.  A walk is long when many
// triangles are about as near as the nearest one; the key of a query is the number of HFB_ORDER_SAMPLES sampled
// mesh vertices within 1.2 x the nearest sample's distance of the shape's centre (correlation 0.5 with the number
// of rounds on config 4).  A counting sort by descending key rewrites the slice of the class-sorted index list;
// results do not depend on the order.
#define HFB_ORDER_SAMPLES 128
__global__ void __launch_bounds__(128) k_bvh_order_keys(const BatchArgs a, const unsigned* lo_p, const unsigned* hi_p,
                                                        unsigned char* keys, unsigned* hist) {
  const unsigned lo = *lo_p, hi = *hi_p;
  for (unsigned k = lo + blockIdx.x * blockDim.x + threadIdx.x; k < hi; k += gridDim.x * blockDim.x) {
    const unsigned i = a.index_list[k];
    const hfb_shape& r1 = a.A.shapes[a.h1[i]];
    const bool swapped = !is_bvh_type(r1.type);
    const hfb_shape& rm = swapped ? a.A.shapes[a.h2[i]] : r1;
    const xf tm = load_xf(swapped ? a.tf2[i].R : a.tf1[i].R);
    const xf ts = load_xf(swapped ? a.tf1[i].R : a.tf2[i].R);
    unsigned key = 0;
    if (is_bvh_type(rm.type)) {
      const BvhDesc d = a.A.bvh_desc[rm.data];
      const double* v = a.A.bvh_verts + 3 * (size_t)d.vert_off;
      const v3 c = mtmul(tm.R, ts.T - tm.T);  // the shape's origin in the mesh frame
      const unsigned stride = d.num_verts > HFB_ORDER_SAMPLES ? d.num_verts / HFB_ORDER_SAMPLES : 1u;
      double dmin = DBL_MAX;
      for (unsigned j = 0, q = 0; j < HFB_ORDER_SAMPLES && q < d.num_verts; ++j, q += stride) {
        const v3 e = mk(v[3 * q], v[3 * q + 1], v[3 * q + 2]) - c;
        const double d2 = sqn(e);
        dmin = d2 < dmin ? d2 : dmin;
      }
      const double lim = dmin * (1.2 * 1.2);
      for (unsigned j = 0, q = 0; j < HFB_ORDER_SAMPLES && q < d.num_verts; ++j, q += stride) {
        const v3 e = mk(v[3 * q], v[3 * q + 1], v[3 * q + 2]) - c;
        key += sqn(e) <= lim ? 1u : 0u;
      }
    }
    keys[k - lo] = (unsigned char)key;
    atomicAdd(hist + key, 1u);
  }
}
// descending keys: cursor[key] = number of queries with a larger key
__global__ void k_bvh_order_scan(const unsigned* hist, unsigned* cursor) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    unsigned run = 0;
    for (int key = HFB_ORDER_SAMPLES; key >= 0; --key) {
      cursor[key] = run;
      run += hist[key];
    }
  }
}
__global__ void __launch_bounds__(128) k_bvh_order_scatter(const uint32_t* index_list, const unsigned* lo_p,
                                                           const unsigned* hi_p, const unsigned char* keys,
                                                           unsigned* cursor, uint32_t* out_list) {
  const unsigned lo = *lo_p, hi = *hi_p;
  for (unsigned k = lo + blockIdx.x * blockDim.x + threadIdx.x; k < hi; k += gridDim.x * blockDim.x) {
    const unsigned pos = atomicAdd(cursor + keys[k - lo], 1u);
    out_list[lo + pos] = index_list[k];
  }
}

// --------------------------------------------------- pair-class counting sort ---
__device__ __forceinline__ int type_index(uint32_t t) {
  switch (t) {
    case HFB_GEOM_BOX: return 0;
    case HFB_GEOM_SPHERE: return 1;
    case HFB_GEOM_CAPSULE: return 2;
    case HFB_GEOM_CONE: return 3;
    case HFB_GEOM_CYLINDER: return 4;
    case HFB_GEOM_ELLIPSOID: return 5;
    case HFB_GEOM_CONVEX: return 6;
    case HFB_GEOM_TRIANGLE: return 7;
    case HFB_BV_OBB:
    case HFB_BV_OBBRSS: return 9;
    case HFB_GEOM_PLANE:
    case HFB_GEOM_HALFSPACE: return 10;
    default: return 8;
  }
}
__device__ __forceinline__ int pair_bin(uint32_t t1, uint32_t t2) {
  const int a = type_index(t1), b = type_index(t2);
  if (a == 9 && b == 9) return HFB_BIN_BVH2;
  if (a == 9 || b == 9) return HFB_BIN_BVH;
  if (a == 8 || b == 8) return HFB_BIN_UNKNOWN;
  if (a == 10 || b == 10) {  // the plane family is closed-form against everything (src/distance/*_plane.cpp, *_halfspace.cpp)
    const int o = a == 10 ? b : a;
    return (o == 6 || o == 7) ? HFB_BIN_CONVEX : HFB_BIN_PLANE;  // hull / triangle partners need the vertex-set supports
  }
  if (a >= 6 || b >= 6) return HFB_BIN_CONVEX;
  if (is_closed_form((int)t1, (int)t2)) {  // same predicate the per-pair dispatch uses
    if (a == 1 && b == 1) return 0;
    if (a == 1 && b == 2) return 1;
    if (a == 2 && b == 1) return 2;
    if (a == 1 && b == 4) return 3;
    if (a == 4 && b == 1) return 4;
    if (a == 0 && b == 1) return 5;
    if (a == 1 && b == 0) return 6;
    return 7;  // capsule-capsule
  }
  return HFB_BIN_GJK0 + a * 6 + b;
}

// type of a handle; 0 (no such geometry -> HFB_BIN_UNKNOWN) for one the arena never issued
__device__ __forceinline__ uint32_t handle_type(const hfb_shape* shapes, uint32_t nshapes, uint32_t h) {
  return h < nshapes ? shapes[h].type : 0u;
}
__global__ void __launch_bounds__(256) k_bin_hist(const hfb_shape* shapes, uint32_t nshapes, const uint32_t* h1,
                                                  const uint32_t* h2, unsigned n, unsigned* hist) {
  __shared__ unsigned sh[HFB_NBINS];
  if (threadIdx.x < HFB_NBINS) sh[threadIdx.x] = 0;
  __syncthreads();
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    atomicAdd(&sh[pair_bin(handle_type(shapes, nshapes, h1[i]), handle_type(shapes, nshapes, h2[i]))], 1u);
  __syncthreads();
  if (threadIdx.x < HFB_NBINS && sh[threadIdx.x]) atomicAdd(&hist[threadIdx.x], sh[threadIdx.x]);
}
// offsets[b] = first slot of bin b (offsets[HFB_NBINS] = n); cursor = running write position
__global__ void k_bin_scan(const unsigned* hist, unsigned* offsets, unsigned* cursor) {
  if (threadIdx.x == 0) {
    unsigned acc = 0;
    for (int b = 0; b < HFB_NBINS; ++b) {
      offsets[b] = acc;
      cursor[b] = acc;
      acc += hist[b];
    }
    offsets[HFB_NBINS] = acc;
  }
}
// A block takes a window of HFB_SCATTER_ITEMS * 256 consecutive pairs: ranks inside the block by shared-memory
// atomics, ONE global reservation per class and block, then the writes.  (The first form reserved per warp and class
// through __match_any_sync + a global atomic: 300 k atomics on 49 addresses per 1 M pairs.)  A class's slice of the list is now made of runs of pairs from the same window, which also keeps the
// gathers of the kernels that follow close together.
#define HFB_SCATTER_ITEMS 8
__global__ void __launch_bounds__(256) k_bin_scatter(const hfb_shape* shapes, uint32_t nshapes, const uint32_t* h1,
                                                     const uint32_t* h2, unsigned n, unsigned* cursor, uint32_t* perm) {
  __shared__ unsigned cnt[HFB_NBINS], base[HFB_NBINS];
  if (threadIdx.x < HFB_NBINS) cnt[threadIdx.x] = 0;
  __syncthreads();
  const unsigned w0 = blockIdx.x * (256u * HFB_SCATTER_ITEMS);
  unsigned char key[HFB_SCATTER_ITEMS];
  unsigned short rank[HFB_SCATTER_ITEMS];
#pragma unroll
  for (int j = 0; j < HFB_SCATTER_ITEMS; ++j) {
    const unsigned i = w0 + (unsigned)j * 256u + threadIdx.x;
    key[j] = 0xff;
    rank[j] = 0;
    if (i < n) {
      key[j] = (unsigned char)pair_bin(handle_type(shapes, nshapes, h1[i]), handle_type(shapes, nshapes, h2[i]));
      rank[j] = (unsigned short)atomicAdd(&cnt[key[j]], 1u);
    }
  }
  __syncthreads();
  if (threadIdx.x < HFB_NBINS && cnt[threadIdx.x]) base[threadIdx.x] = atomicAdd(&cursor[threadIdx.x], cnt[threadIdx.x]);
  __syncthreads();
#pragma unroll
  for (int j = 0; j < HFB_SCATTER_ITEMS; ++j) {
    const unsigned i = w0 + (unsigned)j * 256u + threadIdx.x;
    if (i < n) perm[base[key[j]] + rank[j]] = i;
  }
}


// ------------------------------------------------------------ object-table batches ---
// hfb_batch_*_objects: a scene is a table of objects (geometry handle + pose) and a list of index pairs, the
// batched form of collide(const CollisionObject*, const CollisionObject*, ...) (collision.h:58-61).  The pairs are
// expanded on the device into the (h1, tf1, h2, tf2) rows every kernel reads, so the host sends 8 B per pair and
// 100 B per object instead of 200 B per pair.  An index past the table becomes handle 0xffffffff: the pair comes
// back as HFB_PATH_UNSUPPORTED (see load_shape).
__global__ void __launch_bounds__(256) k_expand_pairs(const uint32_t* obj_h, const hfb_transform* obj_tf, unsigned n_obj,
                                                      const uint32_t* pi, const uint32_t* pj, unsigned n, uint32_t* h1,
                                                      hfb_transform* tf1, uint32_t* h2, hfb_transform* tf2) {
  // 12 lanes move one 96-byte pose as 8-byte words: 2 poses per pair
  const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
  for (unsigned i = t; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t a = pi[i], b = pj[i];
    h1[i] = a < n_obj ? obj_h[a] : 0xffffffffu;
    h2[i] = b < n_obj ? obj_h[b] : 0xffffffffu;
  }
  const size_t words = (size_t)n * 24;  // doubles of tf1 and tf2 together
  for (size_t w = t; w < words; w += (size_t)gridDim.x * blockDim.x) {
    const unsigned i = (unsigned)(w / 24), k = (unsigned)(w % 24);
    const uint32_t o = k < 12 ? pi[i] : pj[i];
    const double v = o < n_obj ? reinterpret_cast<const double*>(obj_tf + o)[k % 12] : 0.0;
    (k < 12 ? reinterpret_cast<double*>(tf1 + i) : reinterpret_cast<double*>(tf2 + i))[k % 12] = v;
  }
}
// host pipeline (host_batch_pipelined): the records of the EPA pairs of a batch, compacted with their pair ids -- the
// chunks' rows went to the host before EPA ran
template <class OutT>
__global__ void __launch_bounds__(256) k_gather_epa_rows(const EpaItem* queue, const unsigned* count, const OutT* out,
                                                         uint32_t* ids, OutT* rows) {
  const unsigned n = *count;
  for (unsigned k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const unsigned i = queue[k].pair;
    ids[k] = i;
    rows[k] = out[i];
  }
}
// compact result modes: the distance alone (DistanceResult::min_distance) ...
__global__ void __launch_bounds__(256) k_pick_min_distance(const hfb_distance_result* r, unsigned n, double* d) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) d[i] = r[i].min_distance;
}
// ... and collide() as a bit per pair (isCollision()) plus the records of the colliding pairs only, appended in no
// particular order together with their pair ids
__global__ void __launch_bounds__(256) k_compact_contacts(const hfb_contact* r, unsigned n, unsigned base, uint32_t* flags,
                                                          unsigned* count, uint32_t* ids, hfb_contact* recs, unsigned cap) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool hit = i < n && r[i].num_contacts > 0;
  const unsigned m = __ballot_sync(0xffffffffu, hit);
  const unsigned lane = threadIdx.x & 31u;
  if (lane == 0 && i < n) flags[i >> 5] = m;  // (chunks are multiples of 32 pairs)
  if (!m) return;
  unsigned pos = 0;
  if (lane == 0) pos = atomicAdd(count, (unsigned)__popc(m));
  pos = __shfl_sync(0xffffffffu, pos, 0) + (unsigned)__popc(m & ((1u << lane) - 1u));
  if (hit && pos < cap) {
    ids[pos] = base + i;
    recs[pos] = r[i];
  }
}

// ----------------------------------------------------- convex support kernel --
// One warp per query: streams the SoA vertex block (coalesced 256-B rows) and
// reduces with shuffles.  Algorithmic traffic per query: 24*nv + 24 + 28 bytes.
__global__ void __launch_bounds__(256) k_convex_support(const ConvexDesc* cvx, const double* pool,
                                                        const uint32_t* ids, const double* dirs,
                                                        int32_t* idx_out, double* sup_out, unsigned n) {
  const unsigned warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const unsigned nwarps = (gridDim.x * blockDim.x) >> 5;
  const unsigned lane = threadIdx.x & 31u;
  for (unsigned q = warp; q < n; q += nwarps) {
    const ConvexDesc d = cvx[ids[q]];
    const double* x = pool + d.off;
    const double* y = x + d.vpad;
    const double* z = y + d.vpad;
    const double dx = dirs[3 * q], dy = dirs[3 * q + 1], dz = dirs[3 * q + 2];
    // same NaN rules as shape_support (hfb_shapes.cuh): the answer is the serial scan's for any direction
    double best = -(double)INFINITY;
    int bi = 0x7fffffff;
    bool first = true;
    for (unsigned i = lane; i < d.nv; i += 32) {
      const double v = (x[i] * dx + y[i] * dy) + z[i] * dz;
      if (first) {
        if (v == v) {
          best = v;
          bi = (int)i;
          first = false;
        } else if (i == 0) {
          best = (double)INFINITY;
          bi = -1;
          first = false;
        }
      } else if (v > best) {
        best = v;
        bi = (int)i;
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, best, off);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
      if (ov > best || (ov == best && oi < bi)) {
        best = ov;
        bi = oi;
      }
    }
    if (bi < 0) bi = 0;
    if (lane == 0) {
      idx_out[q] = bi;
      sup_out[3 * q] = x[bi];
      sup_out[3 * q + 1] = y[bi];
      sup_out[3 * q + 2] = z[bi];
    }
  }
}

// ===================================================================== host ===
namespace {

constexpr size_t kChunk = 1u << 17;  // pairs per pipelined chunk of the host entry points

template <int G, int CAPS, int MODE, int PATHS, int MINB = 1, bool STAGE = false>
int launch_pairs(hfb_ctx* ctx, const BatchArgs& a, unsigned work, cudaStream_t s) {
  if (work == 0) return HFB_OK;
  const int threads = 128;
  const unsigned groups_per_block = threads / G;
  unsigned blocks = (work + groups_per_block - 1) / groups_per_block;
  const unsigned cap = (unsigned)ctx->num_sms * 32u;  // grid-stride beyond this
  if (blocks > cap) blocks = cap;
  const size_t smem = (STAGE && (G > 1) && (CAPS & CAP_CONVEX)) ? (size_t)groups_per_block * sizeof(StageGroup) : 0;
  if (smem > 48 * 1024) {
    const void* fn = reinterpret_cast<const void*>(&k_pairs<G, CAPS, MODE, PATHS, MINB, STAGE>);
    if (!ctx->func_cfg.count(fn)) {
      CK(cudaFuncSetAttribute(k_pairs<G, CAPS, MODE, PATHS, MINB, STAGE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      ctx->func_cfg[fn] = 1;
    }
  }
  {
    KTimer kt(ctx, s, (CAPS & CAP_CONVEX) ? 4 : (PATHS == PATH_CLOSED ? 3 : 0));
    k_pairs<G, CAPS, MODE, PATHS, MINB, STAGE><<<blocks, threads, smem, s>>>(a);
  }
  ctx->stats.kernel_launches++;
  CK(cudaGetLastError());
  return HFB_OK;
}

template <int G, int CAPS, int MODE, int TIER>
int launch_epa(hfb_ctx* ctx, const BatchArgs& a, cudaStream_t s) {
  const int threads = EpaCfg<G, TIER>::THREADS;
  const size_t smem = EpaCfg<G, TIER>::GPB * sizeof(typename EpaCfg<G, TIER>::WS);
  const void* fn = reinterpret_cast<const void*>(&k_epa<G, CAPS, MODE, TIER>);
  int per_sm = 0;
  auto it = ctx->func_cfg.find(fn);
  if (it == ctx->func_cfg.end()) {
    CK(cudaFuncSetAttribute(k_epa<G, CAPS, MODE, TIER>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_epa<G, CAPS, MODE, TIER>, threads, smem));
    if (per_sm < 1) per_sm = 1;
    ctx->func_cfg[fn] = per_sm;
  } else {
    per_sm = it->second;
  }
  int blocks = ctx->num_sms * per_sm;
  // tier 0: one support-point slot per resident group (the kernel is grid-persistent: fewer blocks only run longer)
  if (TIER == 0 && (unsigned)(blocks * EpaCfg<G, TIER>::GPB) > a.epa_sup_groups)
    blocks = (int)(a.epa_sup_groups / EpaCfg<G, TIER>::GPB);
  if (blocks < 1) return fail(ctx, HFB_ERR_CUDA, "EPA support-point store missing");
  {
    KTimer kt(ctx, s, 1);
    k_epa<G, CAPS, MODE, TIER><<<blocks, threads, smem, s>>>(a);
  }
  ctx->stats.kernel_launches++;
  CK(cudaGetLastError());
  return HFB_OK;
}

template <int CAPS, int MODE, int TIER>
int launch_epa_g(hfb_ctx* ctx, const BatchArgs& a, cudaStream_t s) {
  // tier 1 runs the few pairs that outgrew tier 0 on an almost idle GPU: its time is the serial chain of the longest of
  // them, which wide groups shorten (the closest-face scan and the new faces' geometry are spread over the lanes)
  if constexpr (TIER == 1) {
    return launch_epa<HFB_GE_TIER1, CAPS, MODE, 1>(ctx, a, s);
  } else {
    switch (ctx->ge) {
      case 4: return launch_epa<4, CAPS, MODE, 0>(ctx, a, s);
      case 8: return launch_epa<8, CAPS, MODE, 0>(ctx, a, s);
      case 16: return launch_epa<16, CAPS, MODE, 0>(ctx, a, s);
      default: return launch_epa<32, CAPS, MODE, 0>(ctx, a, s);
    }
  }
}
template <int MODE>
int launch_pairs_convex(hfb_ctx* ctx, const BatchArgs& a, unsigned work, cudaStream_t s) {
  switch (ctx->gc) {
    case 1: return launch_pairs<1, CAPS_ALLP, MODE, PATH_BOTH>(ctx, a, work, s);
    case 2: return launch_pairs<2, CAPS_ALLP, MODE, PATH_BOTH>(ctx, a, work, s);
    case 4:
      if (a.stage) return launch_pairs<4, CAPS_ALLP, MODE, PATH_BOTH, 1, true>(ctx, a, work, s);
      return launch_pairs<4, CAPS_ALLP, MODE, PATH_BOTH>(ctx, a, work, s);
    case 8:
      if (a.stage) return launch_pairs<8, CAPS_ALLP, MODE, PATH_BOTH, 1, true>(ctx, a, work, s);
      return launch_pairs<8, CAPS_ALLP, MODE, PATH_BOTH>(ctx, a, work, s);
    case 16: return launch_pairs<16, CAPS_ALLP, MODE, PATH_BOTH>(ctx, a, work, s);
    default: return launch_pairs<32, CAPS_ALLP, MODE, PATH_BOTH>(ctx, a, work, s);
  }
}

// the support-point store of k_epa's first tier (one slot per resident lane group) into `a`
cudaError_t reserve_epa_sup(hfb_ctx* ctx, Slot& sl, BatchArgs& a) {
  const size_t groups = (size_t)ctx->num_sms * HFB_EPA_SUP_GROUPS_PER_SM;
  const cudaError_t e = sl.sup.reserve(groups * 6 * EpaPolySmall::MAXV * sizeof(double));
  a.epa_sup = static_cast<double*>(sl.sup.p);
  a.epa_sup_groups = e == cudaSuccess ? (unsigned)groups : 0u;
  return e;
}

// runs one (sub)batch whose inputs/outputs are already device-resident:
//   counting sort of the pairs by class -> closed-form kernel, GJK kernel (thread per pair),
//   convex/triangle kernel (lane group per pair) -> EPA kernel over the queue
template <int MODE>
int run_device_batch(hfb_ctx* ctx, Slot& sl, BatchArgs a, cudaStream_t s, int epa_mode = 0) {
  // epa_mode 0: the whole batch; 1 / 2: phase 1 only (first / a later chunk of a host batch), the EPA items stay in the
  // queue for run_deferred_epa
  const unsigned n = a.n;
  if (n == 0) return HFB_OK;
  CK(sl.queue.reserve((size_t)n * sizeof(EpaItem)));
  // counters: [0] EPA queue count, [1] running EPA total, [2] retry count, [3] tier-1 work counter, [4..4+kMaxParts] queue marks (mark[0] = 0,
  // mark[j+1] = queue count after part j of phase 1), [16..16+kMaxParts) EPA work counters, [24], [25] k_bvh work counters,
  // [32..) hist (NBINS), offsets (NBINS+1), cursor (NBINS)
  const size_t ncnt = 32 + 3 * (HFB_NBINS + 2);
  if (!sl.counters.p) {
    CK(sl.counters.reserve(ncnt * sizeof(unsigned)));
    CK(cudaMemsetAsync(sl.counters.p, 0, ncnt * sizeof(unsigned), s));
  }
  if (!sl.epa_stream) {
    CK(cudaStreamCreateWithFlags(&sl.epa_stream, cudaStreamNonBlocking));
    for (int k = 0; k < kMaxParts; ++k) CK(cudaEventCreateWithFlags(&sl.ev_part[k], cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&sl.ev_join, cudaEventDisableTiming));
    int least = 0, greatest = 0;
    CK(cudaDeviceGetStreamPriorityRange(&least, &greatest));
    CK(cudaStreamCreateWithPriority(&sl.work_stream, cudaStreamNonBlocking, greatest));
    CK(cudaEventCreateWithFlags(&sl.ev_fork, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&sl.ev_work, cudaEventDisableTiming));
  }
  CK(sl.lists.reserve((size_t)n * sizeof(uint32_t)));
  CK(sl.retry.reserve((size_t)n * sizeof(uint32_t)));
  a.queue = static_cast<EpaItem*>(sl.queue.p);
  a.retry = static_cast<uint32_t*>(sl.retry.p);
  a.cont = nullptr;
  a.cont_cap = 0;
  if (ctx->epa_resume > 0) {  // HFB_EPA_RESUME: continuation records for that many retries per batch (0: retries start over)
    const size_t cap = (size_t)ctx->epa_resume < (size_t)n ? (size_t)ctx->epa_resume : (size_t)n;
    CK(sl.cont.reserve(cap * sizeof(EpaCont)));
    a.cont = static_cast<EpaCont*>(sl.cont.p);
    a.cont_cap = (unsigned)cap;
  }
  if (a.P.compute_penetration) CK(reserve_epa_sup(ctx, sl, a));
  unsigned* cnt = static_cast<unsigned*>(sl.counters.p);
  unsigned* mark = cnt + 4;
  unsigned* heads = cnt + 16;
  unsigned* hist = cnt + 32;
  unsigned* offsets = hist + HFB_NBINS + 1;
  unsigned* cursor = offsets + HFB_NBINS + 2;
  uint32_t* perm = static_cast<uint32_t*>(sl.lists.p);
  a.queue_count = cnt;
  a.retry_count = cnt + 2;
  a.epa_lo = a.epa_hi = nullptr;
  a.epa_head = nullptr;
  a.sub_idx = 0;
  a.sub_cnt = 1;
  a.stage = (unsigned)(ctx->stage != 0);
  a.gjk_work = nullptr;
  a.iter_quorum = 0;
  a.A = ctx->dview;
  if (epa_mode != 2) CK(cudaMemsetAsync(cnt, 0, sizeof(unsigned), s));  // (a later chunk appends to the queue)
  CK(cudaMemsetAsync(cnt + 2, 0, 30 * sizeof(unsigned), s));
  CK(cudaMemsetAsync(hist, 0, HFB_NBINS * sizeof(unsigned), s));
  {
    KTimer kt(ctx, s, 2);
    unsigned hb = (n + 255) / 256;
    if (hb > (unsigned)ctx->num_sms * 8u) hb = (unsigned)ctx->num_sms * 8u;
    k_bin_hist<<<hb, 256, 0, s>>>(ctx->dview.shapes, ctx->dview.nshapes, a.h1, a.h2, n, hist);
    k_bin_scan<<<1, 32, 0, s>>>(hist, offsets, cursor);
    k_bin_scatter<<<(n + 256 * HFB_SCATTER_ITEMS - 1) / (256 * HFB_SCATTER_ITEMS), 256, 0, s>>>(ctx->dview.shapes, ctx->dview.nshapes, a.h1, a.h2, n, cursor, perm);
  }
  ctx->stats.kernel_launches += 3;
  CK(cudaGetLastError());
  a.index_list = perm;
  int rc;
  const bool mixed = ctx->arena.has_convex || ctx->arena.has_tri;
  if (mixed && ctx->hull_sort) {  // HFB_HULL_SORT: the hull / triangle class ordered by the handle of its first operand
    CK(sl.hsort.reserve(hull_sort_bytes(n)));
    const uint32_t* sorted = nullptr;
    int nl = 0;
    {
      KTimer kt(ctx, s, 2);
      if (hull_sort_launch(a.h1, n, perm, offsets, HFB_BIN_CONVEX, sl.hsort.p, &sorted, s, &nl) != 0)
        return fail(ctx, HFB_ERR_CUDA, "hull sort launch failed");
    }
    ctx->stats.kernel_launches += (uint64_t)nl;
    a.index_list = sorted;
  }
  const bool want_epa = a.P.compute_penetration;
  // fork: GJK, the hull / triangle kernel and EPA on the work stream; the closed forms (nothing reads their rows) and
  // the mesh walks stay on the caller's stream, which waits for the work stream before the batch returns
  cudaStream_t ws = sl.work_stream;
  CK(cudaEventRecord(sl.ev_fork, s));
  CK(cudaStreamWaitEvent(ws, sl.ev_fork, 0));

  // EPA over the queue items pushed since the previous mark.  Parts other than the last go to the
  // side stream, where they overlap phase 1 of the parts that follow; an EPA item is long and there
  // are few of them, so run at the end they would leave most of the GPU idle.
  int parts_done = 0;
  auto epa_after_part = [&](bool last) -> int {
    if (!want_epa || epa_mode) return HFB_OK;
    const int j = parts_done++;
    if (cudaMemcpyAsync(mark + j + 1, cnt, sizeof(unsigned), cudaMemcpyDeviceToDevice, ws) != cudaSuccess)
      return fail(ctx, HFB_ERR_CUDA, "queue mark copy failed");
    BatchArgs ae = a;
    ae.epa_lo = mark + j;
    ae.epa_hi = mark + j + 1;
    ae.epa_head = heads + j;
    cudaStream_t es = ws;
    if (!last) {
      es = sl.epa_stream;
      if (cudaEventRecord(sl.ev_part[j], ws) != cudaSuccess || cudaStreamWaitEvent(es, sl.ev_part[j], 0) != cudaSuccess)
        return fail(ctx, HFB_ERR_CUDA, "event record/wait failed");
    } else if (j > 0) {
      // the side stream's launches finish before the caller's stream moves past this batch
      if (cudaEventRecord(sl.ev_join, sl.epa_stream) != cudaSuccess || cudaStreamWaitEvent(ws, sl.ev_join, 0) != cudaSuccess)
        return fail(ctx, HFB_ERR_CUDA, "event record/wait failed");
    }
    int r = mixed ? launch_epa_g<CAPS_ALL, MODE, 0>(ctx, ae, es) : launch_epa_g<CAP_PRIM, MODE, 0>(ctx, ae, es);
    if (r || !last) return r;
    // tier 1 over the retry list, after every tier-0 launch of this batch
    ae.epa_head = cnt + 3;
    return mixed ? launch_epa_g<CAPS_ALL, MODE, 1>(ctx, ae, ws) : launch_epa_g<CAP_PRIM, MODE, 1>(ctx, ae, ws);
  };

  BatchArgs ac = a, ag = a, av = a;
  ac.range_lo = offsets + 0;
  ac.range_hi = offsets + HFB_BIN_GJK0;
  ag.range_lo = offsets + HFB_BIN_GJK0;
  ag.range_hi = offsets + HFB_BIN_CONVEX;
  av.range_lo = offsets + HFB_BIN_CONVEX;
  av.range_hi = offsets + HFB_BIN_BVH;
  if ((rc = launch_pairs<1, CAP_PRIM | CAP_PLANE, MODE, PATH_CLOSED>(ctx, ac, n, s))) return rc;
  // the class populations are only known on the device, so both GJK ranges are cut the same way
  // cutting phase 1 costs more in kernel tails than the overlap returns, so one part is the default; HFB_NSUB asks
  // for more
  unsigned nsub = ctx->nsub > 0 ? (unsigned)ctx->nsub : 1u;
  if (!want_epa) nsub = 1;
  if (nsub > (unsigned)(kMaxParts / 2)) nsub = kMaxParts / 2;
  const unsigned sub_work = (n + nsub - 1) / nsub;
  for (unsigned j = 0; j < nsub; ++j) {
    ag.sub_idx = j;
    ag.sub_cnt = nsub;
    switch (ctx->minb) {  // register budget of the GJK kernel: 255 / 168 / 128 registers per thread
      case 3: rc = launch_pairs<1, CAP_PRIM, MODE, PATH_GJKROUTE, 3>(ctx, ag, sub_work, ws); break;
      case 4: rc = launch_pairs<1, CAP_PRIM, MODE, PATH_GJKROUTE, 4>(ctx, ag, sub_work, ws); break;
      default:
        if (ctx->refill) {
          ag.gjk_work = cnt + 26 + j;
          ag.iter_quorum = (unsigned)ctx->iter_quorum;
          const unsigned blocks = (unsigned)ctx->num_sms * 2u;  // 255 registers: 2 blocks of 128 per SM
          {
            KTimer kt(ctx, ws, 0);
            k_gjk_refill<MODE><<<blocks, 128, 0, ws>>>(ag);
          }
          ctx->stats.kernel_launches++;
          if (cudaGetLastError() != cudaSuccess) return fail(ctx, HFB_ERR_CUDA, "k_gjk_refill launch failed");
          rc = HFB_OK;
        } else if (ctx->gjk_npass > 0 && nsub == 1) {
          CK(sl.gstate.reserve(gjk_pass_state_bytes(n)));
          CK(sl.glist.reserve(2 * (size_t)n * sizeof(uint32_t)));
          CK(sl.gcnt.reserve(8 * sizeof(unsigned)));
          int nl = 0;
          uint32_t* la = static_cast<uint32_t*>(sl.glist.p);
          const bool early_epa = ctx->gjk_npass > 1 && ctx->epa_overlap && want_epa;
          {
            KTimer kt(ctx, ws, 0);
            if (gjk_passes_first(ag, MODE, n, sl.gstate.p, la, static_cast<unsigned*>(sl.gcnt.p), ctx->gjk_steps, ctx->gjk_npass,
                                 ctx->num_sms, ws, &nl) != 0)
              return fail(ctx, HFB_ERR_CUDA, "GJK pass launch failed");
          }
          // EPA of the pairs the first pass finished starts on the side stream, next to the remaining passes (which
          // only keep a fraction of the GPU busy)
          if (early_epa && (rc = epa_after_part(false))) return rc;
          {
            KTimer kt(ctx, ws, 0);
            if (gjk_passes_rest(ag, MODE, n, sl.gstate.p, la, la + n, static_cast<unsigned*>(sl.gcnt.p), ctx->gjk_steps,
                                ctx->gjk_npass, ctx->num_sms, ws, &nl) != 0)
              return fail(ctx, HFB_ERR_CUDA, "GJK pass launch failed");
          }
          ctx->stats.kernel_launches += (uint64_t)nl;
          rc = HFB_OK;
        } else {
          rc = launch_pairs<1, CAP_PRIM, MODE, PATH_GJKROUTE, 1>(ctx, ag, sub_work, ws);
        }
    }
    if (rc) return rc;
    if ((rc = epa_after_part(!mixed && j + 1 == nsub))) return rc;
  }
  if (mixed) {
    for (unsigned j = 0; j < nsub; ++j) {
      av.sub_idx = j;
      av.sub_cnt = nsub;
      if ((rc = launch_pairs_convex<MODE>(ctx, av, sub_work, ws))) return rc;
      if ((rc = epa_after_part(j + 1 == nsub))) return rc;
    }
  }
  if (ctx->arena.has_bvh) {
    const int threads = 64;
    unsigned blocks = (n + threads - 1) / threads;
    const unsigned cap = (unsigned)ctx->num_sms * (unsigned)ctx->bvh_bps;
    if (blocks > cap) blocks = cap;
    CK(sl.bvh_ws.reserve((size_t)ctx->num_sms * 4u * 2 * threads * sizeof(EpaWs)));
    if (!sl.bvh_cnt.p) {
      CK(sl.bvh_cnt.reserve(8 * sizeof(unsigned long long)));
      CK(cudaMemsetAsync(sl.bvh_cnt.p, 0, 8 * sizeof(unsigned long long), s));
    }
    BatchArgs ab = a;
    ab.bvh_ws = static_cast<EpaWs*>(sl.bvh_ws.p);
    ab.bvh_counters = static_cast<unsigned long long*>(sl.bvh_cnt.p);
    ab.range_lo = offsets + HFB_BIN_BVH;
    ab.range_hi = offsets + HFB_BIN_BVH2;
    ab.bvh_work = cnt + 24;
    if (ctx->bvh_order) {
      CK(sl.okeys.reserve((size_t)n));
      CK(sl.ohist.reserve(2 * (HFB_ORDER_SAMPLES + 1) * sizeof(unsigned)));
      CK(sl.olist.reserve((size_t)n * sizeof(uint32_t)));
      unsigned* ohist = static_cast<unsigned*>(sl.ohist.p);
      unsigned* ocur = ohist + HFB_ORDER_SAMPLES + 1;
      CK(cudaMemsetAsync(ohist, 0, 2 * (HFB_ORDER_SAMPLES + 1) * sizeof(unsigned), s));
      const unsigned ob = (n + 127) / 128 < (unsigned)ctx->num_sms * 8u ? (n + 127) / 128 : (unsigned)ctx->num_sms * 8u;
      KTimer kt(ctx, s, 2);
      k_bvh_order_keys<<<ob, 128, 0, s>>>(ab, ab.range_lo, ab.range_hi, static_cast<unsigned char*>(sl.okeys.p), ohist);
      k_bvh_order_scan<<<1, 32, 0, s>>>(ohist, ocur);
      k_bvh_order_scatter<<<ob, 128, 0, s>>>(ab.index_list, ab.range_lo, ab.range_hi,
                                             static_cast<const unsigned char*>(sl.okeys.p), ocur,
                                             static_cast<uint32_t*>(sl.olist.p));
      ctx->stats.kernel_launches += 3;
      CK(cudaGetLastError());
      ab.index_list = static_cast<const uint32_t*>(sl.olist.p);  // only its [lo, hi) slice is written -- and read
    }
    bool walked = false;
    if constexpr (MODE == 0) {
      if (ctx->bvhq) {  // distance(): the task-system walk
        const unsigned qb = bvhq_blocks(ctx->num_sms, n);
        const int cap = ctx->arena.max_bvh_depth + 3;
        const BvhqSizes z = bvhq_sizes(qb, n, cap);
        CK(sl.qprep.reserve(z.prep));
        CK(sl.qstacks.reserve(z.stacks));
        CK(sl.qtl.reserve(z.treelets));
        CK(sl.qws.reserve(z.ws));
        CK(sl.qsv.reserve(z.saves));
        BvhqLaunch L{};
        L.A = ab.A;
        L.h1 = ab.h1; L.tf1 = ab.tf1; L.h2 = ab.h2; L.tf2 = ab.tf2;
        L.guess_in = ab.guess_in; L.hint_in = ab.hint_in;
        L.out = static_cast<hfb_distance_result*>(ab.out);
        L.index_list = ab.index_list;
        L.range_lo = ab.range_lo; L.range_hi = ab.range_hi;
        L.P = ab.P; L.B = ab.B;
        L.prep = static_cast<QPrep*>(sl.qprep.p);
        L.stacks = static_cast<QStackEnt*>(sl.qstacks.p);
        L.treelets = static_cast<QTreelet*>(sl.qtl.p);
        L.ws = static_cast<EpaWs*>(sl.qws.p);
        L.saves = static_cast<QLeafSave*>(sl.qsv.p);
        L.gjk_chunk = ctx->bvh_chunk;
        L.work = ab.bvh_work;
        L.counters = ab.bvh_counters;
        L.stack_cap = cap;
        L.spec_after = ctx->bvh_spec;
        L.spec_big_after = ctx->bvh_spec < 0 ? 0x7fffffff : ctx->bvh_spec + ctx->bvh_spec_big;
        L.bv_gens = ctx->bvh_gens;
        L.warps = ctx->bvh_warps;
        {
          KTimer kt(ctx, s, 5);
          if (bvhq_launch(L, qb, n, s) != 0) return fail(ctx, HFB_ERR_CUDA, "k_bvhq launch failed");
        }
        ctx->stats.kernel_launches += 2;
        walked = true;
      }
    }
    if (!walked) {
      {
        KTimer kt(ctx, s, 5);
        if (ctx->bvh_minb >= 8) k_bvh<MODE, BVK_SHAPE, 8><<<blocks * 2, threads, 0, s>>>(ab);
        else if (ctx->bvh_quorum == 1) k_bvh<MODE, BVK_SHAPE, 4, 1><<<blocks, threads, 0, s>>>(ab);  // HFB_BVH_QUORUM=1
        else k_bvh<MODE, BVK_SHAPE, 4><<<blocks, threads, 0, s>>>(ab);
      }
      ctx->stats.kernel_launches++;
      CK(cudaGetLastError());
    }
    {  // (mesh, mesh) pairs, own instantiation: an empty range costs one launch
      ab.index_list = a.index_list;  // (the reordered list holds the (mesh, shape) slice only)
      ab.range_lo = offsets + HFB_BIN_BVH2;
      ab.range_hi = offsets + HFB_NBINS;
      ab.bvh_work = cnt + 25;
      {
        KTimer kt(ctx, s, 5);
        k_bvh<MODE, BVK_MESH, 4><<<blocks, threads, 0, s>>>(ab);
      }
      ctx->stats.kernel_launches++;
      CK(cudaGetLastError());
    }
  }
  CK(cudaEventRecord(sl.ev_work, ws));
  CK(cudaStreamWaitEvent(s, sl.ev_work, 0));
  ctx->stats.pairs_processed += n;
  return HFB_OK;
}

// EPA over everything the chunks of a host batch queued (run_device_batch with epa_mode 1 / 2), with the batch's base
// pointers: one tier-0 and one tier-1 launch for the whole batch instead of one EPA tail per chunk
template <int MODE>
int run_deferred_epa(hfb_ctx* ctx, Slot& sl, BatchArgs a, cudaStream_t s) {
  if (!a.P.compute_penetration) return HFB_OK;
  unsigned* cnt = static_cast<unsigned*>(sl.counters.p);
  unsigned* mark = cnt + 4;
  unsigned* heads = cnt + 16;
  a.queue = static_cast<EpaItem*>(sl.queue.p);
  a.retry = static_cast<uint32_t*>(sl.retry.p);
  a.queue_count = cnt;
  a.retry_count = cnt + 2;
  a.cont = static_cast<EpaCont*>(sl.cont.p);
  a.cont_cap = a.cont ? (unsigned)(((size_t)ctx->epa_resume < (size_t)a.n ? (size_t)ctx->epa_resume : (size_t)a.n)) : 0u;
  if (a.cont && sl.cont.cap < (size_t)a.cont_cap * sizeof(EpaCont)) a.cont_cap = (unsigned)(sl.cont.cap / sizeof(EpaCont));
  CK(reserve_epa_sup(ctx, sl, a));
  a.A = ctx->dview;
  a.index_list = nullptr;
  a.pair_base = 0;
  CK(cudaMemsetAsync(cnt + 2, 0, 30 * sizeof(unsigned), s));  // retry count, tier-1 counter, marks (mark[0] = 0), heads
  CK(cudaMemcpyAsync(mark + 1, cnt, sizeof(unsigned), cudaMemcpyDeviceToDevice, s));
  a.epa_lo = mark;
  a.epa_hi = mark + 1;
  a.epa_head = heads;
  const bool mixed = ctx->arena.has_convex || ctx->arena.has_tri;
  int r = mixed ? launch_epa_g<CAPS_ALL, MODE, 0>(ctx, a, s) : launch_epa_g<CAP_PRIM, MODE, 0>(ctx, a, s);
  if (r) return r;
  a.epa_head = cnt + 3;
  return mixed ? launch_epa_g<CAPS_ALL, MODE, 1>(ctx, a, s) : launch_epa_g<CAP_PRIM, MODE, 1>(ctx, a, s);
}

// what an object-table call adds to a batch: the table on the device, the pair indices on the host
struct ObjSrc {
  size_t n_objects;
  const uint32_t* d_handles;
  const hfb_transform* d_tfs;
  const uint32_t* first;
  const uint32_t* second;
};
// compact result modes of the object-table calls (null pointers: full records into `out`)
struct OutMode {
  double* min_out = nullptr;       // distance(): min_distance only, 8 B per pair
  uint32_t* flags = nullptr;       // collide(): one bit per pair ...
  uint32_t* n_hits = nullptr;      // ... and the records of the colliding pairs (at most `cap`) with their pair ids
  uint32_t* hit_ids = nullptr;
  hfb_contact* hit_recs = nullptr;
  uint32_t cap = 0;
};

// ---- the host pipeline of large batches -----------------------------------------------------------------------------
// The rotating-slot pipeline below (host_batch) runs every chunk to the end, EPA included, before its rows go back:
// with the kernels of round 2 a chunk of 256 Ki pairs is a third sort + GJK and two thirds EPA tail -- the latency of
// its longest pair with the GPU nearly empty -- and four chunks pay four tails.  Here the whole batch lives on the
// device: phase 1 (class sort, closed forms, GJK) runs chunk by chunk as the uploads arrive and each chunk's rows start
// their way back at once; EPA runs ONCE over the items of all chunks (run_deferred_epa); the records of the EPA pairs
// (1.2 % of config 2) follow compacted, and the host puts them in place.  Three streams: uploads, kernels, downloads.
template <int MODE, typename OutT>
int host_batch_pipelined(hfb_ctx* ctx, size_t n, const uint32_t* h1, const hfb_transform* tf1, const uint32_t* h2,
                         const hfb_transform* tf2, const SolverP& P, const CollideP& Cp, const BvhReq& Bq, OutT* out,
                         const ObjSrc* obj, double* min_out) {
  int rc;
  Slot& sl = ctx->slots[0];
  cudaStream_t sC = sl.stream, sU = ctx->slots[1].stream, sD = ctx->slots[2].stream;
  static const bool trace = getenv("HFB_PIPE_TRACE") != nullptr;  // debugging aid: host clock at the milestones of a call
  const auto t0 = std::chrono::steady_clock::now();
  auto stamp = [&](const char* what) {
    if (trace) fprintf(stderr, "[hfb pipe] %-28s %8.3f ms\n", what, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
  };
  // How many chunks: a chunk's phase 1 has a floor whatever its size (the serial iteration chains of the longest pairs
  // in the GJK passes), so chunks are only worth their overlap: about one per 0.6 ms of PCIe time (uploads and
  // downloads share the link), at least 128 Ki pairs each.  1 M pairs: a scene +
  // distances only (16 B per pair) -> 1 chunk; a scene + full rows (104 B) -> 3; pair rows + full rows (296 B) -> 8.
  size_t chunk;
  if (ctx->chunk > 0) {
    chunk = (size_t)ctx->chunk;
  } else {
    const double bytes_per_pair = (obj ? 8.0 : 200.0) + (min_out ? 8.0 : (double)sizeof(OutT));
    const double pcie_ms = (double)n * bytes_per_pair / 57e6;
    size_t want = (size_t)(pcie_ms / 0.6 + 0.5);
    const size_t most = n / kChunk ? n / kChunk : 1;
    if (want < 1) want = 1;
    if (want > most) want = most;
    chunk = (n + want - 1) / want;
  }
  chunk = (chunk + 31) & ~(size_t)31;
  const size_t nchunks = (n + chunk - 1) / chunk;
  while (ctx->pipe_events.size() < 2 * nchunks + 2) {
    cudaEvent_t e;
    CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    ctx->pipe_events.push_back(e);
  }
  CK(ctx->big_h1.reserve(n * 4));
  CK(ctx->big_h2.reserve(n * 4));
  CK(ctx->big_tf1.reserve(n * sizeof(hfb_transform)));
  CK(ctx->big_tf2.reserve(n * sizeof(hfb_transform)));
  CK(ctx->big_out.reserve(n * sizeof(OutT)));
  if (obj) {
    CK(ctx->big_pi.reserve(n * 4));
    CK(ctx->big_pj.reserve(n * 4));
  }
  if (min_out) CK(ctx->big_min.reserve(n * 8));
  // the queue and the retry list take the EPA items of every chunk (run_device_batch asks for a chunk's worth: no
  // reallocation once they hold the batch's)
  CK(sl.queue.reserve(n * sizeof(EpaItem)));
  CK(sl.retry.reserve(n * sizeof(uint32_t)));
  uint32_t* d_h1 = static_cast<uint32_t*>(ctx->big_h1.p);
  uint32_t* d_h2 = static_cast<uint32_t*>(ctx->big_h2.p);
  hfb_transform* d_tf1 = static_cast<hfb_transform*>(ctx->big_tf1.p);
  hfb_transform* d_tf2 = static_cast<hfb_transform*>(ctx->big_tf2.p);
  OutT* d_out = static_cast<OutT*>(ctx->big_out.p);
  auto drain = [&]() {
    for (int k = 0; k < kSlots; ++k) cudaStreamSynchronize(ctx->slots[k].stream);
  };
  if (obj) {  // the object table was uploaded on slot 0's stream = sC: in order with the expansion kernels
  }
  size_t done = 0;
  for (size_t c = 0; c < nchunks; ++c) {
    const size_t m = (n - done < chunk) ? (n - done) : chunk;
    cudaEvent_t ev_up = ctx->pipe_events[2 * c], ev_ph = ctx->pipe_events[2 * c + 1];
    if (obj) {
      CK(cudaMemcpyAsync(static_cast<uint32_t*>(ctx->big_pi.p) + done, obj->first + done, m * 4, cudaMemcpyHostToDevice, sU));
      CK(cudaMemcpyAsync(static_cast<uint32_t*>(ctx->big_pj.p) + done, obj->second + done, m * 4, cudaMemcpyHostToDevice, sU));
    } else {
      CK(cudaMemcpyAsync(d_h1 + done, h1 + done, m * 4, cudaMemcpyHostToDevice, sU));
      CK(cudaMemcpyAsync(d_h2 + done, h2 + done, m * 4, cudaMemcpyHostToDevice, sU));
      CK(cudaMemcpyAsync(d_tf1 + done, tf1 + done, m * sizeof(hfb_transform), cudaMemcpyHostToDevice, sU));
      CK(cudaMemcpyAsync(d_tf2 + done, tf2 + done, m * sizeof(hfb_transform), cudaMemcpyHostToDevice, sU));
    }
    CK(cudaEventRecord(ev_up, sU));
    CK(cudaStreamWaitEvent(sC, ev_up, 0));
    if (obj) {
      unsigned eb = (unsigned)((m * 24 + 255) / 256);
      if (eb > (unsigned)ctx->num_sms * 16u) eb = (unsigned)ctx->num_sms * 16u;
      k_expand_pairs<<<eb, 256, 0, sC>>>(obj->d_handles, obj->d_tfs, (unsigned)obj->n_objects,
                                         static_cast<const uint32_t*>(ctx->big_pi.p) + done,
                                         static_cast<const uint32_t*>(ctx->big_pj.p) + done, (unsigned)m, d_h1 + done, d_tf1 + done,
                                         d_h2 + done, d_tf2 + done);
      ctx->stats.kernel_launches++;
      CK(cudaGetLastError());
    }
    BatchArgs a{};
    a.n = (unsigned)m;
    a.h1 = d_h1 + done;
    a.h2 = d_h2 + done;
    a.tf1 = d_tf1 + done;
    a.tf2 = d_tf2 + done;
    a.out = d_out + done;
    a.P = P;
    a.C = Cp;
    a.B = Bq;
    a.pair_base = (unsigned)done;
    if ((rc = run_device_batch<MODE>(ctx, sl, a, sC, c == 0 ? 1 : 2))) {
      drain();
      return rc;
    }
    if constexpr (MODE == 0) {
      if (min_out) {
        k_pick_min_distance<<<(unsigned)((m + 255) / 256), 256, 0, sC>>>(d_out + done, (unsigned)m,
                                                                          static_cast<double*>(ctx->big_min.p) + done);
        ctx->stats.kernel_launches++;
      }
    }
    CK(cudaEventRecord(ev_ph, sC));
    CK(cudaStreamWaitEvent(sD, ev_ph, 0));
    if (min_out) CK(cudaMemcpyAsync(min_out + done, static_cast<double*>(ctx->big_min.p) + done, m * 8, cudaMemcpyDeviceToHost, sD));
    else CK(cudaMemcpyAsync(out + done, d_out + done, m * sizeof(OutT), cudaMemcpyDeviceToHost, sD));
    // the chunk's handles / object indices are validated AFTER its work is enqueued, while the GPU is busy with it (8 MB
    // of host reads per 1 M pairs, in front of a single-chunk call otherwise).  The device side is safe against
    // a bad value (k_expand_pairs, handle_type, load_shape: such a pair comes back unsupported); the call fails.
    if (obj) {
      const uint32_t no = (uint32_t)(obj->n_objects > 0xffffffffull ? 0xffffffffull : obj->n_objects);
      uint32_t bad = 0;
      for (size_t i = done; i < done + m; ++i) bad |= (uint32_t)(obj->first[i] >= no) | (uint32_t)(obj->second[i] >= no);
      if (bad) {
        drain();
        return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "object index out of range");
      }
    } else if ((rc = check_handles(ctx, h1 + done, m)) || (rc = check_handles(ctx, h2 + done, m))) {
      drain();
      return rc;
    }
    done += m;
  }
  stamp("chunks enqueued");
  if (trace) {
    cudaStreamSynchronize(sC);
    stamp("phase 1 of all chunks done");
  }
  // EPA of the whole batch, then the records it produced, compacted
  BatchArgs ag{};
  ag.n = (unsigned)n;
  ag.h1 = d_h1;
  ag.h2 = d_h2;
  ag.tf1 = d_tf1;
  ag.tf2 = d_tf2;
  ag.out = d_out;
  ag.P = P;
  ag.C = Cp;
  ag.B = Bq;
  unsigned epa_pairs = 0;
  if (P.compute_penetration) {
    if ((rc = run_deferred_epa<MODE>(ctx, sl, ag, sC))) {
      drain();
      return rc;
    }
    CK(ctx->fix_ids.reserve(n * 4));
    CK(ctx->fix_rows.reserve(n * sizeof(OutT)));
    const unsigned* d_cnt = static_cast<const unsigned*>(sl.counters.p);
    k_gather_epa_rows<OutT><<<(unsigned)ctx->num_sms * 2u, 256, 0, sC>>>(static_cast<const EpaItem*>(sl.queue.p), d_cnt, d_out,
                                                                         static_cast<uint32_t*>(ctx->fix_ids.p),
                                                                         static_cast<OutT*>(ctx->fix_rows.p));
    ctx->stats.kernel_launches++;
    CK(cudaGetLastError());
    cudaEvent_t ev_epa = ctx->pipe_events[2 * nchunks];
    CK(cudaEventRecord(ev_epa, sC));
    CK(cudaStreamWaitEvent(sD, ev_epa, 0));
    CK(cudaMemcpyAsync(&epa_pairs, d_cnt, sizeof(unsigned), cudaMemcpyDeviceToHost, sD));
    if (trace) {
      cudaStreamSynchronize(sC);
      stamp("EPA + gather done");
    }
    CK(cudaStreamSynchronize(sD));  // every chunk's rows are on the host now, and the count
    stamp("rows + count on the host");
    ctx->pipe_epa_frac = (double)epa_pairs / (double)n;
    if (epa_pairs > n / 16) {
      // many EPA pairs (half of the hull pairs of config 3): placing their records one by one costs the host more than
      // taking every record again (25 ns per scattered row against 1.7 ns per row of a plain copy)
      if (min_out) {
        k_pick_min_distance<<<(unsigned)((n + 255) / 256), 256, 0, sD>>>(reinterpret_cast<const hfb_distance_result*>(d_out), (unsigned)n,
                                                                          static_cast<double*>(ctx->big_min.p));
        CK(cudaMemcpyAsync(min_out, ctx->big_min.p, n * 8, cudaMemcpyDeviceToHost, sD));
      } else {
        CK(cudaMemcpyAsync(out, d_out, n * sizeof(OutT), cudaMemcpyDeviceToHost, sD));
      }
      CK(cudaStreamSynchronize(sD));
    } else if (epa_pairs) {
      const size_t need = (size_t)epa_pairs * (4 + sizeof(OutT)) + 64;
      if (ctx->pin_fix_cap < need) {
        if (ctx->pin_fix) cudaFreeHost(ctx->pin_fix);
        ctx->pin_fix = nullptr;
        ctx->pin_fix_cap = 0;
        CK(cudaHostAlloc(&ctx->pin_fix, need + need / 2, cudaHostAllocDefault));
        ctx->pin_fix_cap = need + need / 2;
      }
      OutT* hrows = static_cast<OutT*>(ctx->pin_fix);
      uint32_t* hids = reinterpret_cast<uint32_t*>(static_cast<unsigned char*>(ctx->pin_fix) + (size_t)epa_pairs * sizeof(OutT));
      CK(cudaMemcpyAsync(hrows, ctx->fix_rows.p, (size_t)epa_pairs * sizeof(OutT), cudaMemcpyDeviceToHost, sD));
      CK(cudaMemcpyAsync(hids, ctx->fix_ids.p, (size_t)epa_pairs * 4, cudaMemcpyDeviceToHost, sD));
      CK(cudaStreamSynchronize(sD));
      if constexpr (MODE == 0) {
        if (min_out) {
          for (unsigned k = 0; k < epa_pairs; ++k) min_out[hids[k]] = hrows[k].min_distance;
        } else {
          for (unsigned k = 0; k < epa_pairs; ++k) out[hids[k]] = hrows[k];
        }
      } else {
        for (unsigned k = 0; k < epa_pairs; ++k) out[hids[k]] = hrows[k];
      }
    }
  }
  for (int k = 0; k < kSlots; ++k) CK(cudaStreamSynchronize(ctx->slots[k].stream));
  stamp("done");
  return HFB_OK;
}

template <int MODE, typename Req, typename OutT>
int host_batch(hfb_ctx* ctx, size_t n, const uint32_t* h1, const hfb_transform* tf1, const uint32_t* h2,
               const hfb_transform* tf2, const Req* req, const SolverP& P, const CollideP& Cp, const BvhReq& Bq,
               OutT* out, const hfb_guess_out* go, hfb_contact* extra_out = nullptr, uint32_t* counts_out = nullptr,
               unsigned extra_cap = 0, const ObjSrc* obj = nullptr, const OutMode* om = nullptr) {
  int rc;
  if ((rc = check_ready(ctx))) return rc;
  if (n == 0) return HFB_OK;
  const bool compact = om && (om->min_out || om->flags);
  if (obj ? (!obj->first || !obj->second) : (!h1 || !h2 || !tf1 || !tf2)) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "null buffer");
  if (!out && !compact) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "null buffer");
  CK(cudaSetDevice(ctx->device));
  const bool cached = req->q.gjk_initial_guess == HFB_GUESS_CACHED;
  const double* gin = cached ? req->q.cached_gjk_guess : nullptr;
  const int32_t* hin = cached ? req->q.cached_support_func_guess : nullptr;
  {  // large plain batches: phase 1 chunk by chunk, EPA once (host_batch_pipelined)
    const bool plain = !go && !extra_out && !counts_out && !(om && om->flags) && !gin && !hin;
    // (full records only: with 8 bytes per pair down there is nothing to overlap and the rotating slots serve;
    // HFB_HOST_PIPE=2 sends those calls here as well)
    const bool min_only = om && om->min_out;
    bool take = ctx->host_pipe && plain && n >= kChunk && n <= (size_t)16 << 20 && (min_only ? ctx->host_pipe > 1 : out != nullptr);
    if (take && ctx->host_pipe < 2 && ctx->pipe_epa_frac > 1.0 / 16 && ++ctx->pipe_skipped % 16 != 0) take = false;
    if (take) {
      if constexpr (MODE == 0)
        return host_batch_pipelined<MODE, OutT>(ctx, n, h1, tf1, h2, tf2, P, Cp, Bq, out, obj, om ? om->min_out : nullptr);
      else
        return host_batch_pipelined<MODE, OutT>(ctx, n, h1, tf1, h2, tf2, P, Cp, Bq, out, obj, nullptr);
    }
  }
  size_t done = 0;
  int si = 0;
  // object-table calls send 8 B per pair up: fewer, larger chunks (256 Ki); the row form is bound by its 200 B per pair
  // of H2D and takes 128 Ki
  size_t chunk = ctx->chunk > 0 ? (size_t)ctx->chunk : (obj ? 2 * kChunk : kChunk);
  chunk = (chunk + 31) & ~(size_t)31;  // the compact collide mode writes whole 32-pair flag words per chunk
  unsigned* d_hits = nullptr;
  if (om && om->flags) {
    CK(ctx->cmp_flags.reserve(((n + 31) / 32) * 4));
    CK(ctx->cmp_count.reserve(sizeof(unsigned)));
    CK(ctx->cmp_ids.reserve((size_t)om->cap * 4 + 4));
    CK(ctx->cmp_recs.reserve((size_t)om->cap * sizeof(hfb_contact) + 8));
    d_hits = static_cast<unsigned*>(ctx->cmp_count.p);
    CK(cudaMemsetAsync(d_hits, 0, sizeof(unsigned), ctx->slots[0].stream));
  }
  if (obj || d_hits) {  // the object table (uploaded by the caller on slot 0's stream) and the zeroed counter come first
    if (!ctx->obj_ready) CK(cudaEventCreateWithFlags(&ctx->obj_ready, cudaEventDisableTiming));
    CK(cudaEventRecord(ctx->obj_ready, ctx->slots[0].stream));
    for (int k = 1; k < kSlots; ++k) CK(cudaStreamWaitEvent(ctx->slots[k].stream, ctx->obj_ready, 0));
  }
  while (done < n) {
    const size_t m = (n - done < chunk) ? (n - done) : chunk;
    // handles are validated chunk by chunk, while the previous chunks are in flight.  A bad handle in a
    // later chunk therefore surfaces after earlier chunks ran; the call still fails as a whole.
    if (obj) {
      const uint32_t no = (uint32_t)(obj->n_objects > 0xffffffffull ? 0xffffffffull : obj->n_objects);
      uint32_t bad = 0;  // (branch-free: vectorised by the host compiler)
      for (size_t i = done; i < done + m; ++i) bad |= (uint32_t)(obj->first[i] >= no) | (uint32_t)(obj->second[i] >= no);
      if (bad) {
        for (int k = 0; k < kSlots; ++k) cudaStreamSynchronize(ctx->slots[k].stream);
        return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "object index out of range");
      }
    } else if ((rc = check_handles(ctx, h1 + done, m)) || (rc = check_handles(ctx, h2 + done, m))) {
      for (int k = 0; k < kSlots; ++k) cudaStreamSynchronize(ctx->slots[k].stream);
      return rc;
    }
    Slot& sl = ctx->slots[si];
    cudaStream_t s = sl.stream;
    // the slot's previous chunk must have drained before its buffers are reused
    CK(cudaStreamSynchronize(s));
    CK(sl.h1.reserve(m * 4));
    CK(sl.h2.reserve(m * 4));
    CK(sl.tf1.reserve(m * sizeof(hfb_transform)));
    CK(sl.tf2.reserve(m * sizeof(hfb_transform)));
    CK(sl.out.reserve(m * sizeof(OutT)));
    if (obj) {
      CK(sl.pi.reserve(m * 4));
      CK(sl.pj.reserve(m * 4));
      CK(cudaMemcpyAsync(sl.pi.p, obj->first + done, m * 4, cudaMemcpyHostToDevice, s));
      CK(cudaMemcpyAsync(sl.pj.p, obj->second + done, m * 4, cudaMemcpyHostToDevice, s));
      unsigned eb = (unsigned)((m * 24 + 255) / 256);
      if (eb > (unsigned)ctx->num_sms * 16u) eb = (unsigned)ctx->num_sms * 16u;
      k_expand_pairs<<<eb, 256, 0, s>>>(obj->d_handles, obj->d_tfs, (unsigned)obj->n_objects,
                                        static_cast<const uint32_t*>(sl.pi.p), static_cast<const uint32_t*>(sl.pj.p),
                                        (unsigned)m, static_cast<uint32_t*>(sl.h1.p), static_cast<hfb_transform*>(sl.tf1.p),
                                        static_cast<uint32_t*>(sl.h2.p), static_cast<hfb_transform*>(sl.tf2.p));
      ctx->stats.kernel_launches++;
      CK(cudaGetLastError());
    } else {
      CK(cudaMemcpyAsync(sl.h1.p, h1 + done, m * 4, cudaMemcpyHostToDevice, s));
      CK(cudaMemcpyAsync(sl.h2.p, h2 + done, m * 4, cudaMemcpyHostToDevice, s));
      CK(cudaMemcpyAsync(sl.tf1.p, tf1 + done, m * sizeof(hfb_transform), cudaMemcpyHostToDevice, s));
      CK(cudaMemcpyAsync(sl.tf2.p, tf2 + done, m * sizeof(hfb_transform), cudaMemcpyHostToDevice, s));
    }
    BatchArgs a{};
    a.n = (unsigned)m;
    a.h1 = static_cast<const uint32_t*>(sl.h1.p);
    a.h2 = static_cast<const uint32_t*>(sl.h2.p);
    a.tf1 = static_cast<const hfb_transform*>(sl.tf1.p);
    a.tf2 = static_cast<const hfb_transform*>(sl.tf2.p);
    a.out = sl.out.p;
    a.P = P;
    a.C = Cp;
    a.B = Bq;
    if (gin) {
      CK(sl.gin.reserve(m * 24));
      CK(cudaMemcpyAsync(sl.gin.p, gin + 3 * done, m * 24, cudaMemcpyHostToDevice, s));
      a.guess_in = static_cast<const double*>(sl.gin.p);
    }
    if (hin) {
      CK(sl.hin.reserve(m * 8));
      CK(cudaMemcpyAsync(sl.hin.p, hin + 2 * done, m * 8, cudaMemcpyHostToDevice, s));
      a.hint_in = static_cast<const int32_t*>(sl.hin.p);
    }
    if (go && go->cached_gjk_guess) {
      CK(sl.gout.reserve(m * 24));
      a.guess_out = static_cast<double*>(sl.gout.p);
    }
    if (go && go->cached_support_func_guess) {
      CK(sl.hout.reserve(m * 8));
      a.hint_out = static_cast<int32_t*>(sl.hout.p);
    }
    if (counts_out) {  // hfb_batch_collide_contacts
      CK(sl.ccnt.reserve(m * sizeof(uint32_t)));
      CK(cudaMemsetAsync(sl.ccnt.p, 0xff, m * sizeof(uint32_t), s));  // pairs no mesh kernel writes keep the mark
      a.counts = static_cast<uint32_t*>(sl.ccnt.p);
      if (extra_out && extra_cap) {
        CK(sl.extra.reserve(m * (size_t)extra_cap * sizeof(hfb_contact)));
        a.extra = static_cast<hfb_contact*>(sl.extra.p);
        a.extra_cap = extra_cap;
      }
    }
    if ((rc = run_device_batch<MODE>(ctx, sl, a, s))) return rc;
    if (a.counts) CK(cudaMemcpyAsync(counts_out + done, a.counts, m * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    if (a.extra)
      CK(cudaMemcpyAsync(extra_out + done * extra_cap, a.extra, m * (size_t)extra_cap * sizeof(hfb_contact),
                         cudaMemcpyDeviceToHost, s));
    if constexpr (MODE == 0) {
      if (om && om->min_out) {
        CK(sl.cmp.reserve(m * 8));
        k_pick_min_distance<<<(unsigned)((m + 255) / 256), 256, 0, s>>>(static_cast<const hfb_distance_result*>(sl.out.p),
                                                                         (unsigned)m, static_cast<double*>(sl.cmp.p));
        ctx->stats.kernel_launches++;
        CK(cudaMemcpyAsync(om->min_out + done, sl.cmp.p, m * 8, cudaMemcpyDeviceToHost, s));
      }
    } else {
      if (om && om->flags) {
        k_compact_contacts<<<(unsigned)((m + 255) / 256), 256, 0, s>>>(
            static_cast<const hfb_contact*>(sl.out.p), (unsigned)m, (unsigned)done,
            static_cast<uint32_t*>(ctx->cmp_flags.p) + done / 32, d_hits, static_cast<uint32_t*>(ctx->cmp_ids.p),
            static_cast<hfb_contact*>(ctx->cmp_recs.p), om->cap);
        ctx->stats.kernel_launches++;
      }
    }
    if (out) CK(cudaMemcpyAsync(out + done, sl.out.p, m * sizeof(OutT), cudaMemcpyDeviceToHost, s));
    if (a.guess_out)
      CK(cudaMemcpyAsync(go->cached_gjk_guess + 3 * done, a.guess_out, m * 24, cudaMemcpyDeviceToHost, s));
    if (a.hint_out)
      CK(cudaMemcpyAsync(go->cached_support_func_guess + 2 * done, a.hint_out, m * 8, cudaMemcpyDeviceToHost, s));
    done += m;
    si = (si + 1) % kSlots;
  }
  for (int k = 0; k < kSlots; ++k) CK(cudaStreamSynchronize(ctx->slots[k].stream));
  if (om && om->flags) {
    unsigned hits = 0;
    CK(cudaMemcpy(&hits, d_hits, sizeof(unsigned), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(om->flags, ctx->cmp_flags.p, ((n + 31) / 32) * 4, cudaMemcpyDeviceToHost));
    if (om->n_hits) *om->n_hits = hits;
    const unsigned kept = hits < om->cap ? hits : om->cap;
    if (kept && om->hit_ids) CK(cudaMemcpy(om->hit_ids, ctx->cmp_ids.p, (size_t)kept * 4, cudaMemcpyDeviceToHost));
    if (kept && om->hit_recs) CK(cudaMemcpy(om->hit_recs, ctx->cmp_recs.p, (size_t)kept * sizeof(hfb_contact), cudaMemcpyDeviceToHost));
  }
  return HFB_OK;
}

template <int MODE, typename Req>
int device_batch(hfb_ctx* ctx, size_t n, const uint32_t* h1, const hfb_transform* tf1, const uint32_t* h2,
                 const hfb_transform* tf2, const Req* req, const SolverP& P, const CollideP& Cp, const BvhReq& Bq,
                 void* out, const hfb_guess_out* go, void* stream) {
  int rc;
  if ((rc = check_ready(ctx))) return rc;
  if (n == 0) return HFB_OK;
  if (n > 0xffffffffull) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "batch too large");
  if (!h1 || !h2 || !tf1 || !tf2 || !out) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "null buffer");
  CK(cudaSetDevice(ctx->device));
  const bool cached = req->q.gjk_initial_guess == HFB_GUESS_CACHED;
  BatchArgs a{};
  a.n = (unsigned)n;
  a.h1 = h1;
  a.h2 = h2;
  a.tf1 = tf1;
  a.tf2 = tf2;
  a.out = out;
  a.P = P;
  a.C = Cp;
  a.B = Bq;
  a.guess_in = cached ? req->q.cached_gjk_guess : nullptr;
  a.hint_in = cached ? req->q.cached_support_func_guess : nullptr;
  a.guess_out = go ? go->cached_gjk_guess : nullptr;
  a.hint_out = go ? go->cached_support_func_guess : nullptr;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if ((rc = after_device_calls(ctx, st))) return rc;
  rc = run_device_batch<MODE>(ctx, ctx->dev_slot, a, st);
  if (int e = last_device_call(ctx, st)) return e;
  return rc;
}

}  // namespace

// ==================================================================== C-ABI ===
extern "C" {

const char* hfb_version(void) { return "hppfcl_b200 0.1 (sm_90a, fp64, fmad=false)"; }

void hfb_default_distance_request(hfb_distance_request* r) {
  std::memset(r, 0, sizeof(*r));
  r->q.gjk_max_iterations = 128;
  r->q.epa_max_iterations = 64;
  r->q.gjk_tolerance = 1e-6;
  r->q.epa_tolerance = 1e-6;
  r->q.collision_distance_threshold = 1e-12;
  r->enable_signed_distance = 1;
  r->enable_nearest_points = 1;
}
void hfb_default_collision_request(hfb_collision_request* r) {
  std::memset(r, 0, sizeof(*r));
  r->q.gjk_max_iterations = 128;
  r->q.epa_max_iterations = 64;
  r->q.gjk_tolerance = 1e-6;
  r->q.epa_tolerance = 1e-6;
  r->q.collision_distance_threshold = 1e-12;
  r->num_max_contacts = 1;
  r->enable_contact = 1;
  r->security_margin = 0;
  r->break_distance = 1e-3;
  r->distance_upper_bound = DBL_MAX;
}

int hfb_ctx_create(int device, hfb_ctx** out) {
  if (!out) return HFB_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count)
    return HFB_ERR_NO_DEVICE;  // no CPU fallback by design
  if (cudaSetDevice(device) != cudaSuccess) return HFB_ERR_NO_DEVICE;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return HFB_ERR_NO_DEVICE;
  hfb_ctx* c = new hfb_ctx();
  c->device = device;
  c->num_sms = prop.multiProcessorCount;
  auto env_g = [](const char* name, int dflt) {
    const char* v = getenv(name);
    const int g = v ? atoi(v) : dflt;
    return (g == 8 || g == 16 || g == 32) ? g : dflt;
  };
  c->gc = env_g("HFB_GC", HFB_GC_DEFAULT);
  if (const char* v4 = getenv("HFB_GC")) {
    const int g = atoi(v4);
    if (g == 1 || g == 2 || g == 4) c->gc = g;  // phase 1 also comes with 1, 2, 4 lanes per pair
  }
  c->ge = env_g("HFB_GE", HFB_GE_DEFAULT);
  if (const char* v4 = getenv("HFB_GE"))
    if (atoi(v4) == 4) c->ge = 4;
  if (const char* mb = getenv("HFB_MINB")) c->minb = atoi(mb);
  if (const char* ns = getenv("HFB_NSUB")) c->nsub = atoi(ns);
  if (const char* bm = getenv("HFB_BVH_MINB")) c->bvh_minb = atoi(bm);
  if (const char* bo = getenv("HFB_BVH_ORDER")) c->bvh_order = atoi(bo) != 0;
  if (const char* bq2 = getenv("HFB_BVHQ")) c->bvhq = atoi(bq2) != 0;
  if (const char* bs = getenv("HFB_BVH_SPEC")) c->bvh_spec = atoi(bs);
  if (const char* bc = getenv("HFB_BVH_GJK_CHUNK")) c->bvh_chunk = atoi(bc) > 0 ? atoi(bc) : 1;
  if (const char* hs = getenv("HFB_HULL_SORT")) c->hull_sort = atoi(hs) != 0;
  if (const char* hp = getenv("HFB_HOST_PIPE")) c->host_pipe = atoi(hp) < 0 ? 0 : atoi(hp);
  if (const char* er = getenv("HFB_EPA_RESUME")) c->epa_resume = atoi(er) > 0 ? atoi(er) : 0;
  if (const char* gp = getenv("HFB_GJK_PASSES")) {
    c->gjk_npass = 0;
    int k = 0;
    for (const char* q = gp; *q && k < 7;) {
      const int v = atoi(q);
      if (v > 0) c->gjk_steps[k++] = v;
      while (*q && *q != ',') ++q;
      if (*q == ',') ++q;
    }
    c->gjk_npass = k > 0 ? k + 1 : 0;
  }
  if (const char* bw = getenv("HFB_BVH_WARPS")) c->bvh_warps = atoi(bw) >= 16 ? 16 : (atoi(bw) >= 12 ? 12 : 8);
  if (const char* eo = getenv("HFB_EPA_OVERLAP")) c->epa_overlap = atoi(eo) != 0;
  if (const char* bg = getenv("HFB_BVH_GENS")) c->bvh_gens = atoi(bg) > 0 ? atoi(bg) : 1;
  if (const char* bb = getenv("HFB_BVH_SPEC_BIG")) c->bvh_spec_big = atoi(bb) >= 0 ? atoi(bb) : 0;
  if (const char* bq = getenv("HFB_BVH_QUORUM"))
    if (atoi(bq) == 1) c->bvh_quorum = 1;
  if (const char* bp = getenv("HFB_BVH_BPS")) {
    const int v = atoi(bp);
    if (v >= 1 && v <= 4) c->bvh_bps = v;  // the workspace is sized for 4
  }
  if (const char* rf = getenv("HFB_REFILL")) c->refill = atoi(rf);
  if (const char* st = getenv("HFB_STAGE")) c->stage = atoi(st);
  if (const char* ch = getenv("HFB_CHUNK")) c->chunk = atoi(ch);
  if (const char* iq = getenv("HFB_ITER_QUORUM")) c->iter_quorum = atoi(iq);
  for (int k = 0; k < kSlots; ++k)
    if (cudaStreamCreateWithFlags(&c->slots[k].stream, cudaStreamNonBlocking) != cudaSuccess) {
      delete c;
      return HFB_ERR_CUDA;
    }
  *out = c;
  return HFB_OK;
}

void hfb_ctx_destroy(hfb_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  hfb_comm_destroy(c);
  auto destroy_streams = [](Slot& s) {
    if (s.stream) cudaStreamDestroy(s.stream);
    if (s.epa_stream) cudaStreamDestroy(s.epa_stream);
    if (s.work_stream) cudaStreamDestroy(s.work_stream);
    for (cudaEvent_t e : s.ev_part)
      if (e) cudaEventDestroy(e);
    if (s.ev_join) cudaEventDestroy(s.ev_join);
    if (s.ev_fork) cudaEventDestroy(s.ev_fork);
    if (s.ev_work) cudaEventDestroy(s.ev_work);
  };
  for (int k = 0; k < kSlots; ++k) destroy_streams(c->slots[k]);
  destroy_streams(c->dev_slot);
  if (c->dev_done) cudaEventDestroy(c->dev_done);
  if (c->pin_fix) cudaFreeHost(c->pin_fix);
  for (cudaEvent_t e : c->pipe_events) cudaEventDestroy(e);
  for (hfb_env* e : c->envs) delete e;
  for (hfb_robot* r : c->robots) delete r;
  if (c->obj_ready) cudaEventDestroy(c->obj_ready);
  delete c;  // and with it every device buffer of the context (DevBuf)
}

const char* hfb_last_error(const hfb_ctx* c) { return c ? c->err.c_str() : "null context"; }

int hfb_geom_register_shapes(hfb_ctx* ctx, const hfb_shape* shapes, size_t n, uint32_t* handles_out) {
  if (!ctx || (!shapes && n)) return HFB_ERR_INVALID_ARGUMENT;
  for (size_t i = 0; i < n; ++i) {
    uint32_t h;
    if (shapes[i].type == HFB_GEOM_PLANE || shapes[i].type == HFB_GEOM_HALFSPACE)  // (a 40-byte record has no room for n and d)
      return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "planes and halfspaces are registered with hfb_geom_register_halfspaces");
    if (!ctx->arena.add_shape(shapes[i], &h)) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "bad convex id in shape record");
    if (handles_out) handles_out[i] = h;
  }
  ctx->committed = false;
  return HFB_OK;
}

int hfb_geom_register_halfspaces(hfb_ctx* ctx, uint32_t type, const double* n_d, const double* ssr, size_t count,
                                 uint32_t* handles_out) {
  if (!ctx || (!n_d && count) || (type != HFB_GEOM_PLANE && type != HFB_GEOM_HALFSPACE))
    return HFB_ERR_INVALID_ARGUMENT;
  for (size_t i = 0; i < count; ++i) {
    uint32_t h;
    if (!ctx->arena.add_halfspace(type, n_d + 4 * i, n_d[4 * i + 3], ssr ? ssr[i] : 0.0, &h))
      return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "bad plane record");
    if (handles_out) handles_out[i] = h;
  }
  ctx->committed = false;
  return HFB_OK;
}

int hfb_geom_register_convex_batch(hfb_ctx* ctx, const double* points, uint32_t num_points, uint32_t count,
                                   uint32_t* first_id) {
  if (!ctx || !points || num_points == 0 || count == 0 || !first_id) return HFB_ERR_INVALID_ARGUMENT;
  for (uint32_t k = 0; k < count; ++k) {
    const uint32_t id = ctx->arena.add_convex(points + 3 * (size_t)num_points * k, num_points);
    if (k == 0) *first_id = id;
  }
  ctx->committed = false;
  return HFB_OK;
}
int hfb_geom_register_convex(hfb_ctx* ctx, const double* points, uint32_t num_points, uint32_t* convex_id) {
  if (!ctx || !points || num_points == 0 || !convex_id) return HFB_ERR_INVALID_ARGUMENT;
  *convex_id = ctx->arena.add_convex(points, num_points);
  ctx->committed = false;
  return HFB_OK;
}

int hfb_bvh_build_obbrss(const double* vertices, uint32_t num_vertices, const uint32_t* triangles,
                         uint32_t num_triangles, hfb_bvh_node* nodes_out, uint32_t nodes_capacity) {
  if (num_triangles == 0 || nodes_capacity < 2 * num_triangles - 1) return HFB_ERR_INVALID_ARGUMENT;
  return build_obbrss_tree(vertices, num_vertices, triangles, num_triangles, nodes_out) ? HFB_OK
                                                                                        : HFB_ERR_INVALID_ARGUMENT;
}

int hfb_geom_register_bvh_obbrss(hfb_ctx* ctx, const hfb_bvh_node* nodes, uint32_t num_nodes, const double* vertices,
                                 uint32_t num_vertices, const uint32_t* triangles, uint32_t num_triangles,
                                 uint32_t* bvh_id) {
  if (!ctx || !nodes || !vertices || !triangles || !bvh_id) return HFB_ERR_INVALID_ARGUMENT;
  if (!ctx->arena.add_bvh(nodes, num_nodes, vertices, num_vertices, triangles, num_triangles, bvh_id))
    return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "malformed OBBRSS BVH (child links / primitive ids / vertex ids)");
  ctx->committed = false;
  return HFB_OK;
}

int hfb_geom_register_bvh_obb(hfb_ctx* ctx, const hfb_bvh_node* nodes, uint32_t num_nodes, const double* vertices,
                              uint32_t num_vertices, const uint32_t* triangles, uint32_t num_triangles, uint32_t* bvh_id) {
  if (!ctx || !nodes || !vertices || !triangles || !bvh_id) return HFB_ERR_INVALID_ARGUMENT;
  if (!ctx->arena.add_bvh(nodes, num_nodes, vertices, num_vertices, triangles, num_triangles, bvh_id, 1))
    return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "malformed OBB BVH (child links / primitive ids / vertex ids / depth)");
  ctx->committed = false;
  return HFB_OK;
}

int hfb_geom_commit(hfb_ctx* ctx) {
  if (!ctx) return HFB_ERR_INVALID_ARGUMENT;
  CK(cudaSetDevice(ctx->device));
  const HostArena& A = ctx->arena;
  auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
  const size_t bs = up(A.shapes.size() * sizeof(hfb_shape));
  const size_t bc = up(A.cvx.size() * sizeof(ConvexDesc));
  const size_t bp = up(A.pool.size() * sizeof(double));
  const size_t bn = up(A.bvh_nodes.size() * sizeof(hfb_bvh_node));
  const size_t bv = up(A.bvh_verts.size() * sizeof(double));
  const size_t bt = up(A.bvh_tris.size() * sizeof(uint32_t));
  const size_t bd = up(A.bvh_desc.size() * sizeof(BvhDesc));
  const size_t bl = up(A.shapes.size() * 6 * sizeof(double));
  ctx->local_aabbs.assign(A.shapes.size() * 6, NAN);
  for (size_t i = 0; i < A.shapes.size(); ++i) {
    LocalAabb b;
    if (shape_local_aabb(A, A.shapes[i], b))
      for (int k = 0; k < 3; ++k) {
        ctx->local_aabbs[6 * i + k] = b.mn[k];
        ctx->local_aabbs[6 * i + 3 + k] = b.mx[k];
      }
  }
  CK(cudaDeviceSynchronize());
  CK(ctx->d_arena.reserve(bs + bc + bp + bn + bv + bt + bd + bl + 256));
  unsigned char* base = static_cast<unsigned char*>(ctx->d_arena.p);
  if (!A.shapes.empty()) CK(cudaMemcpy(base, A.shapes.data(), A.shapes.size() * sizeof(hfb_shape), cudaMemcpyHostToDevice));
  if (!A.cvx.empty()) CK(cudaMemcpy(base + bs, A.cvx.data(), A.cvx.size() * sizeof(ConvexDesc), cudaMemcpyHostToDevice));
  if (!A.pool.empty()) CK(cudaMemcpy(base + bs + bc, A.pool.data(), A.pool.size() * sizeof(double), cudaMemcpyHostToDevice));
  ctx->dview.shapes = reinterpret_cast<const hfb_shape*>(base);
  ctx->dview.cvx = reinterpret_cast<const ConvexDesc*>(base + bs);
  ctx->dview.pool = reinterpret_cast<const double*>(base + bs + bc);
  ctx->dview.nshapes = (uint32_t)A.shapes.size();
  ctx->dview.ncvx = (uint32_t)A.cvx.size();
  unsigned char* pb = base + bs + bc + bp;
  if (!A.bvh_nodes.empty()) {
    CK(cudaMemcpy(pb, A.bvh_nodes.data(), A.bvh_nodes.size() * sizeof(hfb_bvh_node), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(pb + bn, A.bvh_verts.data(), A.bvh_verts.size() * sizeof(double), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(pb + bn + bv, A.bvh_tris.data(), A.bvh_tris.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(pb + bn + bv + bt, A.bvh_desc.data(), A.bvh_desc.size() * sizeof(BvhDesc), cudaMemcpyHostToDevice));
  }
  ctx->dview.bvh_nodes = reinterpret_cast<const hfb_bvh_node*>(pb);
  ctx->dview.bvh_verts = reinterpret_cast<const double*>(pb + bn);
  ctx->dview.bvh_tris = reinterpret_cast<const uint32_t*>(pb + bn + bv);
  ctx->dview.bvh_desc = reinterpret_cast<const BvhDesc*>(pb + bn + bv + bt);
  ctx->dview.nbvh = (uint32_t)A.bvh_desc.size();
  {
    unsigned char* pl = base + bs + bc + bp + bn + bv + bt + bd;
    if (!ctx->local_aabbs.empty())
      CK(cudaMemcpy(pl, ctx->local_aabbs.data(), ctx->local_aabbs.size() * sizeof(double), cudaMemcpyHostToDevice));
    ctx->dview.local_aabbs = reinterpret_cast<const double*>(pl);
  }
  ctx->committed = true;
  ++ctx->commits;
  return HFB_OK;
}

int hfb_geom_device_arena(hfb_ctx* ctx, void** base, size_t* bytes) {
  int rc;
  if ((rc = check_ready(ctx))) return rc;
  if (base) *base = ctx->d_arena.p;
  if (bytes) *bytes = ctx->d_arena.cap;
  return HFB_OK;
}

size_t hfb_geom_num_shapes(const hfb_ctx* ctx) { return ctx ? ctx->arena.shapes.size() : 0; }
int hfb_geom_clear(hfb_ctx* ctx) {
  if (!ctx) return HFB_ERR_INVALID_ARGUMENT;
  CK(cudaSetDevice(ctx->device));
  CK(cudaDeviceSynchronize());
  ctx->arena = HostArena();
  ctx->dview = ArenaView{};
  ctx->committed = false;
  ++ctx->clears;
  return HFB_OK;
}

int hfb_geom_update_shapes(hfb_ctx* ctx, const uint32_t* handles, const hfb_shape* shapes, size_t n) {
  if (!ctx || ((!handles || !shapes) && n)) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  for (size_t i = 0; i < n; ++i)  // all or nothing
    if (handles[i] >= ctx->arena.shapes.size()) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "shape handle out of range");
  for (size_t i = 0; i < n; ++i) {
    if (shapes[i].type == HFB_GEOM_PLANE || shapes[i].type == HFB_GEOM_HALFSPACE)  // (no room for n and d in a record)
      return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "a plane is moved by its pose, or registered anew (hfb_geom_register_halfspaces)");
    if (!ctx->arena.valid_shape(shapes[i])) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "bad shape record");
  }
  for (size_t i = 0; i < n; ++i) ctx->arena.set_shape(handles[i], shapes[i]);
  ctx->committed = false;
  return HFB_OK;
}

int hfb_geom_update_convex(hfb_ctx* ctx, uint32_t convex_id, const double* points, uint32_t num_points) {
  if (!ctx || !points) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->arena.set_convex(convex_id, points, num_points))
    return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "unknown convex id or a different number of points");
  ctx->committed = false;
  return HFB_OK;
}

int hfb_geom_release_shapes(hfb_ctx* ctx, const uint32_t* handles, size_t n) {
  if (!ctx || (!handles && n)) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  for (size_t i = 0; i < n; ++i)
    if (handles[i] >= ctx->arena.shapes.size()) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "shape handle out of range");
  hfb_shape gone;
  std::memset(&gone, 0, sizeof(gone));  // type 0: no such geometry
  for (size_t i = 0; i < n; ++i) ctx->arena.set_shape(handles[i], gone);
  ctx->committed = false;
  return HFB_OK;
}

int hfb_batch_distance(hfb_ctx* ctx, size_t n, const uint32_t* h1, const hfb_transform* tf1,
                       const uint32_t* h2, const hfb_transform* tf2, const hfb_distance_request* req,
                       hfb_distance_result* out, const hfb_guess_out* go) {
  if (!ctx || !req) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (int rc = validate_query(req->q)) return fail(ctx, rc, "invalid request");
  return host_batch<0>(ctx, n, h1, tf1, h2, tf2, req, solver_from_distance_request(*req), CollideP{0, 0},
                       BvhReq{/* rel_err, abs_err: see hfb_distance_request */ 0, 0, 0, 0, 0, 1, req->enable_nearest_points != 0, req->q.gjk_initial_guess}, out, go);
}

int hfb_batch_distance_device(hfb_ctx* ctx, size_t n, const uint32_t* h1, const hfb_transform* tf1,
                              const uint32_t* h2, const hfb_transform* tf2, const hfb_distance_request* req,
                              hfb_distance_result* out, const hfb_guess_out* go, void* stream) {
  if (!ctx || !req) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (int rc = validate_query(req->q)) return fail(ctx, rc, "invalid request");
  return device_batch<0>(ctx, n, h1, tf1, h2, tf2, req, solver_from_distance_request(*req), CollideP{0, 0},
                         BvhReq{/* rel_err, abs_err: see hfb_distance_request */ 0, 0, 0, 0, 0, 1, req->enable_nearest_points != 0, req->q.gjk_initial_guess}, out, go, stream);
}

// collision.cpp:73-76: security_margin == -inf => result.clear(), no contact
__global__ void k_clear_contacts(hfb_contact* out, unsigned n) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  PairOut o;
  o.status = pack_status(0, 0, HFB_PATH_UNSUPPORTED);
  o.iterations = 0;
  CollideP C{0, 0};
  write_contact(o, C, out + i);
  out[i].status = 0;
}

int hfb_batch_collide(hfb_ctx* ctx, size_t n, const uint32_t* h1, const hfb_transform* tf1,
                      const uint32_t* h2, const hfb_transform* tf2, const hfb_collision_request* req,
                      hfb_contact* out, const hfb_guess_out* go) {
  if (!ctx || !req) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  bool minus_inf;
  if (int rc = collide_prelude(ctx, req, &minus_inf)) return rc;
  if (minus_inf) {
    if (int rc = check_ready(ctx)) return rc;
    if (n == 0) return HFB_OK;
    Slot& sl = ctx->slots[0];
    CK(sl.out.reserve(n * sizeof(hfb_contact)));
    k_clear_contacts<<<(unsigned)((n + 255) / 256), 256, 0, sl.stream>>>(static_cast<hfb_contact*>(sl.out.p), (unsigned)n);
    ctx->stats.kernel_launches++;
    CK(cudaMemcpyAsync(out, sl.out.p, n * sizeof(hfb_contact), cudaMemcpyDeviceToHost, sl.stream));
    CK(cudaStreamSynchronize(sl.stream));
    return HFB_OK;
  }
  CollideP C{req->security_margin, req->q.collision_distance_threshold};
  return host_batch<1>(ctx, n, h1, tf1, h2, tf2, req, solver_from_collision_request(*req), C,
                       BvhReq{0, 0, req->security_margin, req->break_distance, req->q.collision_distance_threshold,
                              req->num_max_contacts, true, req->q.gjk_initial_guess},
                       out, go);
}

int hfb_batch_collide_contacts(hfb_ctx* ctx, size_t n, const uint32_t* h1, const hfb_transform* tf1, const uint32_t* h2,
                               const hfb_transform* tf2, const hfb_collision_request* req, hfb_contact* out,
                               uint32_t max_extra, hfb_contact* extra, uint32_t* counts, const hfb_guess_out* go) {
  if (!ctx || !req || !counts || (max_extra && !extra)) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  bool minus_inf;
  if (int rc = collide_prelude(ctx, req, &minus_inf)) return rc;
  if (minus_inf) {  // collision.cpp:73-76: cleared results, no contacts
    if (int rc = check_ready(ctx)) return rc;
    if (n && !out) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "null buffer");
    for (size_t i = 0; i < n; ++i) {
      bvh_init_contact(&out[i]);
      out[i].status = 0;
      counts[i] = 0;
    }
    return HFB_OK;
  }
  CollideP C{req->security_margin, req->q.collision_distance_threshold};
  const int rc = host_batch<1>(ctx, n, h1, tf1, h2, tf2, req, solver_from_collision_request(*req), C,
                               BvhReq{0, 0, req->security_margin, req->break_distance, req->q.collision_distance_threshold,
                                      req->num_max_contacts, true, req->q.gjk_initial_guess},
                               out, go, extra, counts, max_extra);
  if (rc) return rc;
  for (size_t i = 0; i < n; ++i)
    if (counts[i] == 0xffffffffu) counts[i] = out[i].num_contacts;  // shape pairs: at most one contact
  return HFB_OK;
}

int hfb_batch_collide_device(hfb_ctx* ctx, size_t n, const uint32_t* h1, const hfb_transform* tf1,
                             const uint32_t* h2, const hfb_transform* tf2, const hfb_collision_request* req,
                             hfb_contact* out, const hfb_guess_out* go, void* stream) {
  if (!ctx || !req) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  bool minus_inf;
  if (int rc = collide_prelude(ctx, req, &minus_inf)) return rc;
  if (minus_inf) {
    if (int rc = check_ready(ctx)) return rc;
    if (n == 0) return HFB_OK;
    if (n > 0xffffffffull) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "batch too large");
    if (!out) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "null buffer");
    k_clear_contacts<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(out, (unsigned)n);
    ctx->stats.kernel_launches++;
    CK(cudaGetLastError());
    return HFB_OK;
  }
  CollideP C{req->security_margin, req->q.collision_distance_threshold};
  return device_batch<1>(ctx, n, h1, tf1, h2, tf2, req, solver_from_collision_request(*req), C,
                         BvhReq{0, 0, req->security_margin, req->break_distance, req->q.collision_distance_threshold,
                                req->num_max_contacts, true, req->q.gjk_initial_guess},
                         out, go, stream);
}


// ---- object-table entry points ------------------------------------------------------------------------
static int upload_objects(hfb_ctx* ctx, const hfb_object_pairs* sc, ObjSrc* o) {
  if (!sc) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "null scene");
  if (int rc = check_ready(ctx)) return rc;
  if (sc->n_pairs > 0xffffffffull || sc->n_objects > 0xffffffffull) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "batch too large");
  if (sc->n_objects && (!sc->object_handles || !sc->object_tfs)) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "null buffer");
  if (int rc = check_handles(ctx, sc->object_handles, sc->n_objects)) return rc;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s0 = ctx->slots[0].stream;
  CK(ctx->obj_h.reserve(sc->n_objects * 4 + 4));
  CK(ctx->obj_tf.reserve(sc->n_objects * sizeof(hfb_transform) + 8));
  if (sc->n_objects) {
    CK(cudaMemcpyAsync(ctx->obj_h.p, sc->object_handles, sc->n_objects * 4, cudaMemcpyHostToDevice, s0));
    CK(cudaMemcpyAsync(ctx->obj_tf.p, sc->object_tfs, sc->n_objects * sizeof(hfb_transform), cudaMemcpyHostToDevice, s0));
  }
  o->n_objects = sc->n_objects;
  o->d_handles = static_cast<const uint32_t*>(ctx->obj_h.p);
  o->d_tfs = static_cast<const hfb_transform*>(ctx->obj_tf.p);
  o->first = sc->first;
  o->second = sc->second;
  return HFB_OK;
}

int hfb_batch_distance_objects(hfb_ctx* ctx, const hfb_object_pairs* scene, const hfb_distance_request* req,
                               hfb_distance_result* out, double* min_distance_out, const hfb_guess_out* go) {
  if (!ctx || !req) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (int rc = validate_query(req->q)) return fail(ctx, rc, "invalid request");
  ObjSrc o;
  if (int rc = upload_objects(ctx, scene, &o)) return rc;
  OutMode om;
  om.min_out = min_distance_out;
  return host_batch<0>(ctx, scene->n_pairs, nullptr, nullptr, nullptr, nullptr, req, solver_from_distance_request(*req),
                       CollideP{0, 0}, bvh_req_of_distance(req), out, go, nullptr, nullptr, 0, &o, &om);
}

int hfb_batch_collide_objects(hfb_ctx* ctx, const hfb_object_pairs* scene, const hfb_collision_request* req,
                              hfb_contact* out, const hfb_compact_contacts* compact, const hfb_guess_out* go) {
  if (!ctx || !req) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  bool minus_inf;
  if (int rc = collide_prelude(ctx, req, &minus_inf)) return rc;
  if (compact && (!compact->flags || (compact->capacity && (!compact->pair_ids || !compact->contacts))))
    return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "null buffer");
  ObjSrc o;
  if (int rc = upload_objects(ctx, scene, &o)) return rc;
  const size_t n = scene->n_pairs;
  if (minus_inf) {  // collision.cpp:73-76: cleared results, no contacts
    if (n && !out && !compact) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "null buffer");
    CK(cudaStreamSynchronize(ctx->slots[0].stream));
    for (size_t i = 0; out && i < n; ++i) {
      bvh_init_contact(&out[i]);
      out[i].status = 0;
    }
    if (compact) {
      std::memset(compact->flags, 0, ((n + 31) / 32) * 4);
      if (compact->n_colliding) *compact->n_colliding = 0;
    }
    return HFB_OK;
  }
  OutMode om;
  if (compact) {
    om.flags = compact->flags;
    om.n_hits = compact->n_colliding;
    om.hit_ids = compact->pair_ids;
    om.hit_recs = compact->contacts;
    om.cap = compact->capacity;
  }
  CollideP C{req->security_margin, req->q.collision_distance_threshold};
  return host_batch<1>(ctx, n, nullptr, nullptr, nullptr, nullptr, req, solver_from_collision_request(*req), C,
                       bvh_req_of_collision(req), out, go, nullptr, nullptr, 0, &o, &om);
}

}  // extern "C"

BvhReq bvh_req_of_distance(const hfb_distance_request* req) {
  return BvhReq{/* rel_err, abs_err: see hfb_distance_request */ 0, 0, 0, 0, 0, 1, req->enable_nearest_points != 0, req->q.gjk_initial_guess};
}
BvhReq bvh_req_of_collision(const hfb_collision_request* req) {
  return BvhReq{0, 0, req->security_margin, req->break_distance, req->q.collision_distance_threshold, req->num_max_contacts, true,
                req->q.gjk_initial_guess};
}

// device-resident scene: the pairs are expanded into the context's scratch rows, then the batch runs as
// hfb_batch_*_device does
template <int MODE, typename Req>
int objects_device(hfb_ctx* ctx, const hfb_object_pairs* sc, const Req* req, const SolverP& P, const CollideP& Cp,
                          const BvhReq& Bq, void* out, const hfb_guess_out* go, void* stream) {
  if (!sc) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "null scene");
  if (int rc = check_ready(ctx)) return rc;
  const size_t n = sc->n_pairs;
  if (n == 0) return HFB_OK;
  if (n > 0xffffffffull || sc->n_objects > 0xffffffffull) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "batch too large");
  if (!sc->object_handles || !sc->object_tfs || !sc->first || !sc->second || !out) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "null buffer");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = after_device_calls(ctx, st)) return rc;
  ctx->dev_used = true;  // (the expansion below already writes the shared scratch; device_batch records the event)
  ctx->dev_last_stream = st;
  Slot& sl = ctx->dev_slot;
  CK(sl.h1.reserve(n * 4));
  CK(sl.h2.reserve(n * 4));
  CK(sl.tf1.reserve(n * sizeof(hfb_transform)));
  CK(sl.tf2.reserve(n * sizeof(hfb_transform)));
  unsigned eb = (unsigned)((n * 24 + 255) / 256);
  if (eb > (unsigned)ctx->num_sms * 16u) eb = (unsigned)ctx->num_sms * 16u;
  k_expand_pairs<<<eb, 256, 0, st>>>(sc->object_handles, sc->object_tfs, (unsigned)sc->n_objects, sc->first, sc->second,
                                     (unsigned)n, static_cast<uint32_t*>(sl.h1.p), static_cast<hfb_transform*>(sl.tf1.p),
                                     static_cast<uint32_t*>(sl.h2.p), static_cast<hfb_transform*>(sl.tf2.p));
  ctx->stats.kernel_launches++;
  CK(cudaGetLastError());
  return device_batch<MODE>(ctx, n, static_cast<const uint32_t*>(sl.h1.p), static_cast<const hfb_transform*>(sl.tf1.p),
                            static_cast<const uint32_t*>(sl.h2.p), static_cast<const hfb_transform*>(sl.tf2.p), req, P, Cp,
                            Bq, out, go, stream);
}
template int objects_device<0, hfb_distance_request>(hfb_ctx*, const hfb_object_pairs*, const hfb_distance_request*,
                                                     const SolverP&, const CollideP&, const BvhReq&, void*,
                                                     const hfb_guess_out*, void*);
template int objects_device<1, hfb_collision_request>(hfb_ctx*, const hfb_object_pairs*, const hfb_collision_request*,
                                                      const SolverP&, const CollideP&, const BvhReq&, void*,
                                                      const hfb_guess_out*, void*);

extern "C" {

int hfb_batch_distance_objects_device(hfb_ctx* ctx, const hfb_object_pairs* d_scene, const hfb_distance_request* req,
                                      hfb_distance_result* d_out, const hfb_guess_out* d_go, void* stream) {
  if (!ctx || !req) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (int rc = validate_query(req->q)) return fail(ctx, rc, "invalid request");
  return objects_device<0>(ctx, d_scene, req, solver_from_distance_request(*req), CollideP{0, 0}, bvh_req_of_distance(req), d_out,
                           d_go, stream);
}

int hfb_batch_collide_objects_device(hfb_ctx* ctx, const hfb_object_pairs* d_scene, const hfb_collision_request* req,
                                     hfb_contact* d_out, const hfb_guess_out* d_go, void* stream) {
  if (!ctx || !req) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  bool minus_inf;
  if (int rc = collide_prelude(ctx, req, &minus_inf)) return rc;
  if (minus_inf) {
    if (int rc = check_ready(ctx)) return rc;
    if (!d_scene || d_scene->n_pairs == 0) return HFB_OK;
    if (d_scene->n_pairs > 0xffffffffull || !d_out) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "bad buffer");
    k_clear_contacts<<<(unsigned)((d_scene->n_pairs + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(d_out, (unsigned)d_scene->n_pairs);
    ctx->stats.kernel_launches++;
    CK(cudaGetLastError());
    return HFB_OK;
  }
  CollideP C{req->security_margin, req->q.collision_distance_threshold};
  return objects_device<1>(ctx, d_scene, req, solver_from_collision_request(*req), C, bvh_req_of_collision(req), d_out, d_go, stream);
}

int hfb_batch_convex_support_device(hfb_ctx* ctx, size_t n, const uint32_t* ids, const double* dirs,
                                    int32_t* idx, double* sup, void* stream) {
  int rc;
  if ((rc = check_ready(ctx))) return rc;
  if (n == 0) return HFB_OK;
  CK(cudaSetDevice(ctx->device));
  const int threads = 256;
  unsigned blocks = (unsigned)((n + 7) / 8);
  const unsigned cap = (unsigned)ctx->num_sms * 16u;
  if (blocks > cap) blocks = cap;
  {
    KTimer kt(ctx, static_cast<cudaStream_t>(stream), 2);
    k_convex_support<<<blocks, threads, 0, static_cast<cudaStream_t>(stream)>>>(ctx->dview.cvx, ctx->dview.pool, ids, dirs, idx, sup, (unsigned)n);
  }
  ctx->stats.kernel_launches++;
  CK(cudaGetLastError());
  return HFB_OK;
}

int hfb_batch_convex_support(hfb_ctx* ctx, size_t n, const uint32_t* ids, const double* dirs, int32_t* idx,
                             double* sup) {
  int rc;
  if ((rc = check_ready(ctx))) return rc;
  if (n == 0) return HFB_OK;
  std::lock_guard<std::mutex> lk(ctx->mu);
  for (size_t i = 0; i < n; ++i)
    if (ids[i] >= ctx->arena.cvx.size()) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "convex id out of range");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->slots[0].stream;
  CK(ctx->sup_ids.reserve(n * 4));
  CK(ctx->sup_dirs.reserve(n * 24));
  CK(ctx->sup_idx.reserve(n * 4));
  CK(ctx->sup_out.reserve(n * 24));
  CK(cudaMemcpyAsync(ctx->sup_ids.p, ids, n * 4, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(ctx->sup_dirs.p, dirs, n * 24, cudaMemcpyHostToDevice, s));
  if ((rc = hfb_batch_convex_support_device(ctx, n, static_cast<uint32_t*>(ctx->sup_ids.p),
                                            static_cast<double*>(ctx->sup_dirs.p),
                                            static_cast<int32_t*>(ctx->sup_idx.p),
                                            static_cast<double*>(ctx->sup_out.p), s)))
    return rc;
  CK(cudaMemcpyAsync(idx, ctx->sup_idx.p, n * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(sup, ctx->sup_out.p, n * 24, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return HFB_OK;
}

// development aid (not in the header): phase profile of k_bvhq of the *_device entry points since the context was
// created -- clock cycles of thread 0 summed over the blocks in the BV / leaf / EPA phases, cycles, EPA phases
int hfb_debug_bvh_profile(hfb_ctx* ctx, unsigned long long out[5]) {
  if (!ctx || !out) return HFB_ERR_INVALID_ARGUMENT;
  CK(cudaSetDevice(ctx->device));
  CK(cudaDeviceSynchronize());
  unsigned long long v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (ctx->dev_slot.bvh_cnt.p) CK(cudaMemcpy(v, ctx->dev_slot.bvh_cnt.p, sizeof(v), cudaMemcpyDeviceToHost));
  for (int k = 0; k < 5; ++k) out[k] = v[3 + k];
  return HFB_OK;
}

int hfb_set_profiling(hfb_ctx* ctx, int enable) {
  if (!ctx) return HFB_ERR_INVALID_ARGUMENT;
  ctx->profiling = enable != 0;
  return HFB_OK;
}

int hfb_get_kernel_times(hfb_ctx* ctx, hfb_kernel_times* out, int reset) {
  if (!ctx || !out) return HFB_ERR_INVALID_ARGUMENT;
  CK(cudaSetDevice(ctx->device));
  CK(cudaDeviceSynchronize());
  for (auto& e : ctx->events) {
    float ms = 0;
    cudaEventElapsedTime(&ms, e.a, e.b);
    if (e.kind == 0) { ctx->ktimes.pairs_ms += ms; ctx->ktimes.pairs_launches++; }
    else if (e.kind == 1) { ctx->ktimes.epa_ms += ms; ctx->ktimes.epa_launches++; }
    else if (e.kind == 3) { ctx->ktimes.closed_ms += ms; ctx->ktimes.closed_launches++; }
    else if (e.kind == 4) { ctx->ktimes.convex_ms += ms; ctx->ktimes.convex_launches++; }
    else if (e.kind == 5) { ctx->ktimes.bvh_ms += ms; ctx->ktimes.bvh_launches++; }
    else { ctx->ktimes.other_ms += ms; ctx->ktimes.other_launches++; }
    cudaEventDestroy(e.a);
    cudaEventDestroy(e.b);
  }
  ctx->events.clear();
  *out = ctx->ktimes;
  if (reset) ctx->ktimes = hfb_kernel_times{};
  return HFB_OK;
}

int hfb_get_stats(hfb_ctx* ctx, hfb_stats* out) {
  if (!ctx || !out) return HFB_ERR_INVALID_ARGUMENT;
  CK(cudaSetDevice(ctx->device));
  CK(cudaDeviceSynchronize());
  uint64_t epa = 0;
  auto add = [&](Slot& s) -> cudaError_t {
    if (!s.counters.p) return cudaSuccess;
    unsigned v[2] = {0, 0};
    cudaError_t e = cudaMemcpy(v, s.counters.p, sizeof(v), cudaMemcpyDeviceToHost);
    epa += v[1];
    return e;
  };
  for (int k = 0; k < kSlots; ++k) CK(add(ctx->slots[k]));
  CK(add(ctx->dev_slot));
  uint64_t bvt = 0, lft = 0, wdt = 0;
  auto addb = [&](Slot& s) -> cudaError_t {
    if (!s.bvh_cnt.p) return cudaSuccess;
    unsigned long long v[3] = {0, 0, 0};
    cudaError_t e = cudaMemcpy(v, s.bvh_cnt.p, sizeof(v), cudaMemcpyDeviceToHost);
    bvt += v[0];
    lft += v[1];
    wdt += v[2];
    return e;
  };
  for (int k = 0; k < kSlots; ++k) CK(addb(ctx->slots[k]));
  CK(addb(ctx->dev_slot));
  ctx->stats.bv_tests = bvt;
  ctx->stats.leaf_tests = lft;
  ctx->stats.watchdog_trips = wdt;
  ctx->stats.epa_pairs = epa;
  *out = ctx->stats;
  return HFB_OK;
}

}  // extern "C"
