// GJK for the primitive pairs of a batch in PASSES (replaces the single kernel k_pairs<1, CAP_PRIM, MODE,
// PATH_GJKROUTE> on the GJK-routed classes; same per-pair operations: pair_gjk_begin / gjk_step / pair_gjk_end of
// hfb_pair.cuh, i.e. GJK::evaluate src/narrowphase/gjk.cpp:188-370 and the extractors narrowphase.h:589-656).
//
// Why.  In the single kernel few lanes of a warp are active per instruction and the warps stall on instruction
// fetch.  A pair needs 3 to 26 iterations, so
// a warp that keeps its 32 pairs until the last one has converged idles most of its lanes; and set-up, iteration
// and witness extraction together are ~13 000 instructions against an instruction cache of 2 000 (32 KB L1.5 per
// SM), with the warps of an SM spread all over them.  Here:
//   k_gjk_first   set-up + the first K1 iterations of every pair            -> solver state (GjkSaved) to HBM
//   k_gjk_more    K2, K3, ... more iterations of the pairs still running, which each pass compacts into a list
//                 (the last pass runs to convergence)
//   k_gjk_end     status machine + witness points of every pair: result record, or an EPA queue item
// Every kernel is small, and the later passes run full warps of the long pairs.  The state costs 424 B per pair
// and pass of HBM traffic (0.5 M pairs: 0.2 GB).
#include "hfb_gjkpass.h"

#include <cub/cub.cuh>

namespace {

// (16-byte aligned: 432 B = 27 x 16, so that the copies to and from HBM can move 16 bytes per instruction)
struct __align__(16) GjkSaved {
  GjkState g;
  GjkLoop L;
  int done;  // 1: converged in the first pass (extracted early, so that its EPA can start), 2: in a later pass, 0: running
  int _pad;
};
#define HFB_GJK_UNKNOWN_TYPES (-99)  // status of a pair whose node types no kernel knows (reported as unsupported)

struct PassArgs {
  GjkSaved* state;           // one per position of the class-sorted GJK range
  const uint32_t* in_list;   // positions still running (null: the whole range)
  const unsigned* in_count;
  uint32_t* out_list;        // positions still running after this pass (null: last pass)
  unsigned* out_count;
  int steps;
  int which;  // k_gjk_end: the pairs with this `done` value
  unsigned char* flags;  // k_gjk_first: 1 per position still running, for the ordered compaction (null: append by atomics)
};

__device__ __forceinline__ void append_running(const PassArgs& p, bool more, unsigned pos) {
  const unsigned m = __ballot_sync(0xffffffffu, more);
  if (!m) return;
  const unsigned lane = threadIdx.x & 31u;
  unsigned base = 0;
  if (lane == (unsigned)(__ffs(m) - 1)) base = atomicAdd(p.out_count, (unsigned)__popc(m));
  base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
  if (more) p.out_list[base + (unsigned)__popc(m & ((1u << lane) - 1u))] = pos;
}

__global__ void __launch_bounds__(128) k_gjk_first(const BatchArgs a, const PassArgs p) {
  const unsigned lo = *a.range_lo, hi = *a.range_hi;
  const unsigned stride = gridDim.x * blockDim.x;
  for (unsigned k0 = lo + blockIdx.x * blockDim.x; k0 < hi; k0 += stride) {  // (warp-uniform trip count)
    const unsigned k = k0 + threadIdx.x;
    bool more = false;
    if (k < hi) {
      const unsigned i = a.index_list[k];
      const PairIn in = load_pair_in<CAP_PRIM>(a, i);
      GjkSaved sv;
      sv._pad = 0;
      if (!type_known(in.s1.type) || !type_known(in.s2.type)) {
        sv.g.status = HFB_GJK_UNKNOWN_TYPES;
      } else {
        GjkSetup S;
        PairOut o;
        pair_gjk_begin<CAP_PRIM>(in, a.P, S, sv.L, sv.g, o);
        more = true;
        for (int s = 0; s < p.steps && more; ++s) more = gjk_step<1, CAP_PRIM>(S.a, S.b, S.md, a.P.gjk, sv.g, sv.L);
      }
      sv.done = more ? 0 : 1;
      p.state[k - lo] = sv;
      if (p.flags) p.flags[k - lo] = more ? 1 : 0;
    }
    if (p.out_list && !p.flags) append_running(p, more, k - lo);
  }
}

__global__ void __launch_bounds__(128) k_gjk_more(const BatchArgs a, const PassArgs p) {
  const unsigned lo = *a.range_lo;
  const unsigned n = *p.in_count;
  const unsigned stride = gridDim.x * blockDim.x;
  for (unsigned q0 = blockIdx.x * blockDim.x; q0 < n; q0 += stride) {
    const unsigned q = q0 + threadIdx.x;
    bool more = false;
    unsigned pos = 0;
    if (q < n) {
      pos = p.in_list[q];
      const unsigned i = a.index_list[lo + pos];
      const PairIn in = load_pair_in<CAP_PRIM>(a, i);
      GjkSetup S;
      make_setup<CAP_PRIM>(in, S);
      GjkSaved sv = p.state[pos];
      more = true;
      for (int s = 0; s < p.steps && more; ++s) more = gjk_step<1, CAP_PRIM>(S.a, S.b, S.md, a.P.gjk, sv.g, sv.L);
      sv.done = more ? 0 : 2;
      p.state[pos] = sv;
    }
    if (p.out_list) append_running(p, more, pos);
  }
}

template <int MODE>
__global__ void __launch_bounds__(128) k_gjk_end(const BatchArgs a, const PassArgs p) {
  const unsigned lo = *a.range_lo, hi = *a.range_hi;
  for (unsigned k = lo + blockIdx.x * blockDim.x + threadIdx.x; k < hi; k += gridDim.x * blockDim.x) {
    if (p.which >= 0 && p.state[k - lo].done != p.which) continue;  // (which < 0: every pair, one launch after the last pass)
    const unsigned i = a.index_list[k];
    const PairIn in = load_pair_in<CAP_PRIM>(a, i);
    GjkState g = p.state[k - lo].g;
    PairOut o;
    if (g.status == HFB_GJK_UNKNOWN_TYPES) {
      pair_phase1<1, CAP_PRIM, PATH_GJKROUTE>(in, a.P, o, g);  // returns at once: HFB_PATH_UNSUPPORTED
      store_result<MODE>(a, i, o);
      continue;
    }
    // what pair_gjk_begin leaves in `o` for the extractors
    o.cached_guess = (a.P.initial_guess == HFB_GUESS_CACHED) ? in.cached_guess : mk(1, 0, 0);
    o.hint0 = in.hint0;
    o.hint1 = in.hint1;
    o.iterations = 0;
    GjkSetup S;
    make_setup<CAP_PRIM>(in, S);
    if (pair_gjk_end(a.P, S, g, o)) push_epa_item(a, i, g);
    else store_result<MODE>(a, i, o);
  }
}

}  // namespace

size_t gjk_pass_state_bytes(size_t n) { return n * sizeof(GjkSaved); }
// flags (n bytes, rounded) + the temporary storage of the ordered compaction
size_t gjk_pass_select_bytes(size_t n) {
  size_t tmp = 0;
  cub::DeviceSelect::Flagged(nullptr, tmp, cub::CountingInputIterator<uint32_t>(0), (const unsigned char*)nullptr, (uint32_t*)nullptr,
                             (unsigned*)nullptr, (int)n);
  return ((n + 255) & ~(size_t)255) + tmp + 256;
}

static unsigned pass_blocks(unsigned n, int num_sms) {
  unsigned blocks = (n + 127) / 128;
  const unsigned cap = (unsigned)num_sms * 32u;
  if (blocks > cap) blocks = cap;
  return blocks ? blocks : 1u;
}
static void launch_end(const BatchArgs& a, int mode, PassArgs p, int which, unsigned blocks, cudaStream_t s) {
  p.which = which;
  if (mode == 0) k_gjk_end<0><<<blocks, 128, 0, s>>>(a, p);
  else k_gjk_end<1><<<blocks, 128, 0, s>>>(a, p);
}

// first pass + extraction of the pairs it finished (their EPA items are in the queue when this returns, so that the
// caller can start EPA on a side stream next to the remaining passes)
int gjk_passes_first(const BatchArgs& a, int mode, unsigned n, void* state, uint32_t* list_a, unsigned* counts,
                     const int* steps, int npass, int num_sms, cudaStream_t s, int* launches, void* select_ws,
                     bool extract_now) {
  if (npass < 1) return (int)cudaErrorInvalidValue;
  cudaError_t e = cudaMemsetAsync(counts, 0, (size_t)npass * sizeof(unsigned), s);
  if (e != cudaSuccess) return (int)e;
  // the survivors of the first pass in CLASS ORDER (a stable compaction of the class-sorted range) rather than in the
  // order the warps happen to finish: the second pass then meets one pair class per warp, as the first did
  unsigned char* flags = (select_ws && npass > 1) ? static_cast<unsigned char*>(select_ws) : nullptr;
  const size_t flag_bytes = ((size_t)n + 255) & ~(size_t)255;
  if (flags && (e = cudaMemsetAsync(flags, 0, flag_bytes, s)) != cudaSuccess) return (int)e;
  const unsigned blocks = pass_blocks(n, num_sms);
  PassArgs p;
  p.state = static_cast<GjkSaved*>(state);
  p.in_list = nullptr;
  p.in_count = nullptr;
  p.out_list = npass > 1 ? list_a : nullptr;
  p.out_count = counts;
  p.steps = npass > 1 ? steps[0] : 0x7fffffff;
  p.which = 0;
  p.flags = flags;
  k_gjk_first<<<blocks, 128, 0, s>>>(a, p);
  if (flags) {
    size_t tmp = gjk_pass_select_bytes(n) - flag_bytes - 256;
    if ((e = cub::DeviceSelect::Flagged(flags + flag_bytes, tmp, cub::CountingInputIterator<uint32_t>(0), flags, list_a, counts, (int)n,
                                        s)) != cudaSuccess)
      return (int)e;
    *launches += 2;  // (the select is two kernels)
  }
  // the pairs this pass finished are extracted now only when somebody waits for their EPA items (EPA on a side
  // stream next to the remaining passes); otherwise one extraction launch after the last pass takes every pair, with
  // full warps
  if (extract_now || npass < 2) {
    launch_end(a, mode, p, npass < 2 ? -1 : 1, blocks, s);
    *launches += 1;
  }
  *launches += 1;
  return (int)cudaGetLastError();
}

// the remaining passes + extraction of the pairs they finished
int gjk_passes_rest(const BatchArgs& a, int mode, unsigned n, void* state, uint32_t* list_a, uint32_t* list_b,
                    unsigned* counts, const int* steps, int npass, int num_sms, cudaStream_t s, int* launches,
                    bool first_extracted) {
  if (npass < 2) return 0;
  const unsigned blocks = pass_blocks(n, num_sms);
  PassArgs p;
  p.state = static_cast<GjkSaved*>(state);
  p.which = 0;
  p.flags = nullptr;
  for (int k = 1; k < npass; ++k) {
    const bool last = k + 1 == npass;
    p.in_list = (k & 1) ? list_a : list_b;
    p.in_count = counts + (k - 1);
    p.out_list = last ? nullptr : ((k & 1) ? list_b : list_a);
    p.out_count = counts + k;
    p.steps = last ? 0x7fffffff : steps[k];
    // the number of running pairs is only known on the device: the grid is sized for the typical survival rate of
    // a pass and strides over whatever there is
    unsigned b = blocks >> (k < 3 ? k : 3);
    if (b < (unsigned)num_sms * 2u) b = (unsigned)num_sms * 2u < blocks ? (unsigned)num_sms * 2u : blocks;
    k_gjk_more<<<b, 128, 0, s>>>(a, p);
    ++*launches;
  }
  launch_end(a, mode, p, first_extracted ? 2 : -1, blocks, s);
  ++*launches;
  return (int)cudaGetLastError();
}
