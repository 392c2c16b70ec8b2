// The C-ABI of the broadphase and of the queries built on it: the broadphase feed (hfb_scene_aabbs*, hfb_broadphase_*),
// hfb_scene_collide(_sets), and the resident environment (hfb_env_*), with the four small kernels only they launch.
// Their candidates go through the narrow phase of hfb_kernels.cu (objects_device); the pair finders are
// hfb_broadphase.cu's.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <initializer_list>
#include <limits>
#include <memory>
#include <mutex>
#include <utility>
#include <vector>

#include <cub/device/device_scan.cuh>

#include "hfb_ctx.h"
#include "hfb_broadphase.cuh"
#include "hfb_broadphase.h"
#include "hfb_validate.cuh"

// hfb_scene_collide: the colliding pairs of a scene -- object indices and contact record -- appended in no
// particular order
__global__ void __launch_bounds__(256) k_compact_scene(const hfb_contact* r, const uint32_t* pf, const uint32_t* ps, unsigned n,
                                                       unsigned* count, uint32_t* first, uint32_t* second, hfb_contact* recs,
                                                       unsigned cap) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool hit = i < n && r[i].num_contacts > 0;
  const unsigned m = __ballot_sync(0xffffffffu, hit);
  if (!m) return;
  const unsigned lane = threadIdx.x & 31u;
  unsigned pos = 0;
  if (lane == 0) pos = atomicAdd(count, (unsigned)__popc(m));
  pos = __shfl_sync(0xffffffffu, pos, 0) + (unsigned)__popc(m & ((1u << lane) - 1u));
  if (hit && pos < cap) {
    first[pos] = pf[i];
    second[pos] = ps[i];
    recs[pos] = r[i];
  }
}
// hfb_env_collide's flags: the A object of a colliding candidate gets flag 1 (every writer stores the same byte);
// count (null: not counted) gets the number of colliding candidates when no compaction counts them
__global__ void __launch_bounds__(256) k_flag_colliding(const hfb_contact* r, const uint32_t* pf, unsigned n, uint8_t* flags,
                                                        unsigned* count) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool hit = i < n && r[i].num_contacts > 0;
  if (hit) flags[pf[i]] = 1;
  if (!count) return;
  const unsigned m = __ballot_sync(0xffffffffu, hit);
  if (m && (threadIdx.x & 31u) == 0) atomicAdd(count, (unsigned)__popc(m));
}
// hfb_env_collide_device: the compacted second indices from the table [A; B] back into B (the count is on the device)
__global__ void __launch_bounds__(256) k_unbase(uint32_t* second, const unsigned* count, unsigned cap, uint32_t base) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < *count && i < cap) second[i] -= base;
}
// hfb_env_collide_configs' verdicts: the configuration (A index / links) of a colliding candidate gets 1; when no
// compaction counts them (counts null: not counted), counts[0] / counts[1] get the colliding candidates before / from
// `split` on (environment pairs, self pairs)
__global__ void __launch_bounds__(256) k_flag_configs(const hfb_contact* r, const uint32_t* pf, unsigned n, unsigned links,
                                                      unsigned split, uint8_t* verdicts, unsigned* counts) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool hit = i < n && r[i].num_contacts > 0;
  if (hit) verdicts[pf[i] / links] = 1;
  if (!counts) return;
  const unsigned me = __ballot_sync(0xffffffffu, hit && i < split), ms = __ballot_sync(0xffffffffu, hit && i >= split);
  if ((threadIdx.x & 31u) == 0) {
    if (me) atomicAdd(counts, (unsigned)__popc(me));
    if (ms) atomicAdd(counts + 1, (unsigned)__popc(ms));
  }
}

// ---- hfb_env_validate_motions: the bookkeeping between rounds (the rules: hfb_validate.cuh) --------------------------
// A round's open segments, sorted by (motion, start): w, the motion's index in the range, and the start position.  The
// per-segment passes run over `bound` entries, a host-side bound on the list's length *n (the device holds it): entries
// past it get 0 in every scanned array.  Per motion w of the range: c (earliest colliding sample), f (start of the
// earliest stuck segment), u (start of the earliest segment closed without a certificate); kValNone for none.
struct ValSegs {
  uint32_t* w;
  uint32_t* a;
};
struct ValMotions {
  uint32_t *c, *f, *u;
};
// round 0: the admitted prefix of the range's 2^d0 segments per motion (val_round0), and each motion's state
__global__ void __launch_bounds__(256) k_val_init(ValSegs sg, size_t n_seg, size_t n_range, uint64_t n_full, uint32_t partial,
                                                  uint32_t per, uint32_t len, ValMotions st, uint32_t* d_n) {
  const size_t n = n_seg > n_range ? n_seg : n_range;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (size_t)gridDim.x * blockDim.x) {
    if (t < n_seg) {
      sg.w[t] = (uint32_t)(t / per);
      sg.a[t] = (uint32_t)(t % per) * len;
    }
    if (t < n_range) {
      const uint32_t adm = val_round0_admitted(t, n_full, partial, per);
      st.c[t] = kValNone;
      st.f[t] = st.u[t] = adm < per ? adm * len : kValNone;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *d_n = (uint32_t)n_seg;
}
// per segment: its cost and whether it starts a run
__global__ void __launch_bounds__(256) k_val_cost(ValSegs sg, const uint32_t* d_n, uint32_t bound, uint32_t len,
                                                  uint32_t* cost, uint32_t* nr) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= bound) return;
  if (i >= *d_n) {
    cost[i] = nr[i] = 0;
    return;
  }
  const bool r = val_new_run(i == 0, i ? sg.w[i - 1] : 0, i ? sg.a[i - 1] : 0, sg.w[i], sg.a[i], len);
  cost[i] = val_cost(r);
  nr[i] = r;
}
// the round's totals from the inclusive scans of the costs and run flags: tot[0] admitted segments, tot[1] samples,
// tot[2] runs (the last admitted segment writes them; zeros for an empty list)
__global__ void __launch_bounds__(256) k_val_admit(const uint32_t* d_n, uint32_t bound, const uint32_t* cscan,
                                                   const uint32_t* rscan, uint32_t cap, uint32_t* tot) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, n = *d_n;
  if (i == 0 && n == 0) tot[0] = tot[1] = tot[2] = 0;
  if (i >= bound || i >= n || !val_admitted(cscan[i], cap)) return;
  if (i + 1 == n || !val_admitted(cscan[i + 1], cap)) {
    tot[0] = i + 1;
    tot[1] = cscan[i];
    tot[2] = rscan[i];
  }
}
// the round's samples (motion, position, whether a segment starts there) and the runs' offsets into them, from the
// n_adm admitted segments
__global__ void __launch_bounds__(256) k_val_samples(ValSegs sg, uint32_t n_adm, uint32_t len, const uint32_t* cscan,
                                                     const uint32_t* nr, const uint32_t* rscan, uint32_t* sw, uint32_t* sk,
                                                     uint8_t* sseg, uint32_t* off) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_adm) return;
  const uint32_t g = val_start_sample(cscan[i]), w = sg.w[i], a = sg.a[i];
  sw[g] = w;
  sk[g] = a;
  sseg[g] = 1;
  if (nr[i]) off[rscan[i] - 1] = g;
  if (i + 1 == n_adm || nr[i + 1]) {  // the run ends here: its last sample
    sw[g + 1] = w;
    sk[g + 1] = a + len;
    sseg[g + 1] = 0;
  }
  if (i + 1 == n_adm) off[rscan[i]] = cscan[i];
}
// each run's first colliding sample (certify's first_invalid) into its motion's c
__global__ void __launch_bounds__(256) k_val_collide(uint32_t n_runs, const int32_t* fi, const uint32_t* off,
                                                     const uint32_t* sw, const uint32_t* sk, ValMotions st) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_runs || fi[r] < 0) return;
  const uint32_t g = off[r] + (uint32_t)fi[r];
  atomicMin(st.c + sw[g], sk[g]);
}
// the segment rules: kids[i] = 2 for a split segment, else 0; a stuck or dropped segment's start into its motion's u,
// a stuck one's into f.  Thread 0 adds the round's unsupported records (*n_unsup) to *acc.
__global__ void __launch_bounds__(256) k_val_rules(ValSegs sg, const uint32_t* d_n, uint32_t bound, uint32_t n_adm,
                                                   bool deepest, uint32_t L, const uint32_t* cscan, const uint8_t* cert,
                                                   const double* sweep, ValMotions st, uint32_t* kids,
                                                   const unsigned* n_unsup, unsigned long long* acc) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) *acc += *n_unsup;
  if (i >= bound) return;
  if (i >= *d_n) {
    kids[i] = 0;
    return;
  }
  const uint32_t w = sg.w[i], a = sg.a[i];
  const bool admitted = i < n_adm;
  bool certified = false, finite = true;
  if (admitted) {
    const uint32_t g = val_start_sample(cscan[i]);
    certified = cert[g];
    for (uint32_t l = 0; l < L; ++l) finite = finite && sweep[(size_t)g * L + l] <= DBL_MAX;  // (NaN, +inf: not)
  }
  const ValRule rule = val_rule(admitted, certified, a, st.c[w], deepest, finite);
  if (rule == VAL_DROPPED || rule == VAL_STUCK) atomicMin(st.u + w, a);
  if (rule == VAL_STUCK) atomicMin(st.f + w, a);
  kids[i] = rule == VAL_SPLIT ? 2u : 0u;
}
// the frontier: of a split segment, the halves that start before its motion's f
__global__ void __launch_bounds__(256) k_val_keep(ValSegs sg, const uint32_t* d_n, uint32_t half, ValMotions st,
                                                  uint32_t* kids) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= *d_n || !kids[i]) return;
  const uint32_t f = st.f[sg.w[i]], a = sg.a[i];
  kids[i] = (uint32_t)val_keep(a, f) + (uint32_t)val_keep(a + half, f);
}
// the next round's list from the exclusive scan of kids, in (motion, start) order, and its length *d_n_next
__global__ void __launch_bounds__(256) k_val_compact(ValSegs sg, const uint32_t* d_n, uint32_t half, ValMotions st,
                                                     const uint32_t* kids, const uint32_t* kscan, ValSegs nx,
                                                     uint32_t* d_n_next) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, n = *d_n;
  if (i >= n) return;
  if (i + 1 == n) *d_n_next = kscan[i] + kids[i];
  if (!kids[i]) return;
  const uint32_t w = sg.w[i], a = sg.a[i], f = st.f[w];
  uint32_t p = kscan[i];
  for (uint32_t b : {a, a + half}) {
    if (!val_keep(b, f)) continue;
    nx.w[p] = w;
    nx.a[p] = b;
    ++p;
  }
}
// the outputs of hfb_env_validate_motions (each array n_motions long): the range's motions from their state
// (val_result), the others -1, 0, -1; wflag[w] = 1 for the range's colliding motions
struct ValOut {
  int8_t* status;
  double* t_valid;
  double* t_collide;
};
__global__ void __launch_bounds__(256) k_val_final(uint32_t n_motions, uint32_t m0, uint32_t n_range, uint32_t D,
                                                   ValMotions st, ValOut o, uint32_t* wflag) {
  const uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n_motions) return;
  if (m < m0 || m - m0 >= n_range) {
    o.status[m] = -1;
    o.t_valid[m] = 0.0;
    o.t_collide[m] = -1.0;
    return;
  }
  const uint32_t w = m - m0;
  val_result(st.c[w], st.u[w], D, o.status + m, o.t_valid + m, o.t_collide + m);
  if (wflag) wflag[w] = st.c[w] != kValNone;
}
// the witness samples: the range's colliding motions, in order (widx: the exclusive scan of wflag), each at its c
__global__ void __launch_bounds__(256) k_val_wsamples(uint32_t n_range, const uint32_t* wflag, const uint32_t* widx,
                                                      ValMotions st, uint32_t* sw, uint32_t* sk, uint8_t* sseg,
                                                      uint32_t* n_w) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n_range) return;
  if (w + 1 == n_range) *n_w = widx[w] + wflag[w];
  if (!wflag[w]) return;
  const uint32_t p = widx[w];
  sw[p] = w;
  sk[p] = st.c[w];
  sseg[p] = 0;
}
// the witnesses of the one-sample motions (hfb_env_collide_motions' outputs over the witness samples) to their
// motions: A indices p * L + i back to link indices
__global__ void __launch_bounds__(256) k_val_witness(uint32_t n_w, uint32_t m0, uint32_t L, const uint32_t* sw,
                                                     const int8_t* kind, const uint32_t* first, const uint32_t* second,
                                                     const hfb_contact* rec, BpMotions o) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_w || kind[p] < 0) return;
  const uint32_t m = m0 + sw[p], base = p * L;
  if (o.kind) o.kind[m] = kind[p];
  if (o.first) o.first[m] = first[p] - base;
  if (o.second) o.second[m] = kind[p] == 0 ? second[p] : second[p] - base;
  if (o.rec) o.rec[m] = rec[p];
}

extern "C" {

// ---- broadphase feed (hfb_broadphase.cuh) -----------------------------------------------------------------
int hfb_scene_aabbs(hfb_ctx* ctx, size_t n, const uint32_t* handles, const hfb_transform* tfs, double* aabbs) {
  if (!ctx || (n && (!handles || !tfs || !aabbs))) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (int rc = check_ready(ctx)) return rc;
  if (int rc = check_handles(ctx, handles, n)) return rc;
  for (size_t i = 0; i < n; ++i) {
    const double* l = ctx->local_aabbs.data() + 6 * (size_t)handles[i];
    if (!(l[0] <= l[3])) return fail(ctx, HFB_ERR_UNSUPPORTED_PAIR, "node type without a local AABB");
    object_aabb(l, l + 3, tfs[i], aabbs + 6 * i);
  }
  return HFB_OK;
}

int hfb_broadphase_pairs(size_t n, const double* aabbs, uint32_t* first, uint32_t* second, size_t capacity,
                         size_t* n_pairs) {
  if ((n && !aabbs) || !n_pairs || (capacity && (!first || !second)) || n > 0xffffffffull) return HFB_ERR_INVALID_ARGUMENT;
  *n_pairs = broadphase_pairs_host(n, aabbs, first, second, capacity);
  return HFB_OK;
}

int hfb_scene_aabbs_device(hfb_ctx* ctx, size_t n, const uint32_t* d_handles, const hfb_transform* d_tfs, double* d_aabbs,
                           void* stream) {
  if (!ctx || (n && (!d_handles || !d_tfs || !d_aabbs)) || n > 0xffffffffull) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (int rc = check_ready(ctx)) return rc;
  CK(cudaSetDevice(ctx->device));
  if (bp_scene_aabbs_launch(ctx->dview.local_aabbs, ctx->dview.nshapes, n, d_handles, d_tfs, d_aabbs,
                            static_cast<cudaStream_t>(stream)) != 0)
    return fail(ctx, HFB_ERR_CUDA, "k_scene_aabbs launch failed");
  ctx->stats.kernel_launches += n ? 1 : 0;
  return HFB_OK;
}

int hfb_broadphase_pairs_device(hfb_ctx* ctx, size_t n, const double* d_aabbs, size_t first_object, size_t num_first_objects,
                                uint32_t* d_first, uint32_t* d_second, size_t capacity, uint32_t* d_n_pairs, void* stream) {
  if (!ctx || (n && !d_aabbs) || !d_n_pairs || (capacity && (!d_first || !d_second)) || n > 0xffffffffull)
    return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  CK(cudaSetDevice(ctx->device));
  CK(ctx->bp_scratch.reserve(bp_scratch_bytes(n)));
  int nl = 0;
  if (bp_pairs_launch(n, d_aabbs, first_object, first_object + (num_first_objects < n ? num_first_objects : n), d_first, d_second,
                      capacity, d_n_pairs, ctx->bp_scratch.p, ctx->num_sms,
                      static_cast<cudaStream_t>(stream), &nl) != 0)
    return fail(ctx, HFB_ERR_CUDA, "broadphase launch failed");
  ctx->stats.kernel_launches += (uint64_t)nl;
  return HFB_OK;
}

}  // extern "C"

// The number of candidate pairs is not known in advance: find(cap, &launches) launches a pair finder that counts every
// candidate in the counter's first word (d_cnt) and stores at most `cap` in each of `lists` (4 bytes per candidate).
// find_all runs it and reads the counter's first n_words words into `words`; when the count exceeded the lists, they
// grow to fit it and it runs once more (the second sweep stores what the first counted).
template <class Find>
static int find_all(hfb_ctx* ctx, cudaStream_t s, std::initializer_list<DevBuf*> lists, const unsigned* d_cnt, Find find,
                    unsigned* words, int n_words) {
  auto lists_cap = [&]() {
    size_t c = ~(size_t)0;
    for (DevBuf* b : lists) c = b->cap / 4 < c ? b->cap / 4 : c;
    return c;
  };
  size_t cap = lists_cap();
  for (int attempt = 0; attempt < 2; ++attempt) {
    int nl = 0;
    if (find(cap, &nl) != 0) return fail(ctx, HFB_ERR_CUDA, "broadphase launch failed");
    ctx->stats.kernel_launches += (uint64_t)nl;
    CK(cudaMemcpyAsync(words, d_cnt, n_words * sizeof(unsigned), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    if (words[0] <= cap) break;
    cap = (size_t)words[0] + words[0] / 8 + 1024;
    for (DevBuf* b : lists) CK(b->reserve(cap * 4));
    cap = lists_cap();
  }
  return HFB_OK;
}
// The part hfb_scene_collide, hfb_scene_collide_sets and hfb_env_collide share, after the upload of the object table
// (d_h, d_tf: n objects): the boxes of its first n_boxes objects, the candidates (find_pairs(d_bb, pf, ps, capacity,
// d_count, &launches) launches a pair finder, all pairs counted in *d_count, at most `capacity` stored) and collide() of
// every candidate over the table, into ctx->sc_out (none when there are no candidates or under minus_inf).
// split_out (may be null): the counter's second word, which a finder may set, read with the count.  entry (may be
// null): a third candidate list the finder fills, grown with the other two.
template <class FindPairs>
static int scene_candidates(hfb_ctx* ctx, cudaStream_t s, size_t n, const uint32_t* d_h, const hfb_transform* d_tf,
                            size_t n_boxes, FindPairs find_pairs, const hfb_collision_request* req, bool minus_inf,
                            unsigned* cand_out, unsigned* split_out = nullptr, DevBuf* entry = nullptr) {
  CK(ctx->sc_bb.reserve(n_boxes * 48));
  CK(ctx->sc_cnt.reserve(16));
  double* d_bb = static_cast<double*>(ctx->sc_bb.p);
  unsigned* d_cnt = static_cast<unsigned*>(ctx->sc_cnt.p);
  if (bp_scene_aabbs_launch(ctx->dview.local_aabbs, ctx->dview.nshapes, n_boxes, d_h, d_tf, d_bb, s) != 0)
    return fail(ctx, HFB_ERR_CUDA, "k_scene_aabbs launch failed");
  ctx->stats.kernel_launches++;
  unsigned words[2] = {0, 0};
  auto find = [&](size_t cap, int* nl) {
    return find_pairs(d_bb, static_cast<uint32_t*>(ctx->sc_pf.p), static_cast<uint32_t*>(ctx->sc_ps.p), cap, d_cnt, nl);
  };
  const int n_words = split_out ? 2 : 1;
  if (int rc = entry ? find_all(ctx, s, {&ctx->sc_pf, &ctx->sc_ps, entry}, d_cnt, find, words, n_words)
                     : find_all(ctx, s, {&ctx->sc_pf, &ctx->sc_ps}, d_cnt, find, words, n_words))
    return rc;
  const unsigned cand = words[0];
  if (split_out) *split_out = words[1];
  *cand_out = cand;
  if (cand == 0 || minus_inf) return HFB_OK;  // collision.cpp:73-76: no contacts under security_margin == -inf
  CK(ctx->sc_out.reserve((size_t)cand * sizeof(hfb_contact)));
  hfb_object_pairs sc;
  sc.n_objects = n;
  sc.object_handles = d_h;
  sc.object_tfs = d_tf;
  sc.n_pairs = cand;
  sc.first = static_cast<const uint32_t*>(ctx->sc_pf.p);
  sc.second = static_cast<const uint32_t*>(ctx->sc_ps.p);
  CollideP C{req->security_margin, req->q.collision_distance_threshold};
  return objects_device<1>(ctx, &sc, req, solver_from_collision_request(*req), C, bvh_req_of_collision(req), ctx->sc_out.p,
                           nullptr, s);
}

// Where a query's outputs go, on stream s.  Host form (dev false): the caller's outputs are host memory; device results
// are downloaded, and the counts the host knows are written once finish() has waited for the downloads.  Device form:
// they are device memory, written in stream order, and finish() does not wait.
struct QueryOut {
  cudaStream_t s;
  bool dev;
  bool pending = false;                                // host form: downloads not waited for yet
  std::vector<std::pair<uint32_t*, unsigned>> counts;  // host form: written by finish()

  cudaError_t zero(void* p, size_t bytes) {
    if (!p || !bytes) return cudaSuccess;
    if (dev) return cudaMemsetAsync(p, 0, bytes, s);
    std::memset(p, 0, bytes);
    return cudaSuccess;
  }
  // `bytes` of device memory at src into dst
  cudaError_t copy(void* dst, const void* src, size_t bytes) {
    if (!dst) return cudaSuccess;
    pending |= !dev;
    return cudaMemcpyAsync(dst, src, bytes, dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, s);
  }
  // the first `width` bytes of each of n records of `pitch` bytes at src (a field, such as the records' min_distance),
  // packed into dst
  cudaError_t copy_field(void* dst, const void* src, size_t width, size_t pitch, size_t n) {
    if (!dst) return cudaSuccess;
    pending |= !dev;
    return cudaMemcpy2DAsync(dst, width, src, pitch, width, n, dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, s);
  }
  // a count the host knows; the device form copies it from d_v when the device holds it there, else from the host
  // (pageable source: staged before the call returns)
  cudaError_t count(uint32_t* dst, unsigned v, const unsigned* d_v = nullptr) {
    if (!dst) return cudaSuccess;
    if (!dev) {
      counts.emplace_back(dst, v);
      return cudaSuccess;
    }
    if (d_v) return cudaMemcpyAsync(dst, d_v, sizeof(unsigned), cudaMemcpyDeviceToDevice, s);
    return cudaMemcpyAsync(dst, &v, sizeof(unsigned), cudaMemcpyHostToDevice, s);
  }
  cudaError_t finish() {
    if (dev) return cudaGetLastError();
    if (pending) {
      if (cudaError_t e = cudaStreamSynchronize(s)) return e;
      pending = false;
    }
    for (const auto& c : counts) *c.first = c.second;
    counts.clear();
    return cudaSuccess;
  }
};

// The colliding ones of scene_candidates' `cand` candidates: compacted (pairs and records, at most out->capacity; not
// when out->flags is set and capacity is 0) and flagged per A object (out->flags, n_flags of them, when set), then
// o.finish().  `second_base` is subtracted from the second indices.
static int scene_output(hfb_ctx* ctx, unsigned cand, uint32_t second_base, const hfb_env_out* out, size_t n_flags,
                        QueryOut& o) {
  const cudaStream_t s = o.s;
  unsigned* d_cnt = static_cast<unsigned*>(ctx->sc_cnt.p);
  const hfb_contact* recs = static_cast<const hfb_contact*>(ctx->sc_out.p);
  const uint32_t* pf = static_cast<const uint32_t*>(ctx->sc_pf.p);
  const bool compact = !out->flags || out->capacity;
  CK(cudaMemsetAsync(d_cnt + 1, 0, sizeof(unsigned), s));
  uint8_t* flags = out->flags;
  if (flags) {
    if (!o.dev) {  // (the host form stages its outputs in the scratch)
      CK(ctx->sc_flags.reserve(n_flags));
      flags = static_cast<uint8_t*>(ctx->sc_flags.p);
    }
    CK(cudaMemsetAsync(flags, 0, n_flags, s));
    k_flag_colliding<<<(cand + 255) / 256, 256, 0, s>>>(recs, pf, cand, flags, compact ? nullptr : d_cnt + 1);
    ctx->stats.kernel_launches++;
  }
  uint32_t *first = out->first, *second = out->second;
  hfb_contact* contacts = out->contacts;
  if (compact) {
    if (!o.dev) {
      CK(ctx->sc_f.reserve((size_t)out->capacity * 4 + 4));
      CK(ctx->sc_s.reserve((size_t)out->capacity * 4 + 4));
      CK(ctx->sc_rec.reserve((size_t)out->capacity * sizeof(hfb_contact) + 8));
      first = static_cast<uint32_t*>(ctx->sc_f.p);
      second = static_cast<uint32_t*>(ctx->sc_s.p);
      contacts = static_cast<hfb_contact*>(ctx->sc_rec.p);
    }
    k_compact_scene<<<(cand + 255) / 256, 256, 0, s>>>(recs, pf, static_cast<const uint32_t*>(ctx->sc_ps.p), cand, d_cnt + 1,
                                                        first, second, contacts, out->capacity);
    ctx->stats.kernel_launches++;
  }
  if (o.dev) {
    const unsigned most = cand < out->capacity ? cand : out->capacity;
    if (compact && second_base && most) {
      k_unbase<<<(most + 255) / 256, 256, 0, s>>>(out->second, d_cnt + 1, out->capacity, second_base);
      ctx->stats.kernel_launches++;
    }
    CK(o.copy(out->n_colliding, d_cnt + 1, sizeof(unsigned)));
    CK(o.finish());
    return HFB_OK;
  }
  // the host form sizes the download by the count
  unsigned hits = 0;
  CK(cudaMemcpyAsync(&hits, d_cnt + 1, sizeof(unsigned), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(o.count(out->n_colliding, hits));
  const unsigned kept = !compact ? 0u : hits < out->capacity ? hits : out->capacity;
  if (kept) {
    CK(o.copy(out->first, first, (size_t)kept * 4));
    CK(o.copy(out->second, second, (size_t)kept * 4));
    CK(o.copy(out->contacts, contacts, (size_t)kept * sizeof(hfb_contact)));
  }
  if (flags) CK(o.copy(out->flags, flags, n_flags));
  CK(o.finish());
  if (second_base)
    for (unsigned k = 0; k < kept; ++k) out->second[k] -= second_base;
  return HFB_OK;
}

// hfb_scene_collide and hfb_scene_collide_sets: boxes of the whole table, candidates, narrow phase, compaction and
// download
template <class FindPairs>
static int scene_collide_table(hfb_ctx* ctx, cudaStream_t s, size_t n, const uint32_t* d_h, const hfb_transform* d_tf,
                               FindPairs find_pairs, uint32_t second_base, const hfb_collision_request* req, bool minus_inf,
                               const hfb_scene_contacts* out) {
  unsigned cand = 0;
  if (int rc = scene_candidates(ctx, s, n, d_h, d_tf, n, find_pairs, req, minus_inf, &cand)) return rc;
  if (out->n_candidates) *out->n_candidates = cand;
  if (cand == 0 || minus_inf) return HFB_OK;
  const hfb_env_out eo{out->first, out->second, out->contacts, out->capacity, out->n_colliding, nullptr, nullptr};
  QueryOut o{s, false};
  return scene_output(ctx, cand, second_base, &eo, 0, o);
}

extern "C" {

// Broadphase + narrow phase of a scene in one call, everything on the device between the upload of the poses and the
// download of the colliding pairs: the batched form of BroadPhaseCollisionManager::collide(callback) with the default
// collision callback (broadphase/default_broadphase_callbacks.h:69-130: collide() of every candidate pair, contacts
// collected).
int hfb_scene_collide(hfb_ctx* ctx, size_t n, const uint32_t* handles, const hfb_transform* tfs, size_t first_object,
                      size_t num_first_objects, const hfb_collision_request* req, const hfb_scene_contacts* out) {
  if (!ctx || !req || !out || (n && (!handles || !tfs))) return HFB_ERR_INVALID_ARGUMENT;
  if (out->capacity && (!out->first || !out->second || !out->contacts)) return HFB_ERR_INVALID_ARGUMENT;
  std::unique_lock<std::mutex> lk(ctx->mu);
  bool minus_inf;
  if (int rc = collide_prelude(ctx, req, &minus_inf)) return rc;
  if (int rc = check_ready(ctx)) return rc;
  if (n > 0xffffffffull) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "scene too large");
  if (int rc = check_handles(ctx, handles, n)) return rc;
  if (out->n_candidates) *out->n_candidates = 0;
  if (out->n_colliding) *out->n_colliding = 0;
  if (n < 2) return HFB_OK;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->slots[0].stream;
  if (int rc = after_device_calls(ctx, s)) return rc;
  CK(ctx->obj_h.reserve(n * 4 + 4));
  CK(ctx->obj_tf.reserve(n * sizeof(hfb_transform) + 8));
  CK(ctx->bp_scratch.reserve(bp_scratch_bytes(n)));
  CK(cudaMemcpyAsync(ctx->obj_h.p, handles, n * 4, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(ctx->obj_tf.p, tfs, n * sizeof(hfb_transform), cudaMemcpyHostToDevice, s));
  const size_t i_hi = first_object + (num_first_objects < n ? num_first_objects : n);
  auto find = [&](const double* d_bb, uint32_t* pf, uint32_t* ps, size_t cap, unsigned* d_cnt, int* nl) {
    return bp_pairs_launch(n, d_bb, first_object, i_hi, pf, ps, cap, d_cnt, ctx->bp_scratch.p, ctx->num_sms, s, nl);
  };
  return scene_collide_table(ctx, s, n, static_cast<const uint32_t*>(ctx->obj_h.p),
                             static_cast<const hfb_transform*>(ctx->obj_tf.p), find, 0u, req, minus_inf, out);
}

// ---- broadphase between two sets: collide(other_manager, callback) / collide(obj, callback) --------------------
// (broadphase/broadphase_collision_manager.h:94-118; grid over B only: hfb_broadphase.cuh)
int hfb_broadphase_cross_pairs(size_t n_a, const double* aabbs_a, size_t n_b, const double* aabbs_b, uint32_t* first,
                               uint32_t* second, size_t capacity, size_t* n_pairs) {
  if ((n_a && !aabbs_a) || (n_b && !aabbs_b) || !n_pairs || (capacity && (!first || !second)) || n_a > 0xffffffffull ||
      n_b > 0xffffffffull)
    return HFB_ERR_INVALID_ARGUMENT;
  *n_pairs = broadphase_cross_pairs_host(n_a, aabbs_a, n_b, aabbs_b, first, second, capacity);
  return HFB_OK;
}

// the self candidates of configurations: collide(callback) over one configuration's objects with a callback that
// keeps only the template's pairs (broadphase_collision_manager.h:104-106), for every configuration of the range
int hfb_broadphase_config_pairs(size_t n_a, const double* aabbs, size_t links_per_config, size_t n_self_pairs,
                                const uint32_t* self_pairs, size_t first_config, size_t num_configs, uint32_t* first,
                                uint32_t* second, size_t capacity, size_t* n_pairs) {
  if ((n_a && !aabbs) || !n_pairs || (capacity && (!first || !second)) || (n_self_pairs && !self_pairs) ||
      n_a > 0xffffffffull || n_self_pairs > 0xffffffffull)
    return HFB_ERR_INVALID_ARGUMENT;
  const size_t L = links_per_config;
  if (config_range_error(n_a, L, first_config, num_configs, n_self_pairs, self_pairs)) return HFB_ERR_INVALID_ARGUMENT;
  *n_pairs = broadphase_config_pairs_host(aabbs, (uint32_t)L, self_pairs, (uint32_t)n_self_pairs, (uint32_t)first_config,
                                          num_configs, first, second, capacity);
  return HFB_OK;
}

// the self pairs whose distance() hfb_env_distance_configs runs (config_dist_pair), for every configuration of the range
int hfb_broadphase_config_distance_pairs(size_t n_a, const double* aabbs, size_t links_per_config, size_t n_self_pairs,
                                         const uint32_t* self_pairs, size_t first_config, size_t num_configs,
                                         double max_distance, uint32_t* first, uint32_t* second, size_t capacity,
                                         size_t* n_pairs) {
  if ((n_a && !aabbs) || !n_pairs || (capacity && (!first || !second)) || (n_self_pairs && !self_pairs) ||
      n_a > 0xffffffffull || n_self_pairs > 0xffffffffull || !(max_distance >= 0))
    return HFB_ERR_INVALID_ARGUMENT;
  const size_t L = links_per_config;
  if (config_range_error(n_a, L, first_config, num_configs, n_self_pairs, self_pairs)) return HFB_ERR_INVALID_ARGUMENT;
  *n_pairs = broadphase_config_distance_pairs_host(aabbs, (uint32_t)L, self_pairs, (uint32_t)n_self_pairs,
                                                   (uint32_t)first_config, num_configs, max_distance, first, second,
                                                   capacity);
  return HFB_OK;
}

// the self pairs whose collide() hfb_env_certify_motions runs (sweep_pair), for the configurations of the motion range,
// with the sides sweep_sides gives them
int hfb_broadphase_sweep_pairs(size_t n_a, const double* aabbs, const double* sweep, size_t links_per_config,
                               size_t n_self_pairs, const uint32_t* self_pairs, size_t n_motions,
                               const uint32_t* motion_offsets, size_t first_motion, size_t num_motions, uint32_t* first,
                               uint32_t* second, size_t capacity, size_t* n_pairs) {
  if ((n_a && (!aabbs || !sweep)) || !n_pairs || (capacity && (!first || !second)) || (n_self_pairs && !self_pairs) ||
      !motion_offsets || n_a > 0xffffffffull || n_self_pairs > 0xffffffffull || n_motions > 0xffffffffull)
    return HFB_ERR_INVALID_ARGUMENT;
  const size_t L = links_per_config;
  const uint32_t* off = motion_offsets;
  if (L == 0 || n_a % L || motion_offsets_error(n_motions, off) || off[n_motions] != n_a / L ||
      first_motion > n_motions || num_motions > n_motions - first_motion || config_template_error(L, n_self_pairs, self_pairs))
    return HFB_ERR_INVALID_ARGUMENT;
  std::vector<double> sides(2 * n_a, std::numeric_limits<double>::quiet_NaN());
  for (size_t m = first_motion; m < first_motion + num_motions; ++m)
    for (size_t i = (size_t)off[m] * L; i < (size_t)off[m + 1] * L; ++i)
      sweep_sides(sweep, i, L, off[m], off[m + 1], &sides[2 * i], &sides[2 * i + 1]);
  const size_t g0 = off[first_motion], ng = off[first_motion + num_motions] - g0;
  size_t count = 0;
  for (size_t t = 0; t < ng * n_self_pairs; ++t) {
    uint32_t a, b;
    if (!sweep_pair(aabbs, sides.data(), (uint32_t)L, self_pairs, (uint32_t)n_self_pairs, (uint32_t)g0, t, &a, &b))
      continue;
    if (count < capacity) {
      first[count] = a;
      second[count] = b;
    }
    ++count;
  }
  *n_pairs = count;
  return HFB_OK;
}

int hfb_broadphase_cross_pairs_device(hfb_ctx* ctx, size_t n_a, const double* d_aabbs_a, size_t first_a, size_t num_a,
                                      size_t n_b, const double* d_aabbs_b, uint32_t* d_first, uint32_t* d_second,
                                      size_t capacity, uint32_t* d_n_pairs, void* stream) {
  if (!ctx || (n_a && !d_aabbs_a) || (n_b && !d_aabbs_b) || !d_n_pairs || (capacity && (!d_first || !d_second)) ||
      n_a > 0xffffffffull || n_b > 0xffffffffull)
    return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  CK(cudaSetDevice(ctx->device));
  CK(ctx->bp_scratch.reserve(bp_cross_scratch_bytes(n_a, n_b)));
  int nl = 0;
  const size_t a_hi = first_a + (num_a < n_a ? num_a : n_a);
  if (bp_cross_pairs_launch(n_a, d_aabbs_a, first_a, a_hi, n_b, d_aabbs_b, d_first, d_second, 0u, capacity, d_n_pairs,
                            ctx->bp_scratch.p, ctx->num_sms, static_cast<cudaStream_t>(stream), &nl) != 0)
    return fail(ctx, HFB_ERR_CUDA, "cross broadphase launch failed");
  ctx->stats.kernel_launches += (uint64_t)nl;
  return HFB_OK;
}

// hfb_scene_collide for two sets: the object table on the device is [A; B], so the candidates are (i, n_a + j) there
// and the narrow phase and the compaction are hfb_scene_collide's own; `second` is turned back into an index in B
// after the download
int hfb_scene_collide_sets(hfb_ctx* ctx, size_t n_a, const uint32_t* handles_a, const hfb_transform* tfs_a, size_t n_b,
                           const uint32_t* handles_b, const hfb_transform* tfs_b, size_t first_a, size_t num_a,
                           const hfb_collision_request* req, const hfb_scene_contacts* out) {
  if (!ctx || !req || !out || (n_a && (!handles_a || !tfs_a)) || (n_b && (!handles_b || !tfs_b)))
    return HFB_ERR_INVALID_ARGUMENT;
  if (out->capacity && (!out->first || !out->second || !out->contacts)) return HFB_ERR_INVALID_ARGUMENT;
  std::unique_lock<std::mutex> lk(ctx->mu);
  bool minus_inf;
  if (int rc = collide_prelude(ctx, req, &minus_inf)) return rc;
  if (int rc = check_ready(ctx)) return rc;
  if (n_a > 0xffffffffull || n_b > 0xffffffffull || n_a + n_b > 0xffffffffull)
    return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "scene too large");
  if (int rc = check_handles(ctx, handles_a, n_a)) return rc;
  if (int rc = check_handles(ctx, handles_b, n_b)) return rc;
  if (out->n_candidates) *out->n_candidates = 0;
  if (out->n_colliding) *out->n_colliding = 0;
  if (n_a == 0 || n_b == 0) return HFB_OK;
  const size_t n = n_a + n_b;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->slots[0].stream;
  if (int rc = after_device_calls(ctx, s)) return rc;
  CK(ctx->obj_h.reserve(n * 4 + 4));
  CK(ctx->obj_tf.reserve(n * sizeof(hfb_transform) + 8));
  CK(ctx->bp_scratch.reserve(bp_cross_scratch_bytes(n_a, n_b)));
  uint32_t* d_h = static_cast<uint32_t*>(ctx->obj_h.p);
  hfb_transform* d_tf = static_cast<hfb_transform*>(ctx->obj_tf.p);
  CK(cudaMemcpyAsync(d_h, handles_a, n_a * 4, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(d_h + n_a, handles_b, n_b * 4, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(d_tf, tfs_a, n_a * sizeof(hfb_transform), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(d_tf + n_a, tfs_b, n_b * sizeof(hfb_transform), cudaMemcpyHostToDevice, s));
  const size_t a_hi = first_a + (num_a < n_a ? num_a : n_a);
  auto find = [&](const double* d_bb, uint32_t* pf, uint32_t* ps, size_t cap, unsigned* d_cnt, int* nl) {
    return bp_cross_pairs_launch(n_a, d_bb, first_a, a_hi, n_b, d_bb + 6 * n_a, pf, ps, (uint32_t)n_a, cap, d_cnt,
                                 ctx->bp_scratch.p, ctx->num_sms, s, nl);
  };
  return scene_collide_table(ctx, s, n, d_h, d_tf, find, (uint32_t)n_a, req, minus_inf, out);
}

}  // extern "C"

// ---- resident environment (hfb_env): set B's table, boxes and cross grid kept on the device ----------------------
// an env of this context whose B is still valid: the geometry was not cleared since its creation, and after a commit
// B's handles are checked again (in range, not released)
static int env_ready(hfb_ctx* ctx, hfb_env* e) {
  if (std::find(ctx->envs.begin(), ctx->envs.end(), e) == ctx->envs.end())
    return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "not an environment of this context");
  if (e->clears != ctx->clears)
    return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "the geometry was cleared since the environment was created (hfb_geom_clear)");
  if (int rc = check_ready(ctx)) return rc;
  if (e->commits != ctx->commits) {
    if (int rc = check_handles(ctx, e->handles.data(), e->n_b)) return rc;
    for (uint32_t h : e->handles)
      if (ctx->arena.shapes[h].type == 0) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "a shape of the environment was released");
    e->commits = ctx->commits;
  }
  return HFB_OK;
}
// at least n_a free slots in front of B in the env's table; B moves (device to device) when the table regrows
static int env_make_room(hfb_ctx* ctx, hfb_env* e, size_t n_a, cudaStream_t s) {
  if (n_a <= e->head) return HFB_OK;
  const size_t head = n_a + n_a / 4;
  DevBuf h, tf;
  cudaError_t err = h.reserve((head + e->n_b) * 4);
  if (err == cudaSuccess) err = tf.reserve((head + e->n_b) * sizeof(hfb_transform));
  if (err == cudaSuccess)
    err = cudaMemcpyAsync(static_cast<uint32_t*>(h.p) + head, static_cast<uint32_t*>(e->h.p) + e->head, e->n_b * 4,
                          cudaMemcpyDeviceToDevice, s);
  if (err == cudaSuccess)
    err = cudaMemcpyAsync(static_cast<hfb_transform*>(tf.p) + head, static_cast<hfb_transform*>(e->tf.p) + e->head,
                          e->n_b * sizeof(hfb_transform), cudaMemcpyDeviceToDevice, s);
  if (err == cudaSuccess) err = cudaStreamSynchronize(s);
  if (err != cudaSuccess) return cuda_fail(ctx, err, "environment table");
  e->h = std::move(h);
  e->tf = std::move(tf);
  e->head = head;
  return HFB_OK;
}
// the cross grid over B's boxes (scratch: the context's bp_scratch) and B's reach
static int env_build(hfb_ctx* ctx, hfb_env* e, cudaStream_t s) {
  CK(ctx->bp_scratch.reserve(bp_cross_scratch_bytes(0, e->n_b)));
  CK(e->reach.reserve(48));
  int nl = 0;
  if (bp_cross_build_launch(e->n_b, static_cast<const double*>(e->bb.p), bp_cross_grid_carve(e->grid.p, e->n_b),
                            ctx->bp_scratch.p, s, &nl) != 0)
    return fail(ctx, HFB_ERR_CUDA, "cross grid launch failed");
  if (bp_dist_reach_launch(e->n_b, static_cast<const double*>(e->bb.p), static_cast<unsigned long long*>(e->reach.p),
                           ctx->num_sms, s, &nl) != 0)
    return fail(ctx, HFB_ERR_CUDA, "k_dist_reach launch failed");
  ctx->stats.kernel_launches += (uint64_t)nl;
  return HFB_OK;
}
// the configurations of a query: A is configurations of `links` objects each, the range is [g0, g0 + ng), and the
// template lists the n self pairs (link i, link j) of a configuration
struct ConfigTpl {
  size_t links, n;
  const uint32_t* pairs;
  size_t g0, ng;
};

// The queries of an env, each run in env_call's frame: check() is the query's own check of the request, under the
// lock; zero(o) zeroes its outputs; empty(): nothing to compute, the outputs stay zero; run(o): the query of A
// (already in the table in front of B) against the env, then its outputs and o.finish().

// hfb_env_collide: boxes of A, the candidates against the built grid, the narrow phase, then the outputs
struct EnvCollide {
  const hfb_collision_request* req;
  const hfb_env_out* out;
  size_t first_a, num_a;
  bool minus_inf = false;

  const ConfigTpl* tpl() const { return nullptr; }
  int check(hfb_ctx* ctx) { return collide_prelude(ctx, req, &minus_inf); }
  int zero(hfb_ctx* ctx, QueryOut& o, size_t n_a) const {
    CK(o.zero(out->n_candidates, sizeof(uint32_t)));
    CK(o.zero(out->n_colliding, sizeof(uint32_t)));
    CK(o.zero(out->flags, n_a));
    return HFB_OK;
  }
  bool empty(const hfb_env* e, size_t n_a) const { return n_a == 0 || e->n_b == 0; }
  int run(hfb_ctx* ctx, hfb_env* e, size_t n_a, QueryOut& o) const {
    const cudaStream_t s = o.s;
    const size_t n_b = e->n_b, a_hi = first_a + (num_a < n_a ? num_a : n_a);
    const BpCrossGrid g = bp_cross_grid_carve(e->grid.p, n_b);
    const double* bb_b = static_cast<const double*>(e->bb.p);
    CK(ctx->bp_scratch.reserve(bp_cross_scratch_bytes(n_a, n_b)));
    auto find = [&](const double* d_bb, uint32_t* pf, uint32_t* ps, size_t cap, unsigned* d_cnt, int* nl) {
      if (int rc = bp_cross_query_reset(g, d_cnt, s)) return rc;
      return bp_cross_query_launch(n_a, d_bb, first_a, a_hi, n_b, bb_b, g, pf, ps, (uint32_t)n_a, cap, d_cnt,
                                   ctx->bp_scratch.p, ctx->num_sms, s, nl);
    };
    const size_t off = e->head - n_a;
    unsigned cand = 0;
    if (int rc = scene_candidates(ctx, s, n_a + n_b, static_cast<const uint32_t*>(e->h.p) + off,
                                  static_cast<const hfb_transform*>(e->tf.p) + off, n_a, find, req, minus_inf, &cand))
      return rc;
    CK(o.count(out->n_candidates, cand, static_cast<const unsigned*>(ctx->sc_cnt.p)));
    if (cand == 0 || minus_inf) {
      CK(o.finish());
      return HFB_OK;
    }
    return scene_output(ctx, cand, (uint32_t)n_a, out, n_a, o);
  }
};

static bool contacts_ok(const hfb_scene_contacts& o) { return !o.capacity || (o.first && o.second && o.contacts); }

// The outputs of hfb_env_collide_configs from the `cand` candidates, the environment pairs before `split`, the self
// pairs from there on: verdicts per configuration, and each kind compacted into its own outputs with its own counter
// (sc_cnt[1], sc_cnt[2]), then o.finish(), as in scene_output.
static int configs_output(hfb_ctx* ctx, unsigned cand, unsigned split, uint32_t second_base, size_t links,
                          size_t n_configs, const hfb_configs_out* out, QueryOut& o) {
  const cudaStream_t s = o.s;
  unsigned* d_cnt = static_cast<unsigned*>(ctx->sc_cnt.p);
  const hfb_contact* recs = static_cast<const hfb_contact*>(ctx->sc_out.p);
  const uint32_t* pf = static_cast<const uint32_t*>(ctx->sc_pf.p);
  const uint32_t* ps = static_cast<const uint32_t*>(ctx->sc_ps.p);
  const bool compact = !out->verdicts || out->env.capacity || out->self.capacity;
  CK(cudaMemsetAsync(d_cnt + 1, 0, 2 * sizeof(unsigned), s));
  uint8_t* verdicts = out->verdicts;
  if (verdicts) {
    if (!o.dev) {  // (the host form stages its outputs in the scratch)
      CK(ctx->sc_flags.reserve(n_configs));
      verdicts = static_cast<uint8_t*>(ctx->sc_flags.p);
    }
    CK(cudaMemsetAsync(verdicts, 0, n_configs, s));
    k_flag_configs<<<(cand + 255) / 256, 256, 0, s>>>(recs, pf, cand, (unsigned)links, split, verdicts,
                                                       compact ? nullptr : d_cnt + 1);
    ctx->stats.kernel_launches++;
  }
  const hfb_scene_contacts* kinds[2] = {&out->env, &out->self};
  const unsigned lo[2] = {0, split}, num[2] = {split, cand - split};
  uint32_t *first[2], *second[2];
  hfb_contact* contacts[2];
  if (!o.dev) {  // both kinds staged in one set of buffers, the self pairs after the environment's
    const size_t total = (size_t)out->env.capacity + out->self.capacity;
    CK(ctx->sc_f.reserve(total * 4 + 4));
    CK(ctx->sc_s.reserve(total * 4 + 4));
    CK(ctx->sc_rec.reserve(total * sizeof(hfb_contact) + 8));
  }
  for (int k = 0; k < 2; ++k) {
    const size_t at = k ? out->env.capacity : 0;
    first[k] = o.dev ? kinds[k]->first : static_cast<uint32_t*>(ctx->sc_f.p) + at;
    second[k] = o.dev ? kinds[k]->second : static_cast<uint32_t*>(ctx->sc_s.p) + at;
    contacts[k] = o.dev ? kinds[k]->contacts : static_cast<hfb_contact*>(ctx->sc_rec.p) + at;
    if (!compact || num[k] == 0) continue;
    k_compact_scene<<<(num[k] + 255) / 256, 256, 0, s>>>(recs + lo[k], pf + lo[k], ps + lo[k], num[k], d_cnt + 1 + k,
                                                          first[k], second[k], contacts[k], kinds[k]->capacity);
    ctx->stats.kernel_launches++;
  }
  if (o.dev) {
    const unsigned most = split < out->env.capacity ? split : out->env.capacity;
    if (compact && most) {  // (only the environment's second indices are in B)
      k_unbase<<<(most + 255) / 256, 256, 0, s>>>(out->env.second, d_cnt + 1, out->env.capacity, second_base);
      ctx->stats.kernel_launches++;
    }
    for (int k = 0; k < 2; ++k) CK(o.copy(kinds[k]->n_colliding, d_cnt + 1 + k, sizeof(unsigned)));
    CK(o.finish());
    return HFB_OK;
  }
  // the host form sizes the downloads by the counts
  unsigned hits[2] = {0, 0}, kept[2];
  CK(cudaMemcpyAsync(hits, d_cnt + 1, 2 * sizeof(unsigned), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  for (int k = 0; k < 2; ++k) {
    CK(o.count(kinds[k]->n_colliding, hits[k]));
    kept[k] = !compact ? 0u : hits[k] < kinds[k]->capacity ? hits[k] : kinds[k]->capacity;
    if (!kept[k]) continue;
    CK(o.copy(kinds[k]->first, first[k], (size_t)kept[k] * 4));
    CK(o.copy(kinds[k]->second, second[k], (size_t)kept[k] * 4));
    CK(o.copy(kinds[k]->contacts, contacts[k], (size_t)kept[k] * sizeof(hfb_contact)));
  }
  if (verdicts) CK(o.copy(out->verdicts, verdicts, n_configs));
  CK(o.finish());
  for (unsigned k = 0; k < kept[0]; ++k) out->env.second[k] -= second_base;
  return HFB_OK;
}

// The candidates of a configurations query (the template in ctx->sc_tpl) and their collide() records in ctx->sc_out:
// one candidate list -- the environment pairs against the built grid, then, after the split is noted in the counter's
// second word, the self pairs appended to it -- and one narrow phase over the table [A; B].  entries: each self pair's
// template entry in ctx->sc_f, at its position in the list.
//
// The general form: cross_boxes(d_bb, &boxes, &launches) gives the A boxes the grid query runs on (it may launch the
// pass that makes them), and self_pairs(d_bb, pf, ps, cap, d_cnt, &launches) appends the self pairs; `entry` (may be
// null) is a third candidate list, grown with the other two.
template <class CrossBoxes, class SelfPairs>
static int configs_candidates(hfb_ctx* ctx, hfb_env* e, size_t n_a, const ConfigTpl& t, const hfb_collision_request* req,
                              bool minus_inf, DevBuf* entry, cudaStream_t s, unsigned* cand, unsigned* split,
                              CrossBoxes cross_boxes, SelfPairs self_pairs) {
  const size_t n_b = e->n_b, links = t.links, g0 = t.g0, ng = t.ng;
  const size_t a_lo = g0 * links, a_hi = (g0 + ng) * links;
  const BpCrossGrid g = bp_cross_grid_carve(e->grid.p, n_b);
  const double* bb_b = static_cast<const double*>(e->bb.p);
  CK(ctx->bp_scratch.reserve(bp_cross_scratch_bytes(n_a, n_b)));
  auto find = [&](const double* d_bb, uint32_t* pf, uint32_t* ps, size_t cap, unsigned* d_cnt, int* nl) {
    const double* d_qb = nullptr;
    int rc = cross_boxes(d_bb, &d_qb, nl);
    if (rc) return rc;
    if (n_b) {
      rc = bp_cross_query_reset(g, d_cnt, s);
      if (!rc)
        rc = bp_cross_query_launch(n_a, d_qb, a_lo, a_hi, n_b, bb_b, g, pf, ps, (uint32_t)n_a, cap, d_cnt,
                                   ctx->bp_scratch.p, ctx->num_sms, s, nl);
    } else {
      rc = (int)cudaMemsetAsync(d_cnt, 0, sizeof(unsigned), s);
    }
    if (!rc) rc = (int)cudaMemcpyAsync(d_cnt + 1, d_cnt, sizeof(unsigned), cudaMemcpyDeviceToDevice, s);
    if (!rc) rc = self_pairs(d_bb, pf, ps, cap, d_cnt, nl);
    return rc;
  };
  const size_t off = e->head - n_a;
  return scene_candidates(ctx, s, n_a + n_b, static_cast<const uint32_t*>(e->h.p) + off,
                          static_cast<const hfb_transform*>(e->tf.p) + off, n_a, find, req, minus_inf, cand, split, entry);
}
static int configs_candidates(hfb_ctx* ctx, hfb_env* e, size_t n_a, const ConfigTpl& t, const hfb_collision_request* req,
                              bool minus_inf, bool entries, cudaStream_t s, unsigned* cand, unsigned* split) {
  const uint32_t* d_tpl = static_cast<const uint32_t*>(ctx->sc_tpl.p);
  return configs_candidates(
      ctx, e, n_a, t, req, minus_inf, entries ? &ctx->sc_f : nullptr, s, cand, split,
      [](const double* d_bb, const double** d_qb, int*) {
        *d_qb = d_bb;
        return 0;
      },
      [&](const double* d_bb, uint32_t* pf, uint32_t* ps, size_t cap, unsigned* d_cnt, int* nl) {
        return bp_config_pairs_launch(d_bb, t.links, d_tpl, t.n, t.g0, t.ng, pf, ps, cap, d_cnt, ctx->num_sms, s, nl,
                                      entries ? static_cast<uint32_t*>(ctx->sc_f.p) : nullptr);
      });
}

// hfb_env_collide_configs: the candidates and their records (configs_candidates), then the outputs
struct EnvCollideConfigs {
  const hfb_collision_request* req;
  const hfb_configs_out* out;
  ConfigTpl t;
  bool minus_inf = false;

  const ConfigTpl* tpl() const { return &t; }
  int check(hfb_ctx* ctx) { return collide_prelude(ctx, req, &minus_inf); }
  int zero(hfb_ctx* ctx, QueryOut& o, size_t n_a) const {
    for (const hfb_scene_contacts* k : {&out->env, &out->self}) {
      CK(o.zero(k->n_candidates, sizeof(uint32_t)));
      CK(o.zero(k->n_colliding, sizeof(uint32_t)));
    }
    CK(o.zero(out->verdicts, n_a / t.links));
    return HFB_OK;
  }
  bool empty(const hfb_env* e, size_t n_a) const { return n_a == 0 || t.ng == 0 || (e->n_b == 0 && t.n == 0); }
  int run(hfb_ctx* ctx, hfb_env* e, size_t n_a, QueryOut& o) const {
    const size_t links = t.links;
    unsigned cand = 0, split = 0;
    if (int rc = configs_candidates(ctx, e, n_a, t, req, minus_inf, false, o.s, &cand, &split)) return rc;
    CK(o.count(out->env.n_candidates, split));
    CK(o.count(out->self.n_candidates, cand - split));
    if (cand == 0 || minus_inf) {
      CK(o.finish());
      return HFB_OK;
    }
    return configs_output(ctx, cand, split, (uint32_t)n_a, links, n_a / links, out, o);
  }
};

// hfb_env_distance's output and cutoff (max_distance >= 0 or +inf), checked before the context is looked at
static bool env_distance_ok(const hfb_env_distance_out* o, double max_distance) {
  return o && (o->nearest || o->min_distance || o->results) && max_distance >= 0;
}

// the rounds of a distance query of A (already in the table in front of B) against the env for A objects [a_lo, a_hi):
// A's boxes (ctx->sc_bb), then rounds of candidates within a growing radius (hfb::BpDistState, in ctx->sc_dist): each
// round's new pairs through distance() over the table [A; B] and into the per-A best.  Blocks for the candidate counts
// once per round (per chunk of A, and once more when the lists grow).  *st: the per-A state; *n_cand: the pairs whose
// distance() ran (clamped to 32 bits); the unsupported ones are counted in ctx->sc_cnt's fourth word.
static int env_distance_rounds(hfb_ctx* ctx, hfb_env* e, size_t n_a, size_t a_lo, size_t a_hi,
                               const hfb_distance_request* req, double maxd, cudaStream_t s, BpDistState* st_out,
                               unsigned* n_cand) {
  const size_t n_b = e->n_b;
  const size_t off = e->head - n_a;
  const uint32_t* d_h = static_cast<const uint32_t*>(e->h.p) + off;
  const hfb_transform* d_tf = static_cast<const hfb_transform*>(e->tf.p) + off;
  const double* bb_b = static_cast<const double*>(e->bb.p);
  const BpCrossGrid g = bp_cross_grid_carve(e->grid.p, n_b);
  CK(ctx->sc_bb.reserve(n_a * 96));  // A's boxes, then the round's query boxes
  CK(ctx->sc_cnt.reserve(16));       // candidates, kept candidates, open A objects, unsupported pairs
  CK(ctx->sc_dist.reserve(bp_dist_state_bytes(n_a)));
  CK(ctx->bp_scratch.reserve(bp_cross_scratch_bytes(n_a, n_b)));
  double* d_ba = static_cast<double*>(ctx->sc_bb.p);
  double* d_bq = d_ba + 6 * n_a;
  unsigned* d_cnt = static_cast<unsigned*>(ctx->sc_cnt.p);
  const BpDistState st = bp_dist_state_carve(ctx->sc_dist.p, n_a, static_cast<const unsigned long long*>(e->reach.p));
  int nl = 0;
  CK(cudaMemsetAsync(d_cnt + 3, 0, sizeof(unsigned), s));
  if (bp_scene_aabbs_launch(ctx->dview.local_aabbs, ctx->dview.nshapes, n_a, d_h, d_tf, d_ba, s) != 0)
    return fail(ctx, HFB_ERR_CUDA, "k_scene_aabbs launch failed");
  ++nl;
  if (bp_dist_init_launch(n_a, d_ba, a_lo, a_hi, st, s, &nl) != 0)
    return fail(ctx, HFB_ERR_CUDA, "k_dist_init launch failed");
  uint64_t total = 0;
  // a query counts its candidates in 32 bits: the range goes through the grid in chunks of A objects whose pairs with
  // all of B number fewer than 2^32, so that no round's count can wrap whatever its radius
  const size_t chunk = n_b ? (0xffffffffull / n_b > 0 ? 0xffffffffull / n_b : 1) : 1;
  for (int round = 0; n_b && a_lo < a_hi; ++round) {
    if (bp_dist_boxes_launch(d_ba, a_lo, a_hi, g, maxd, round, st, d_bq, d_cnt + 2, s, &nl) != 0)
      return fail(ctx, HFB_ERR_CUDA, "k_dist_boxes launch failed");
    bool open = true;
    for (size_t c0 = a_lo; open && c0 < a_hi; c0 += chunk) {
      const size_t c1 = a_hi - c0 > chunk ? c0 + chunk : a_hi;
      // the chunk's candidates less the pairs the round before ran; the open count is the whole round's
      unsigned words[3] = {0, 0, 0};
      auto find = [&](size_t cap, int* launches) {
        uint32_t* pf = static_cast<uint32_t*>(ctx->sc_pf.p);
        uint32_t* ps = static_cast<uint32_t*>(ctx->sc_ps.p);
        int rc = bp_cross_query_reset(g, d_cnt, s);
        if (!rc)
          rc = bp_cross_query_launch(n_a, d_bq, c0, c1, n_b, bb_b, g, pf, ps, (uint32_t)n_a, cap, d_cnt, ctx->bp_scratch.p,
                                     ctx->num_sms, s, launches);
        if (!rc)
          rc = bp_dist_filter_launch(pf, ps, d_cnt, cap, d_ba, bb_b, (uint32_t)n_a, g, maxd, round,
                                     static_cast<uint32_t*>(ctx->sc_f.p), static_cast<uint32_t*>(ctx->sc_s.p), d_cnt + 1,
                                     ctx->num_sms, s, launches);
        return rc;
      };
      if (int rc = find_all(ctx, s, {&ctx->sc_pf, &ctx->sc_ps, &ctx->sc_f, &ctx->sc_s}, d_cnt, find, words, 3)) return rc;
      open = words[2] != 0;  // (0: every object of the range is settled)
      const unsigned kept = words[1];
      total += kept;
      if (!open || kept == 0) continue;
      CK(ctx->sc_drec.reserve((size_t)kept * sizeof(hfb_distance_result)));
      hfb_object_pairs sc;
      sc.n_objects = n_a + n_b;
      sc.object_handles = d_h;
      sc.object_tfs = d_tf;
      sc.n_pairs = kept;
      sc.first = static_cast<const uint32_t*>(ctx->sc_f.p);
      sc.second = static_cast<const uint32_t*>(ctx->sc_s.p);
      if (int rc = objects_device<0>(ctx, &sc, req, solver_from_distance_request(*req), CollideP{0, 0},
                                     bvh_req_of_distance(req), ctx->sc_drec.p, nullptr, s))
        return rc;
      if (bp_dist_reduce_launch(static_cast<const hfb_distance_result*>(ctx->sc_drec.p), sc.first, sc.second, kept,
                                (uint32_t)n_a, maxd, st, d_cnt + 3, s, &nl) != 0)
        return fail(ctx, HFB_ERR_CUDA, "k_dist_min launch failed");
    }
    if (!open) break;
  }
  ctx->stats.kernel_launches += (uint64_t)nl;
  *st_out = st;
  *n_cand = total > 0xffffffffull ? 0xffffffffu : (unsigned)total;
  return HFB_OK;
}

// hfb_env_distance: the rounds over the range, then the per-A outputs
struct EnvDistance {
  const hfb_distance_request* req;
  double maxd;
  const hfb_env_distance_out* out;
  size_t first_a, num_a;

  const ConfigTpl* tpl() const { return nullptr; }
  int check(hfb_ctx* ctx) const {
    if (int rc = validate_query(req->q)) return fail(ctx, rc, "invalid request");
    return HFB_OK;
  }
  int zero(hfb_ctx* ctx, QueryOut& o, size_t) const {
    CK(o.zero(out->n_candidates, sizeof(uint32_t)));
    CK(o.zero(out->n_unsupported, sizeof(uint32_t)));
    return HFB_OK;
  }
  bool empty(const hfb_env*, size_t n_a) const { return n_a == 0; }
  int run(hfb_ctx* ctx, hfb_env* e, size_t n_a, QueryOut& o) const {
    const size_t a_lo = first_a < n_a ? first_a : n_a, a_hi = a_lo + (num_a < n_a - a_lo ? num_a : n_a - a_lo);
    BpDistState st;
    unsigned n_cand = 0;
    if (int rc = env_distance_rounds(ctx, e, n_a, a_lo, a_hi, req, maxd, o.s, &st, &n_cand)) return rc;
    const unsigned* d_cnt = static_cast<const unsigned*>(ctx->sc_cnt.p);
    CK(o.copy(out->nearest, st.nearest, n_a * 4));
    CK(o.copy_field(out->min_distance, st.rec, sizeof(double), sizeof(hfb_distance_result), n_a));  // (the first field)
    CK(o.copy(out->results, st.rec, n_a * sizeof(hfb_distance_result)));
    CK(o.copy(out->n_unsupported, d_cnt + 3, sizeof(unsigned)));
    CK(o.count(out->n_candidates, n_cand));
    CK(o.finish());
    return HFB_OK;
  }
};

// hfb_env_distance_configs' output and cutoff, checked before the context is looked at
static bool configs_distance_ok(const hfb_configs_distance_out* o, double max_distance) {
  return o && (o->kind || o->min_distance || o->results) && max_distance >= 0;
}

// hfb_env_distance_configs (the template in ctx->sc_tpl): the rounds over the range's links, then per chunk of
// configurations the self pairs config_dist_pair runs, distance() of them over the table [A; B], and the winner of
// each configuration from its links' winners and its self records (in ctx->sc_cdist).  Blocks for the self candidate
// count once per chunk (and once more when the lists grow).  Then the outputs.
struct EnvDistanceConfigs {
  const hfb_distance_request* req;
  double maxd;
  const hfb_configs_distance_out* out;
  ConfigTpl t;

  const ConfigTpl* tpl() const { return &t; }
  int check(hfb_ctx* ctx) const {
    if (int rc = validate_query(req->q)) return fail(ctx, rc, "invalid request");
    return HFB_OK;
  }
  int zero(hfb_ctx* ctx, QueryOut& o, size_t) const {
    for (uint32_t* c : {out->n_env_candidates, out->n_self_candidates, out->n_unsupported})
      CK(o.zero(c, sizeof(uint32_t)));
    return HFB_OK;
  }
  bool empty(const hfb_env*, size_t n_a) const { return n_a == 0; }
  int run(hfb_ctx* ctx, hfb_env* e, size_t n_a, QueryOut& o) const {
    const cudaStream_t s = o.s;
    const size_t n_b = e->n_b, links = t.links, n_tpl = t.n, g0 = t.g0, ng = t.ng, n_configs = n_a / links;
    BpDistState st;
    unsigned n_env = 0;
    if (int rc = env_distance_rounds(ctx, e, n_a, g0 * links, (g0 + ng) * links, req, maxd, s, &st, &n_env)) return rc;
    CK(ctx->sc_cdist.reserve(bp_config_dist_bytes(n_configs)));
    const BpConfigDist cs = bp_config_dist_carve(ctx->sc_cdist.p, n_configs);
    const size_t off = e->head - n_a;
    const double* d_ba = static_cast<const double*>(ctx->sc_bb.p);  // (A's boxes, from the rounds)
    unsigned* d_cnt = static_cast<unsigned*>(ctx->sc_cnt.p);
    const uint32_t* d_tpl = static_cast<const uint32_t*>(ctx->sc_tpl.p);
    int nl = 0;
    if (bp_config_dist_init_launch(n_configs, cs, s, &nl) != 0) return fail(ctx, HFB_ERR_CUDA, "k_cfg_init launch failed");
    uint64_t total = 0;
    // the self candidates are counted in 32 bits: chunks of configurations whose template entries number fewer than
    // 2^32 (whole configurations, so that each chunk's winners are final)
    const size_t chunk = n_tpl ? 0xffffffffull / n_tpl : (ng ? ng : 1);
    for (size_t c0 = g0; c0 < g0 + ng; c0 += chunk) {
      const size_t c1 = g0 + ng - c0 > chunk ? c0 + chunk : g0 + ng;
      unsigned kept = 0;
      if (n_tpl) {
        auto find = [&](size_t cap, int* launches) {
          return bp_config_dist_pairs_launch(d_ba, links, d_tpl, n_tpl, c0, c1 - c0, maxd,
                                             static_cast<uint32_t*>(ctx->sc_pf.p), static_cast<uint32_t*>(ctx->sc_ps.p),
                                             static_cast<uint32_t*>(ctx->sc_f.p), cap, d_cnt, ctx->num_sms, s, launches);
        };
        unsigned words[1] = {0};
        if (int rc = find_all(ctx, s, {&ctx->sc_pf, &ctx->sc_ps, &ctx->sc_f}, d_cnt, find, words, 1)) return rc;
        kept = words[0];
        total += kept;
      }
      if (kept) {
        CK(ctx->sc_drec.reserve((size_t)kept * sizeof(hfb_distance_result)));
        hfb_object_pairs sc;
        sc.n_objects = n_a + n_b;
        sc.object_handles = static_cast<const uint32_t*>(e->h.p) + off;
        sc.object_tfs = static_cast<const hfb_transform*>(e->tf.p) + off;
        sc.n_pairs = kept;
        sc.first = static_cast<const uint32_t*>(ctx->sc_pf.p);
        sc.second = static_cast<const uint32_t*>(ctx->sc_ps.p);
        if (int rc = objects_device<0>(ctx, &sc, req, solver_from_distance_request(*req), CollideP{0, 0},
                                       bvh_req_of_distance(req), ctx->sc_drec.p, nullptr, s))
          return rc;
      }
      if (bp_config_dist_reduce_launch(st, c0 * links, c1 * links, links,
                                       static_cast<const hfb_distance_result*>(ctx->sc_drec.p),
                                       static_cast<const uint32_t*>(ctx->sc_pf.p), static_cast<const uint32_t*>(ctx->sc_ps.p),
                                       static_cast<const uint32_t*>(ctx->sc_f.p), kept, maxd, cs, d_cnt + 3, s, &nl) != 0)
        return fail(ctx, HFB_ERR_CUDA, "k_cfg_min launch failed");
    }
    ctx->stats.kernel_launches += (uint64_t)nl;
    const unsigned n_self = total > 0xffffffffull ? 0xffffffffu : (unsigned)total;
    CK(o.copy(out->kind, cs.kind, n_configs));
    CK(o.copy(out->first, cs.first, n_configs * 4));
    CK(o.copy(out->second, cs.second, n_configs * 4));
    CK(o.copy_field(out->min_distance, cs.rec, sizeof(double), sizeof(hfb_distance_result), n_configs));  // (the first field)
    CK(o.copy(out->results, cs.rec, n_configs * sizeof(hfb_distance_result)));
    CK(o.copy(out->n_unsupported, d_cnt + 3, sizeof(unsigned)));
    CK(o.count(out->n_env_candidates, n_env));
    CK(o.count(out->n_self_candidates, n_self));
    CK(o.finish());
    return HFB_OK;
  }
};

// hfb_env_collide_motions' outputs, checked before the context is looked at
static bool motions_ok(const hfb_motions_out* o) { return o && (o->first_invalid || o->kind || o->contacts); }

// the record of a motion without a witness: CollisionResult::clear() (collision_data.h:483-489), as k_mot_init writes it
static hfb_contact cleared_contact() {
  hfb_contact r;
  const double nan = std::numeric_limits<double>::quiet_NaN();
  r.distance = nan;
  for (int k = 0; k < 3; ++k) r.p1[k] = r.p2[k] = r.normal[k] = r.pos[k] = nan;
  r.distance_lower_bound = DBL_MAX;
  r.b1 = r.b2 = -1;
  r.status = r.num_contacts = r.iterations = r._pad = 0;
  return r;
}

// hfb_env_collide_motions (the template in ctx->sc_tpl, the offsets uploaded into ctx->sc_moff): the candidates and
// records of hfb_env_collide_configs over the range's configurations (configs_candidates, with the self pairs' template
// entries when a witness is wanted), then per motion the first colliding sample and its first colliding pair
// (hfb::BpMotions, in ctx->sc_mot).  t.g0 and t.ng are set by motions_args.
struct EnvCollideMotions {
  const hfb_collision_request* req;
  const hfb_motions_out* out;
  ConfigTpl t;
  size_t n_motions;
  const uint32_t* offsets;
  size_t first_motion, num_motions;
  bool minus_inf = false;

  const ConfigTpl* tpl() const { return &t; }
  bool witness() const { return out->kind || out->first || out->second || out->contacts; }
  int check(hfb_ctx* ctx) { return collide_prelude(ctx, req, &minus_inf); }
  int zero(hfb_ctx* ctx, QueryOut& o, size_t) const {
    for (uint32_t* c : {out->n_env_candidates, out->n_env_colliding, out->n_self_candidates, out->n_self_colliding})
      CK(o.zero(c, sizeof(uint32_t)));
    const size_t n = n_motions;
    if (o.dev) {  // (on the caller's stream)
      BpMotions ms{};
      ms.first_invalid = out->first_invalid;
      ms.kind = out->kind;
      ms.first = out->first;
      ms.second = out->second;
      ms.rec = out->contacts;
      int nl = 0;
      if (bp_motions_init_launch(n, ms, o.s, &nl) != 0) return fail(ctx, HFB_ERR_CUDA, "k_mot_init launch failed");
      ctx->stats.kernel_launches += (uint64_t)nl;
      return HFB_OK;
    }
    if (out->first_invalid) std::fill(out->first_invalid, out->first_invalid + n, -1);
    if (out->kind) std::fill(out->kind, out->kind + n, (int8_t)-1);
    if (out->first) std::fill(out->first, out->first + n, 0xffffffffu);
    if (out->second) std::fill(out->second, out->second + n, 0xffffffffu);
    if (out->contacts) std::fill(out->contacts, out->contacts + n, cleared_contact());
    return HFB_OK;
  }
  bool empty(const hfb_env* e, size_t n_a) const { return n_a == 0 || t.ng == 0 || (e->n_b == 0 && t.n == 0); }
  int run(hfb_ctx* ctx, hfb_env* e, size_t n_a, QueryOut& o) const {
    const cudaStream_t s = o.s;
    const bool wit = witness();
    unsigned cand = 0, split = 0;
    if (int rc = configs_candidates(ctx, e, n_a, t, req, minus_inf, wit, s, &cand, &split)) return rc;
    CK(o.count(out->n_env_candidates, split));
    CK(o.count(out->n_self_candidates, cand - split));
    if (cand == 0 || minus_inf) {  // (no colliding pair: the zeroed counts and the no-witness outputs stand)
      CK(o.finish());
      return HFB_OK;
    }
    const size_t n = n_motions;
    CK(ctx->sc_moff.reserve((n + 1) * 4));
    CK(cudaMemcpyAsync(ctx->sc_moff.p, offsets, (n + 1) * 4, cudaMemcpyHostToDevice, s));
    CK(ctx->sc_mot.reserve(bp_motions_bytes(n, !o.dev)));
    BpMotions ms = bp_motions_carve(ctx->sc_mot.p, n, !o.dev);  // (the host form stages its outputs there)
    ms.off = static_cast<const uint32_t*>(ctx->sc_moff.p);
    ms.m0 = (unsigned)first_motion;
    ms.m1 = (unsigned)(first_motion + num_motions);
    if (o.dev) {
      ms.first_invalid = out->first_invalid;
      ms.kind = out->kind;
      ms.first = out->first;
      ms.second = out->second;
      ms.rec = out->contacts;
    } else {
      if (!out->first_invalid) ms.first_invalid = nullptr;
      if (!out->kind) ms.kind = nullptr;
      if (!out->first) ms.first = nullptr;
      if (!out->second) ms.second = nullptr;
      if (!out->contacts) ms.rec = nullptr;
    }
    BpMotions state = ms;  // the device form's outputs hold zero()'s no-witness values already
    if (o.dev) state.first_invalid = nullptr, state.kind = nullptr, state.first = state.second = nullptr, state.rec = nullptr;
    unsigned* d_cnt = static_cast<unsigned*>(ctx->sc_cnt.p);
    CK(cudaMemsetAsync(d_cnt + 1, 0, 2 * sizeof(unsigned), s));
    int nl = 0;
    if (bp_motions_init_launch(n, state, s, &nl) != 0) return fail(ctx, HFB_ERR_CUDA, "k_mot_init launch failed");
    if (bp_motions_reduce_launch(static_cast<const hfb_contact*>(ctx->sc_out.p), static_cast<const uint32_t*>(ctx->sc_pf.p),
                                 static_cast<const uint32_t*>(ctx->sc_ps.p), static_cast<const uint32_t*>(ctx->sc_f.p), cand,
                                 split, t.links, e->n_b, (uint32_t)n_a, wit, ms, d_cnt + 1, s, &nl) != 0)
      return fail(ctx, HFB_ERR_CUDA, "k_mot_min launch failed");
    if (bp_motions_final_launch(ms, s, &nl) != 0) return fail(ctx, HFB_ERR_CUDA, "k_mot_final launch failed");
    ctx->stats.kernel_launches += (uint64_t)nl;
    if (!o.dev) {
      CK(o.copy(out->first_invalid, ms.first_invalid, n * 4));
      CK(o.copy(out->kind, ms.kind, n));
      CK(o.copy(out->first, ms.first, n * 4));
      CK(o.copy(out->second, ms.second, n * 4));
      CK(o.copy(out->contacts, ms.rec, n * sizeof(hfb_contact)));
    }
    CK(o.copy(out->n_env_colliding, d_cnt + 1, sizeof(unsigned)));
    CK(o.copy(out->n_self_colliding, d_cnt + 2, sizeof(unsigned)));
    CK(o.finish());
    return HFB_OK;
  }
};

// hfb_env_certify_motions' outputs, checked before the context is looked at
static bool certify_ok(const hfb_certify_out* o) { return o && (o->first_invalid || o->first_uncertified || o->certified); }

// The certification that hfb_env_certify_motions and hfb_env_validate_motions share, with A in the env's table and the
// template in ctx->sc_tpl: the sides of A's objects of the configurations [t.g0, t.g0 + t.ng) from the device sweep
// bounds d_sweep and their widened boxes (c.sides, the boxes after the 2 * n_a sides), the candidates of the widened
// boxes and of sweep_pair with their collide() records (configs_candidates; *cand and *split as it gives them), then
// bp_certify_launch into c's flags, state and outputs, counting in ctx->sc_cnt[1] (unsupported) and [2] (uncertified).
// c holds the motions (device offsets, [m0, m1)), the configurations (g0, ng), the sides and the pass flags.
static int certify_body(hfb_ctx* ctx, hfb_env* e, size_t n_a, const ConfigTpl& t, const hfb_collision_request* req,
                        bool minus_inf, const BpCertify& c, const double* d_sweep, cudaStream_t s, unsigned* cand,
                        unsigned* split) {
  const size_t links = t.links;
  double* d_wbb = c.sides + 2 * n_a;
  const uint32_t* d_tpl = static_cast<const uint32_t*>(ctx->sc_tpl.p);
  const size_t a_lo = t.g0 * links, a_hi = (t.g0 + t.ng) * links;
  bool sided = false;  // (the finder runs twice when the candidate lists grow; the sides are made once)
  if (int rc = configs_candidates(
          ctx, e, n_a, t, req, minus_inf, nullptr, s, cand, split,
          [&](const double* d_bb, const double** d_qb, int* nl) {
            *d_qb = d_wbb;
            if (sided) return 0;
            sided = true;
            return bp_sweep_sides_launch(d_bb, d_sweep, a_lo, a_hi, c, d_wbb, s, nl);
          },
          [&](const double* d_bb, uint32_t* pf, uint32_t* ps, size_t cap, unsigned* d_cnt, int* nl) {
            return bp_sweep_pairs_launch(d_bb, c, d_tpl, t.n, pf, ps, cap, d_cnt, ctx->num_sms, s, nl);
          }))
    return rc;
  unsigned* d_cnt = static_cast<unsigned*>(ctx->sc_cnt.p);
  CK(cudaMemsetAsync(d_cnt + 1, 0, 2 * sizeof(unsigned), s));
  // under minus_inf no record exists (collision.cpp:73-76): every pair passes, every sample is valid
  const size_t n_recs = minus_inf ? 0 : *cand;
  int nl = 0;
  if (bp_certify_launch(static_cast<const hfb_contact*>(ctx->sc_out.p), static_cast<const uint32_t*>(ctx->sc_pf.p),
                        static_cast<const uint32_t*>(ctx->sc_ps.p), n_recs, *split, (uint32_t)n_a,
                        static_cast<const double*>(ctx->sc_bb.p), static_cast<const double*>(e->bb.p), c, d_cnt + 1, s,
                        &nl) != 0)
    return fail(ctx, HFB_ERR_CUDA, "k_cert_pairs launch failed");
  ctx->stats.kernel_launches += (uint64_t)nl;
  return HFB_OK;
}

// hfb_env_certify_motions (the template in ctx->sc_tpl, the offsets in ctx->sc_moff, the sweep bounds in
// ctx->sc_sweep in the host form): the sides of the range's A objects and their widened boxes (ctx->sc_side), the
// candidates of the widened boxes and of sweep_pair with their collide() records (configs_candidates), then the
// per-sample flags (ctx->sc_cpass) and the per-motion state (hfb::BpCertify, in ctx->sc_mot).  t.g0 and t.ng are set
// by motions_args.
struct EnvCertifyMotions {
  const hfb_collision_request* req;
  const hfb_certify_out* out;
  ConfigTpl t;
  size_t n_motions;
  const uint32_t* offsets;
  size_t first_motion, num_motions;
  const double* sweep;
  bool minus_inf = false;

  const ConfigTpl* tpl() const { return &t; }
  int check(hfb_ctx* ctx) { return collide_prelude(ctx, req, &minus_inf); }
  int zero(hfb_ctx* ctx, QueryOut& o, size_t n_a) const {
    for (uint32_t* c : {out->n_env_candidates, out->n_self_candidates, out->n_unsupported, out->n_uncertified})
      CK(o.zero(c, sizeof(uint32_t)));
    CK(o.zero(out->certified, n_a / t.links));
    const size_t n = n_motions;
    if (o.dev) {  // (on the caller's stream: -1 for every motion)
      int nl = 0;
      for (int32_t* p : {out->first_invalid, out->first_uncertified}) {
        BpMotions ms{};
        ms.first_invalid = p;
        if (p && bp_motions_init_launch(n, ms, o.s, &nl) != 0) return fail(ctx, HFB_ERR_CUDA, "k_mot_init launch failed");
      }
      ctx->stats.kernel_launches += (uint64_t)nl;
      return HFB_OK;
    }
    if (out->first_invalid) std::fill(out->first_invalid, out->first_invalid + n, -1);
    if (out->first_uncertified) std::fill(out->first_uncertified, out->first_uncertified + n, -1);
    return HFB_OK;
  }
  // (with no pair at all the segments with valid sweeps are still certified: only an empty range is empty)
  bool empty(const hfb_env*, size_t n_a) const { return n_a == 0 || t.ng == 0; }
  int run(hfb_ctx* ctx, hfb_env* e, size_t n_a, QueryOut& o) const {
    const cudaStream_t s = o.s;
    const size_t n = n_motions, links = t.links;
    CK(ctx->sc_moff.reserve((n + 1) * 4));
    CK(cudaMemcpyAsync(ctx->sc_moff.p, offsets, (n + 1) * 4, cudaMemcpyHostToDevice, s));
    const double* d_sweep = sweep;
    if (!o.dev) {
      CK(ctx->sc_sweep.reserve(n_a * 8));
      CK(cudaMemcpyAsync(ctx->sc_sweep.p, sweep, n_a * 8, cudaMemcpyHostToDevice, s));
      d_sweep = static_cast<const double*>(ctx->sc_sweep.p);
    }
    CK(ctx->sc_side.reserve(n_a * 64));  // per A object: its two sides (16 bytes), its widened box (48)
    CK(ctx->sc_cpass.reserve(t.ng * 2));
    CK(ctx->sc_mot.reserve(bp_certify_bytes(n, !o.dev)));
    BpCertify c = bp_certify_carve(ctx->sc_mot.p, n, !o.dev);  // (the host form stages its outputs there)
    c.off = static_cast<const uint32_t*>(ctx->sc_moff.p);
    c.m0 = (unsigned)first_motion;
    c.m1 = (unsigned)(first_motion + num_motions);
    c.links = (unsigned)links;
    c.g0 = (unsigned)t.g0;
    c.ng = (unsigned)t.ng;
    c.sides = static_cast<double*>(ctx->sc_side.p);
    c.pass = static_cast<uint8_t*>(ctx->sc_cpass.p);
    if (o.dev) {
      c.first_invalid = out->first_invalid;
      c.first_uncertified = out->first_uncertified;
      c.certified = out->certified ? out->certified + t.g0 : nullptr;
    } else {
      if (!out->first_invalid) c.first_invalid = nullptr;
      if (!out->first_uncertified) c.first_uncertified = nullptr;
      if (out->certified) {
        CK(ctx->sc_flags.reserve(t.ng));
        c.certified = static_cast<uint8_t*>(ctx->sc_flags.p);
      }
    }
    unsigned cand = 0, split = 0;
    if (int rc = certify_body(ctx, e, n_a, t, req, minus_inf, c, d_sweep, s, &cand, &split)) return rc;
    CK(o.count(out->n_env_candidates, split));
    CK(o.count(out->n_self_candidates, cand - split));
    unsigned* d_cnt = static_cast<unsigned*>(ctx->sc_cnt.p);
    if (!o.dev) {
      const size_t m0 = first_motion, nm = num_motions;
      if (out->first_invalid) CK(o.copy(out->first_invalid + m0, c.first_invalid + m0, nm * 4));
      if (out->first_uncertified) CK(o.copy(out->first_uncertified + m0, c.first_uncertified + m0, nm * 4));
      if (out->certified) CK(o.copy(out->certified + t.g0, c.certified, t.ng));
    }
    CK(o.copy(out->n_unsupported, d_cnt + 1, sizeof(unsigned)));
    CK(o.copy(out->n_uncertified, d_cnt + 2, sizeof(unsigned)));
    CK(o.finish());
    return HFB_OK;
  }
};

// hfb_env_validate_motions' pure argument checks, before the context is looked at
static bool validate_ok(size_t n_motions, const double* q_from, const double* q_to, size_t n_self_pairs,
                        const uint32_t* self_pairs, size_t first_motion, size_t num_motions,
                        const hfb_collision_request* req, const hfb_validate_params* p, const hfb_validate_out* o) {
  if (!req || !p || !o || !o->status || !o->t_valid || !o->t_collide || (n_self_pairs && !self_pairs)) return false;
  if (p->initial_depth > p->max_depth || p->max_depth > 30 || p->max_samples < 2) return false;
  if (n_motions > 0xffffffffull || first_motion > n_motions || num_motions > n_motions - first_motion) return false;
  return !(num_motions && (!q_from || !q_to));
}

// an exclusive (ex) or inclusive scan of n uint32 on stream s, CUB's scratch in ctx->sc_vcub
static int val_scan(hfb_ctx* ctx, const uint32_t* in, uint32_t* out, uint32_t n, bool ex, cudaStream_t s) {
  size_t bytes = 0;
  CK(ex ? cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, (int)n, s)
        : cub::DeviceScan::InclusiveSum(nullptr, bytes, in, out, (int)n, s));
  CK(ctx->sc_vcub.reserve(bytes));
  CK(ex ? cub::DeviceScan::ExclusiveSum(ctx->sc_vcub.p, bytes, in, out, (int)n, s)
        : cub::DeviceScan::InclusiveSum(ctx->sc_vcub.p, bytes, in, out, (int)n, s));
  ctx->stats.kernel_launches++;
  return HFB_OK;
}

static unsigned val_blocks(size_t n) { return (unsigned)((n + 255) / 256); }

// hfb_env_validate_motions (include/hppfcl_b200.h states the rounds and their rules): the robot samples each round's
// runs straight into the env's table (k_robot_at), certify_body certifies them as motions, and the k_val_* kernels
// apply the rules and build the next round's list.  The call blocks once per round for its totals (the admitted
// segments, samples and runs that size the launches), where certify_body blocks, and once for the witness count.
// Buffers: ctx->sc_vmot the per-motion state (and the host form's staged outputs), sc_vseg the two lists, sc_vscan the
// per-segment scans, sc_vsmp the samples, sc_vrun the runs and the certified flags, sc_sweep the sweep bounds.
struct EnvValidateMotions {
  const hfb_collision_request* req;
  const hfb_validate_out* out;
  ConfigTpl t;  // links: the robot's L (set by check()); g0 and ng: each round's samples
  hfb_robot* robot;
  size_t n_motions;
  const double* q_from;
  const double* q_to;
  size_t first_motion, num_motions;
  hfb_validate_params p;
  bool minus_inf = false;

  const ConfigTpl* tpl() const { return &t; }
  bool witness() const { return out->kind || out->first || out->second || out->contacts; }
  int check(hfb_ctx* ctx) {
    if (int rc = collide_prelude(ctx, req, &minus_inf)) return rc;
    if (int rc = robot_ready(ctx, robot)) return rc;
    t.links = robot->L;
    return HFB_OK;
  }
  int zero(hfb_ctx* ctx, QueryOut& o, size_t) const {
    CK(o.zero(out->n_rounds, sizeof(uint32_t)));
    for (uint64_t* c : {out->n_samples, out->n_env_candidates, out->n_self_candidates, out->n_unsupported})
      CK(o.zero(c, sizeof(uint64_t)));
    return HFB_OK;
  }
  bool empty(const hfb_env*, size_t) const { return false; }  // (run() writes every motion's outputs)
  int run(hfb_ctx* ctx, hfb_env* e, size_t, QueryOut& o) const {
    const cudaStream_t s = o.s;
    const uint32_t L = (uint32_t)t.links, J = robot->J, D = p.max_depth, d0 = p.initial_depth;
    const size_t n = n_motions, n_range = num_motions, m0 = first_motion;
    // the cap: the caller's, at most 2^29 (so that a round's list, at most twice the samples before it, and the scan of
    // its costs, at most twice its length, stay below 2^31), and within the env calls' 32-bit object count
    // (samples * L + n_b < 2^32)
    uint64_t cap64 = p.max_samples < (1ull << 29) ? p.max_samples : (1ull << 29);
    const uint64_t fit = (0xffffffffull - e->n_b) / L;
    if (fit < cap64) cap64 = fit;
    const uint32_t cap = (uint32_t)cap64;
    hfb::KinAtArgs ka{};
    if (int rc = robot_model_args(ctx, robot, s, &ka)) return rc;
    ka.n_pos = (1u << D) + 1u;
    if (o.dev) {
      ka.q_from = q_from + m0 * J;
      ka.q_to = q_to + m0 * J;
    } else if (n_range) {
      CK(robot->q_in.reserve(n_range * J * 16));
      double* d_q = static_cast<double*>(robot->q_in.p);
      CK(cudaMemcpyAsync(d_q, q_from + m0 * J, n_range * J * 8, cudaMemcpyHostToDevice, s));
      CK(cudaMemcpyAsync(d_q + n_range * J, q_to + m0 * J, n_range * J * 8, cudaMemcpyHostToDevice, s));
      ka.q_from = d_q;
      ka.q_to = d_q + n_range * J;
    }
    // per motion: the state, the witness flags and their scan, then (host form) the staged outputs
    const size_t r4 = up(n_range * 4);
    CK(ctx->sc_vmot.reserve(5 * r4 + (o.dev ? 0 : up(n) * 2 + up(n * 8) * 2 + up(n * 4) * 2 + up(n * sizeof(hfb_contact)))));
    char* vm = static_cast<char*>(ctx->sc_vmot.p);
    const ValMotions st{reinterpret_cast<uint32_t*>(vm), reinterpret_cast<uint32_t*>(vm + r4),
                        reinterpret_cast<uint32_t*>(vm + 2 * r4)};
    uint32_t* wflag = reinterpret_cast<uint32_t*>(vm + 3 * r4);
    uint32_t* widx = reinterpret_cast<uint32_t*>(vm + 4 * r4);
    ValOut vo{out->status, out->t_valid, out->t_collide};
    BpMotions wo{};
    wo.kind = out->kind, wo.first = out->first, wo.second = out->second, wo.rec = out->contacts;
    if (!o.dev) {
      char* at = vm + 5 * r4;
      auto take = [&](size_t bytes) {
        char* q = at;
        at += up(bytes);
        return q;
      };
      vo.status = reinterpret_cast<int8_t*>(take(n));
      vo.t_valid = reinterpret_cast<double*>(take(n * 8));
      vo.t_collide = reinterpret_cast<double*>(take(n * 8));
      int8_t* k = reinterpret_cast<int8_t*>(take(n));
      uint32_t* f = reinterpret_cast<uint32_t*>(take(n * 4));
      uint32_t* sc = reinterpret_cast<uint32_t*>(take(n * 4));
      hfb_contact* r = reinterpret_cast<hfb_contact*>(take(n * sizeof(hfb_contact)));
      if (wo.kind) wo.kind = k;
      if (wo.first) wo.first = f;
      if (wo.second) wo.second = sc;
      if (wo.rec) wo.rec = r;
    }
    CK(ctx->sc_vcnt.reserve(64));
    uint32_t* d_nl = static_cast<uint32_t*>(ctx->sc_vcnt.p);  // the two lists' lengths
    uint32_t* d_tot = d_nl + 2;                                // a round's totals, the witness count
    unsigned long long* d_acc = reinterpret_cast<unsigned long long*>(d_nl + 8);  // the unsupported records
    CK(cudaMemsetAsync(d_acc, 0, 8, s));
    // round 0
    const uint32_t per = 1u << d0;
    uint64_t n_full = 0;
    uint32_t partial = 0;
    val_round0(n_range, per, cap, &n_full, &partial);
    uint64_t bound = n_full * per + partial;  // (<= cap)
    int cur = 0;
    CK(ctx->sc_vseg[0].reserve(bound * 8 + 8));
    if (n_range) {  // (a list of cap / 8 entries: w, then a, as every round reads it)
      const size_t cb = (size_t)(ctx->sc_vseg[0].cap / 8);
      const ValSegs sg{static_cast<uint32_t*>(ctx->sc_vseg[0].p), static_cast<uint32_t*>(ctx->sc_vseg[0].p) + cb};
      const size_t nt = bound > n_range ? bound : n_range;
      const size_t blocks = val_blocks(nt) < (size_t)ctx->num_sms * 8 ? val_blocks(nt) : (size_t)ctx->num_sms * 8;
      k_val_init<<<(unsigned)blocks, 256, 0, s>>>(sg, bound, n_range, n_full, partial, per, 1u << (D - d0), st, d_nl);
      ctx->stats.kernel_launches++;
    }
    uint32_t rounds = 0;
    uint64_t n_samples = 0, n_env = 0, n_self = 0;
    for (uint32_t depth = d0; n_range && bound && depth <= D; ++depth) {
      const uint32_t len = 1u << (D - depth), nb = (uint32_t)bound;
      const size_t cb = (size_t)(ctx->sc_vseg[cur].cap / 8);
      const ValSegs sg{static_cast<uint32_t*>(ctx->sc_vseg[cur].p), static_cast<uint32_t*>(ctx->sc_vseg[cur].p) + cb};
      CK(ctx->sc_vscan.reserve((size_t)nb * 24));
      uint32_t* cost = static_cast<uint32_t*>(ctx->sc_vscan.p);
      uint32_t *cscan = cost + nb, *nr = cost + 2 * (size_t)nb, *rscan = cost + 3 * (size_t)nb;
      uint32_t *kids = cost + 4 * (size_t)nb, *kscan = cost + 5 * (size_t)nb;
      k_val_cost<<<val_blocks(nb), 256, 0, s>>>(sg, d_nl + cur, nb, len, cost, nr);
      ctx->stats.kernel_launches++;
      if (int rc = val_scan(ctx, cost, cscan, nb, false, s)) return rc;
      if (int rc = val_scan(ctx, nr, rscan, nb, false, s)) return rc;
      k_val_admit<<<val_blocks(nb), 256, 0, s>>>(d_nl + cur, nb, cscan, rscan, cap, d_tot);
      ctx->stats.kernel_launches++;
      uint32_t tot[3] = {0, 0, 0};
      CK(cudaMemcpyAsync(tot, d_tot, sizeof tot, cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
      const uint32_t n_adm = tot[0], smp = tot[1], runs = tot[2];
      if (n_adm == 0) break;  // (no open segment left)
      ++rounds;
      n_samples += smp;
      // the samples and runs, the robot's poses and sweeps into the env's table, then the certification of the runs
      CK(ctx->sc_vsmp.reserve((size_t)smp * 9));
      uint32_t* sw = static_cast<uint32_t*>(ctx->sc_vsmp.p);
      uint32_t* sk = sw + smp;
      uint8_t* sseg = reinterpret_cast<uint8_t*>(sk + smp);
      CK(ctx->sc_vrun.reserve(up(((size_t)runs + 1) * 4) + up((size_t)runs * 4) + smp));
      uint32_t* off = static_cast<uint32_t*>(ctx->sc_vrun.p);
      int32_t* fi = reinterpret_cast<int32_t*>(static_cast<char*>(ctx->sc_vrun.p) + up(((size_t)runs + 1) * 4));
      uint8_t* cert = reinterpret_cast<uint8_t*>(fi) + up((size_t)runs * 4);
      k_val_samples<<<val_blocks(n_adm), 256, 0, s>>>(sg, n_adm, len, cscan, nr, rscan, sw, sk, sseg, off);
      ctx->stats.kernel_launches++;
      const size_t n_a = (size_t)smp * L;
      if (int rc = env_make_room(ctx, e, n_a, s)) return rc;
      CK(ctx->sc_sweep.reserve(n_a * 8));
      double* d_sweep = static_cast<double*>(ctx->sc_sweep.p);
      hfb::KinAtArgs a = ka;
      a.n_samples = smp;
      a.m = sw;
      a.k = sk;
      a.seg = sseg;
      a.len = len;
      a.tfs = static_cast<hfb_transform*>(e->tf.p) + (e->head - n_a);
      a.handles = static_cast<uint32_t*>(e->h.p) + (e->head - n_a);
      a.sweep = d_sweep;
      if (int err = hfb::robot_at_launch(a, ctx->num_sms, s))
        return cuda_fail(ctx, static_cast<cudaError_t>(err), "k_robot_at launch");
      ctx->stats.kernel_launches++;
      CK(ctx->sc_side.reserve(n_a * 64));
      CK(ctx->sc_cpass.reserve((size_t)smp * 2));
      CK(ctx->sc_mot.reserve(bp_certify_bytes(runs, false)));
      BpCertify c = bp_certify_carve(ctx->sc_mot.p, runs, false);
      c.off = off;
      c.m0 = 0;
      c.m1 = runs;
      c.links = L;
      c.g0 = 0;
      c.ng = smp;
      c.sides = static_cast<double*>(ctx->sc_side.p);
      c.pass = static_cast<uint8_t*>(ctx->sc_cpass.p);
      c.first_invalid = fi;
      c.certified = cert;
      ConfigTpl tr = t;
      tr.g0 = 0;
      tr.ng = smp;
      unsigned cand = 0, split = 0;
      if (int rc = certify_body(ctx, e, n_a, tr, req, minus_inf, c, d_sweep, s, &cand, &split)) return rc;
      n_env += split;
      n_self += cand - split;
      // the rules, the frontier and the next round's list
      k_val_collide<<<val_blocks(runs), 256, 0, s>>>(runs, fi, off, sw, sk, st);
      k_val_rules<<<val_blocks(nb), 256, 0, s>>>(sg, d_nl + cur, nb, n_adm, depth == D, L, cscan, cert, d_sweep, st, kids,
                                                 static_cast<const unsigned*>(ctx->sc_cnt.p) + 1, d_acc);
      k_val_keep<<<val_blocks(nb), 256, 0, s>>>(sg, d_nl + cur, len / 2, st, kids);
      ctx->stats.kernel_launches += 3;
      if (int rc = val_scan(ctx, kids, kscan, nb, true, s)) return rc;
      const uint64_t next = 2 * (uint64_t)n_adm;
      CK(ctx->sc_vseg[1 - cur].reserve(next * 8 + 8));
      const size_t nc = (size_t)(ctx->sc_vseg[1 - cur].cap / 8);
      const ValSegs nx{static_cast<uint32_t*>(ctx->sc_vseg[1 - cur].p), static_cast<uint32_t*>(ctx->sc_vseg[1 - cur].p) + nc};
      k_val_compact<<<val_blocks(nb), 256, 0, s>>>(sg, d_nl + cur, len / 2, st, kids, kscan, nx, d_nl + 1 - cur);
      ctx->stats.kernel_launches++;
      cur = 1 - cur;
      bound = next;
    }
    // the outputs, then the witnesses: one hfb_env_collide_motions pass over the colliding motions' samples at c
    const bool wit = witness() && n_range;
    if (n) {
      k_val_final<<<val_blocks(n), 256, 0, s>>>((uint32_t)n, (uint32_t)m0, (uint32_t)n_range, D, st, vo,
                                                wit ? wflag : nullptr);
      ctx->stats.kernel_launches++;
      if (witness()) {
        int nl = 0;
        if (bp_motions_init_launch(n, wo, s, &nl) != 0) return fail(ctx, HFB_ERR_CUDA, "k_mot_init launch failed");
        ctx->stats.kernel_launches += (uint64_t)nl;
      }
    }
    if (wit) {
      if (int rc = val_scan(ctx, wflag, widx, (uint32_t)n_range, true, s)) return rc;
      CK(ctx->sc_vsmp.reserve(n_range * 9));
      uint32_t* sw = static_cast<uint32_t*>(ctx->sc_vsmp.p);
      uint32_t* sk = sw + n_range;
      uint8_t* sseg = reinterpret_cast<uint8_t*>(sk + n_range);
      k_val_wsamples<<<val_blocks(n_range), 256, 0, s>>>((uint32_t)n_range, wflag, widx, st, sw, sk, sseg, d_tot + 3);
      ctx->stats.kernel_launches++;
      uint32_t n_w = 0;
      CK(cudaMemcpyAsync(&n_w, d_tot + 3, 4, cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
      if (n_w) {
        const size_t n_a = (size_t)n_w * L;
        if (int rc = env_make_room(ctx, e, n_a, s)) return rc;
        hfb::KinAtArgs a = ka;
        a.n_samples = n_w;
        a.m = sw;
        a.k = sk;
        a.seg = sseg;
        a.tfs = static_cast<hfb_transform*>(e->tf.p) + (e->head - n_a);
        a.handles = static_cast<uint32_t*>(e->h.p) + (e->head - n_a);
        if (int err = hfb::robot_at_launch(a, ctx->num_sms, s))
          return cuda_fail(ctx, static_cast<cudaError_t>(err), "k_robot_at launch");
        ctx->stats.kernel_launches++;
        CK(ctx->sc_vrun.reserve(up((size_t)n_w) + 2 * up((size_t)n_w * 4) + (size_t)n_w * sizeof(hfb_contact)));
        char* r = static_cast<char*>(ctx->sc_vrun.p);
        int8_t* kind = reinterpret_cast<int8_t*>(r);
        uint32_t* first = reinterpret_cast<uint32_t*>(r + up(n_w));
        uint32_t* second = reinterpret_cast<uint32_t*>(r + up(n_w) + up((size_t)n_w * 4));
        hfb_contact* rec = reinterpret_cast<hfb_contact*>(r + up(n_w) + 2 * up((size_t)n_w * 4));
        const hfb_motions_out mo{nullptr, kind, first, second, rec, nullptr, nullptr, nullptr, nullptr};
        std::vector<uint32_t> offsets(n_w + 1);
        for (uint32_t k = 0; k <= n_w; ++k) offsets[k] = k;
        ConfigTpl tw = t;
        tw.g0 = 0;
        tw.ng = n_w;
        EnvCollideMotions q{req, &mo, tw, n_w, offsets.data(), 0, n_w, minus_inf};
        QueryOut inner{s, true};
        if (int rc = q.zero(ctx, inner, n_a)) return rc;
        if (int rc = q.run(ctx, e, n_a, inner)) return rc;
        k_val_witness<<<val_blocks(n_w), 256, 0, s>>>(n_w, (uint32_t)m0, L, sw, kind, first, second, rec, wo);
        ctx->stats.kernel_launches++;
      }
    }
    // the counts: rounds, samples and candidates known here, the unsupported records on the device
    if (o.dev) {
      const uint64_t hv[3] = {n_samples, n_env, n_self};
      uint64_t* dst[3] = {out->n_samples, out->n_env_candidates, out->n_self_candidates};
      if (out->n_rounds) CK(cudaMemcpyAsync(out->n_rounds, &rounds, 4, cudaMemcpyHostToDevice, s));
      for (int k = 0; k < 3; ++k)
        if (dst[k]) CK(cudaMemcpyAsync(dst[k], hv + k, 8, cudaMemcpyHostToDevice, s));
    } else {
      CK(o.copy(out->status, vo.status, n));
      CK(o.copy(out->t_valid, vo.t_valid, n * 8));
      CK(o.copy(out->t_collide, vo.t_collide, n * 8));
      CK(o.copy(out->kind, wo.kind, n));
      CK(o.copy(out->first, wo.first, n * 4));
      CK(o.copy(out->second, wo.second, n * 4));
      CK(o.copy(out->contacts, wo.rec, n * sizeof(hfb_contact)));
    }
    CK(o.copy(out->n_unsupported, d_acc, 8));
    CK(o.finish());
    if (!o.dev) {
      if (out->n_rounds) *out->n_rounds = rounds;
      if (out->n_samples) *out->n_samples = n_samples;
      if (out->n_env_candidates) *out->n_env_candidates = n_env;
      if (out->n_self_candidates) *out->n_self_candidates = n_self;
    }
    return HFB_OK;
  }
  static size_t up(size_t b) { return (b + 255) & ~(size_t)255; }
};

// the arguments of a configurations query beyond the pointers: the layout of A, the configuration range and the template
static int configs_args(hfb_ctx* ctx, size_t n_a, const ConfigTpl& t) {
  if (const char* e = config_range_error(n_a, t.links, t.g0, t.ng, t.n, t.pairs)) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, e);
  return HFB_OK;
}

// hfb_env_collide_motions' and hfb_env_certify_motions' arguments beyond the pointers: the offsets, the motion range,
// then configs_args over the range's configurations (into q.t)
template <class MotionsQuery>
static int motions_args(hfb_ctx* ctx, size_t n_a, MotionsQuery& q) {
  const size_t links = q.t.links, n = q.n_motions;
  const uint32_t* off = q.offsets;
  if (links == 0 || n_a % links) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "n_a is not a multiple of links_per_config");
  if (const char* e = motion_offsets_error(n, off)) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, e);
  if (off[n] != n_a / links) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "motion offsets do not end at n_configs");
  if (q.first_motion > n || q.num_motions > n - q.first_motion)
    return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "motion range past the end");
  q.t.g0 = off[q.first_motion];
  q.t.ng = off[q.first_motion + q.num_motions] - q.t.g0;
  return configs_args(ctx, n_a, q.t);
}

// a query's arguments beyond the pointers: those of a configurations query, or of a motions query
template <class Query>
static int query_args(hfb_ctx* ctx, size_t n_a, Query& q) {
  const ConfigTpl* t = q.tpl();
  return t ? configs_args(ctx, n_a, *t) : HFB_OK;
}
static int query_args(hfb_ctx* ctx, size_t n_a, EnvCollideMotions& q) { return motions_args(ctx, n_a, q); }
static int query_args(hfb_ctx* ctx, size_t n_a, EnvCertifyMotions& q) { return motions_args(ctx, n_a, q); }
// (hfb_env_validate_motions' A is made by the call: only its template, over the robot's links, is the caller's)

// The frame of the hfb_env_* queries (EnvCollide, EnvCollideConfigs, EnvDistance, EnvDistanceConfigs), with their
// pointers checked: the lock, the query's and the env's checks, A uploaded into the env's table in front of B (and
// the template `tpl` of a configurations query into ctx->sc_tpl), then the query.  Host form (Form::host): A and the
// outputs are host memory, the call runs on the context's first stream and blocks, and it returns before the device
// when there is no work.  Device form: they are device memory, the call is ordered on `stream` and records the
// context's device event.
enum class Form { host, device };
template <class Query>
static int env_call(hfb_ctx* ctx, hfb_env* env, Form form, void* stream, size_t n_a, const uint32_t* h_a,
                    const hfb_transform* tf_a, Query q) {
  const bool dev = form == Form::device;
  const ConfigTpl* tpl = q.tpl();
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (int rc = q.check(ctx)) return rc;
  if (int rc = env_ready(ctx, env)) return rc;
  if (n_a > 0xffffffffull || n_a + env->n_b > 0xffffffffull) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "scene too large");
  if (int rc = query_args(ctx, n_a, q)) return rc;
  QueryOut o{dev ? static_cast<cudaStream_t>(stream) : ctx->slots[0].stream, dev};
  if (!dev) {
    if (int rc = check_handles(ctx, h_a, n_a)) return rc;
    if (int rc = q.zero(ctx, o, n_a)) return rc;
    if (q.empty(env, n_a)) return HFB_OK;
  }
  CK(cudaSetDevice(ctx->device));
  if (int rc = after_device_calls(ctx, o.s)) return rc;
  if (dev) {
    if (int rc = q.zero(ctx, o, n_a)) return rc;
    if (q.empty(env, n_a)) return last_device_call(ctx, o.s);
  }
  if (int rc = env_make_room(ctx, env, n_a, o.s)) return rc;
  const size_t off = env->head - n_a;
  const cudaMemcpyKind kind = dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  if (n_a) {  // (hfb_env_validate_motions makes its A itself)
    CK(cudaMemcpyAsync(static_cast<uint32_t*>(env->h.p) + off, h_a, n_a * 4, kind, o.s));
    CK(cudaMemcpyAsync(static_cast<hfb_transform*>(env->tf.p) + off, tf_a, n_a * sizeof(hfb_transform), kind, o.s));
  }
  if (tpl) {
    CK(ctx->sc_tpl.reserve(tpl->n * 8 + 8));
    if (tpl->n) CK(cudaMemcpyAsync(ctx->sc_tpl.p, tpl->pairs, tpl->n * 8, cudaMemcpyHostToDevice, o.s));
  }
  if (int rc = q.run(ctx, env, n_a, o)) return rc;
  return dev ? last_device_call(ctx, o.s) : HFB_OK;
}

extern "C" {

int hfb_env_create(hfb_ctx* ctx, size_t n_b, const uint32_t* handles_b, const hfb_transform* tfs_b, hfb_env** out) {
  if (!ctx || !out || (n_b && (!handles_b || !tfs_b))) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (int rc = check_ready(ctx)) return rc;
  if (n_b > 0xffffffffull) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "scene too large");
  if (int rc = check_handles(ctx, handles_b, n_b)) return rc;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->slots[0].stream;
  if (int rc = after_device_calls(ctx, s)) return rc;
  std::unique_ptr<hfb_env> e(new hfb_env);
  e->n_b = n_b;
  e->handles.assign(handles_b, handles_b + n_b);
  e->commits = ctx->commits;
  e->clears = ctx->clears;
  CK(e->h.reserve(n_b * 4 + 4));
  CK(e->tf.reserve(n_b * sizeof(hfb_transform) + 8));
  CK(e->bb.reserve(n_b * 48 + 8));
  CK(e->grid.reserve(bp_cross_grid_bytes(n_b)));
  if (n_b) {
    CK(cudaMemcpyAsync(e->h.p, handles_b, n_b * 4, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(e->tf.p, tfs_b, n_b * sizeof(hfb_transform), cudaMemcpyHostToDevice, s));
    if (bp_scene_aabbs_launch(ctx->dview.local_aabbs, ctx->dview.nshapes, n_b, static_cast<const uint32_t*>(e->h.p),
                              static_cast<const hfb_transform*>(e->tf.p), static_cast<double*>(e->bb.p), s) != 0)
      return fail(ctx, HFB_ERR_CUDA, "k_scene_aabbs launch failed");
    ctx->stats.kernel_launches++;
  }
  if (int rc = env_build(ctx, e.get(), s)) return rc;
  CK(cudaStreamSynchronize(s));
  ctx->envs.push_back(e.get());
  *out = e.release();
  return HFB_OK;
}

int hfb_env_update(hfb_ctx* ctx, hfb_env* env, size_t m, const uint32_t* indices, const hfb_transform* tfs) {
  if (!ctx || !env || (m && (!indices || !tfs))) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (int rc = env_ready(ctx, env)) return rc;
  std::vector<uint8_t> seen(m ? env->n_b : 0, 0);  // all or nothing: every index checked before anything moves
  for (size_t k = 0; k < m; ++k) {
    if (indices[k] >= env->n_b) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "environment index out of range");
    if (seen[indices[k]]++) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "environment index repeated");
  }
  if (m == 0) return HFB_OK;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->slots[0].stream;
  if (int rc = after_device_calls(ctx, s)) return rc;
  CK(ctx->obj_h.reserve(m * 4 + 4));
  CK(ctx->obj_tf.reserve(m * sizeof(hfb_transform) + 8));
  CK(cudaMemcpyAsync(ctx->obj_h.p, indices, m * 4, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(ctx->obj_tf.p, tfs, m * sizeof(hfb_transform), cudaMemcpyHostToDevice, s));
  if (bp_env_update_launch(ctx->dview.local_aabbs, ctx->dview.nshapes, m, static_cast<const uint32_t*>(ctx->obj_h.p),
                           static_cast<const hfb_transform*>(ctx->obj_tf.p), static_cast<const uint32_t*>(env->h.p) + env->head,
                           static_cast<hfb_transform*>(env->tf.p) + env->head, static_cast<double*>(env->bb.p), s) != 0)
    return fail(ctx, HFB_ERR_CUDA, "k_env_update launch failed");
  ctx->stats.kernel_launches++;
  if (int rc = env_build(ctx, env, s)) return rc;
  CK(cudaStreamSynchronize(s));
  return HFB_OK;
}

int hfb_env_collide(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* handles_a, const hfb_transform* tfs_a,
                    size_t first_a, size_t num_a, const hfb_collision_request* req, const hfb_env_out* out) {
  if (!ctx || !env || !req || !out || (n_a && (!handles_a || !tfs_a))) return HFB_ERR_INVALID_ARGUMENT;
  if (out->capacity && (!out->first || !out->second || !out->contacts)) return HFB_ERR_INVALID_ARGUMENT;
  return env_call(ctx, env, Form::host, nullptr, n_a, handles_a, tfs_a, EnvCollide{req, out, first_a, num_a});
}

int hfb_env_collide_device(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* d_handles_a, const hfb_transform* d_tfs_a,
                           size_t first_a, size_t num_a, const hfb_collision_request* req, const hfb_env_out* d_out,
                           void* stream) {
  if (!ctx || !env || !req || !d_out || (n_a && (!d_handles_a || !d_tfs_a))) return HFB_ERR_INVALID_ARGUMENT;
  if (d_out->capacity && (!d_out->first || !d_out->second || !d_out->contacts)) return HFB_ERR_INVALID_ARGUMENT;
  return env_call(ctx, env, Form::device, stream, n_a, d_handles_a, d_tfs_a, EnvCollide{req, d_out, first_a, num_a});
}

int hfb_env_destroy(hfb_ctx* ctx, hfb_env* env) {
  if (!ctx || !env) return HFB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  auto it = std::find(ctx->envs.begin(), ctx->envs.end(), env);
  if (it == ctx->envs.end()) return fail(ctx, HFB_ERR_INVALID_ARGUMENT, "not an environment of this context");
  CK(cudaSetDevice(ctx->device));
  // what may still read its table: the last device query (each one waits for the one before on another stream) and
  // the host calls' stream
  if (ctx->dev_used) CK(cudaEventSynchronize(ctx->dev_done));
  CK(cudaStreamSynchronize(ctx->slots[0].stream));
  ctx->envs.erase(it);
  delete env;
  return HFB_OK;
}

// A planner's validity check in one call: every configuration of A against the env (hfb_env_collide's pairs) and
// against itself (the template's link pairs per configuration), one verdict per configuration.  The reference asks
// two queries per configuration: DynamicAABBTreeCollisionManager::collide(other_manager, callback) for the
// environment (broadphase_collision_manager.h:94-118) and collide(callback) with a callback that keeps only the
// template's pairs (:104-106), each with CollisionCallBackDefault (default_broadphase_callbacks.cpp:43-60).
int hfb_env_collide_configs(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* handles_a, const hfb_transform* tfs_a,
                            size_t links_per_config, size_t n_self_pairs, const uint32_t* self_pairs, size_t first_config,
                            size_t num_configs, const hfb_collision_request* req, const hfb_configs_out* out) {
  if (!ctx || !env || !req || !out || (n_a && (!handles_a || !tfs_a)) || (n_self_pairs && !self_pairs))
    return HFB_ERR_INVALID_ARGUMENT;
  if (!contacts_ok(out->env) || !contacts_ok(out->self)) return HFB_ERR_INVALID_ARGUMENT;
  return env_call(ctx, env, Form::host, nullptr, n_a, handles_a, tfs_a,
                  EnvCollideConfigs{req, out, {links_per_config, n_self_pairs, self_pairs, first_config, num_configs}});
}

int hfb_env_collide_configs_device(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* d_handles_a,
                                   const hfb_transform* d_tfs_a, size_t links_per_config, size_t n_self_pairs,
                                   const uint32_t* self_pairs, size_t first_config, size_t num_configs,
                                   const hfb_collision_request* req, const hfb_configs_out* d_out, void* stream) {
  if (!ctx || !env || !req || !d_out || (n_a && (!d_handles_a || !d_tfs_a)) || (n_self_pairs && !self_pairs))
    return HFB_ERR_INVALID_ARGUMENT;
  if (!contacts_ok(d_out->env) || !contacts_ok(d_out->self)) return HFB_ERR_INVALID_ARGUMENT;
  return env_call(ctx, env, Form::device, stream, n_a, d_handles_a, d_tfs_a,
                  EnvCollideConfigs{req, d_out, {links_per_config, n_self_pairs, self_pairs, first_config, num_configs}});
}

// A planner's motion validation (hfb_motions_out in include/hppfcl_b200.h): per motion, a run of configurations, the
// first sample whose hfb_env_collide_configs verdict would be 1 and the first colliding pair there -- OMPL's
// DiscreteMotionValidator::checkMotion(s1, s2, lastValid) and hpp-core's discretized path validation over the caller's
// samples.
int hfb_env_collide_motions(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* handles_a, const hfb_transform* tfs_a,
                            size_t links_per_config, size_t n_self_pairs, const uint32_t* self_pairs, size_t n_motions,
                            const uint32_t* motion_offsets, size_t first_motion, size_t num_motions,
                            const hfb_collision_request* req, const hfb_motions_out* out) {
  if (!ctx || !env || !req || !motions_ok(out) || !motion_offsets || (n_a && (!handles_a || !tfs_a)) ||
      (n_self_pairs && !self_pairs))
    return HFB_ERR_INVALID_ARGUMENT;
  return env_call(ctx, env, Form::host, nullptr, n_a, handles_a, tfs_a,
                  EnvCollideMotions{req, out, {links_per_config, n_self_pairs, self_pairs, 0, 0}, n_motions,
                                    motion_offsets, first_motion, num_motions});
}

int hfb_env_collide_motions_device(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* d_handles_a,
                                   const hfb_transform* d_tfs_a, size_t links_per_config, size_t n_self_pairs,
                                   const uint32_t* self_pairs, size_t n_motions, const uint32_t* motion_offsets,
                                   size_t first_motion, size_t num_motions, const hfb_collision_request* req,
                                   const hfb_motions_out* d_out, void* stream) {
  if (!ctx || !env || !req || !motions_ok(d_out) || !motion_offsets || (n_a && (!d_handles_a || !d_tfs_a)) ||
      (n_self_pairs && !self_pairs))
    return HFB_ERR_INVALID_ARGUMENT;
  return env_call(ctx, env, Form::device, stream, n_a, d_handles_a, d_tfs_a,
                  EnvCollideMotions{req, d_out, {links_per_config, n_self_pairs, self_pairs, 0, 0}, n_motions,
                                    motion_offsets, first_motion, num_motions});
}

// A planner's continuous motion validation (hfb_certify_out in include/hppfcl_b200.h): hfb_env_collide_motions'
// first colliding sample per motion, and each segment between consecutive samples certified free from the collide()
// lower bounds of its two end samples and the caller's sweep bounds -- hpp-core's continuous path validation
// (BodyPairCollision's interval from CollisionResult::distance_lower_bound and the maximal velocity).
int hfb_env_certify_motions(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* handles_a, const hfb_transform* tfs_a,
                            const double* sweep, size_t links_per_config, size_t n_self_pairs, const uint32_t* self_pairs,
                            size_t n_motions, const uint32_t* motion_offsets, size_t first_motion, size_t num_motions,
                            const hfb_collision_request* req, const hfb_certify_out* out) {
  if (!ctx || !env || !req || !certify_ok(out) || !motion_offsets || !sweep || (n_a && (!handles_a || !tfs_a)) ||
      (n_self_pairs && !self_pairs))
    return HFB_ERR_INVALID_ARGUMENT;
  return env_call(ctx, env, Form::host, nullptr, n_a, handles_a, tfs_a,
                  EnvCertifyMotions{req, out, {links_per_config, n_self_pairs, self_pairs, 0, 0}, n_motions,
                                    motion_offsets, first_motion, num_motions, sweep});
}

int hfb_env_certify_motions_device(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* d_handles_a,
                                   const hfb_transform* d_tfs_a, const double* d_sweep, size_t links_per_config,
                                   size_t n_self_pairs, const uint32_t* self_pairs, size_t n_motions,
                                   const uint32_t* motion_offsets, size_t first_motion, size_t num_motions,
                                   const hfb_collision_request* req, const hfb_certify_out* d_out, void* stream) {
  if (!ctx || !env || !req || !certify_ok(d_out) || !motion_offsets || !d_sweep || (n_a && (!d_handles_a || !d_tfs_a)) ||
      (n_self_pairs && !self_pairs))
    return HFB_ERR_INVALID_ARGUMENT;
  return env_call(ctx, env, Form::device, stream, n_a, d_handles_a, d_tfs_a,
                  EnvCertifyMotions{req, d_out, {links_per_config, n_self_pairs, self_pairs, 0, 0}, n_motions,
                                    motion_offsets, first_motion, num_motions, d_sweep});
}

// A planner's progressive motion validation (hfb_validate_out in include/hppfcl_b200.h): each motion sampled by the
// robot on the device, certified segment by segment, and the uncertified segments split until each motion is proven
// free, found colliding or at its resolution -- hpp-core's continuous path validation (Dichotomy / Progressive).
int hfb_env_validate_motions(hfb_ctx* ctx, hfb_env* env, hfb_robot* robot, size_t n_motions, const double* q_from,
                             const double* q_to, size_t n_self_pairs, const uint32_t* self_pairs, size_t first_motion,
                             size_t num_motions, const hfb_collision_request* req, const hfb_validate_params* p,
                             const hfb_validate_out* out) {
  if (!ctx || !env || !robot ||
      !validate_ok(n_motions, q_from, q_to, n_self_pairs, self_pairs, first_motion, num_motions, req, p, out))
    return HFB_ERR_INVALID_ARGUMENT;
  return env_call(ctx, env, Form::host, nullptr, 0, nullptr, nullptr,
                  EnvValidateMotions{req, out, {0, n_self_pairs, self_pairs, 0, 0}, robot, n_motions, q_from, q_to,
                                     first_motion, num_motions, *p});
}

int hfb_env_validate_motions_device(hfb_ctx* ctx, hfb_env* env, hfb_robot* robot, size_t n_motions,
                                    const double* d_q_from, const double* d_q_to, size_t n_self_pairs,
                                    const uint32_t* self_pairs, size_t first_motion, size_t num_motions,
                                    const hfb_collision_request* req, const hfb_validate_params* p,
                                    const hfb_validate_out* d_out, void* stream) {
  if (!ctx || !env || !robot ||
      !validate_ok(n_motions, d_q_from, d_q_to, n_self_pairs, self_pairs, first_motion, num_motions, req, p, d_out))
    return HFB_ERR_INVALID_ARGUMENT;
  return env_call(ctx, env, Form::device, stream, 0, nullptr, nullptr,
                  EnvValidateMotions{req, d_out, {0, n_self_pairs, self_pairs, 0, 0}, robot, n_motions, d_q_from,
                                     d_q_to, first_motion, num_motions, *p});
}

// Each A object's nearest B object (hfb_env_distance_out in include/hppfcl_b200.h): the result of
// NaiveCollisionManager::distance(obj, callback) over B (broadphase_bruteforce.cpp:99-110) with a callback that runs
// distance() with a fresh DistanceResult on every pair and keeps the smallest eligible one, the first in B's order on
// ties.  Boxes only skip pairs that cannot be eligible or cannot beat the best found.
int hfb_env_distance(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* handles_a, const hfb_transform* tfs_a,
                     size_t first_a, size_t num_a, const hfb_distance_request* req, double max_distance,
                     const hfb_env_distance_out* out) {
  if (!ctx || !env || !req || !env_distance_ok(out, max_distance) || (n_a && (!handles_a || !tfs_a))) return HFB_ERR_INVALID_ARGUMENT;
  return env_call(ctx, env, Form::host, nullptr, n_a, handles_a, tfs_a,
                  EnvDistance{req, max_distance, out, first_a, num_a});
}

int hfb_env_distance_device(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* d_handles_a, const hfb_transform* d_tfs_a,
                            size_t first_a, size_t num_a, const hfb_distance_request* req, double max_distance,
                            const hfb_env_distance_out* d_out, void* stream) {
  if (!ctx || !env || !req || !env_distance_ok(d_out, max_distance) || (n_a && (!d_handles_a || !d_tfs_a)))
    return HFB_ERR_INVALID_ARGUMENT;
  return env_call(ctx, env, Form::device, stream, n_a, d_handles_a, d_tfs_a,
                  EnvDistance{req, max_distance, d_out, first_a, num_a});
}

// Each configuration's clearance (hfb_configs_distance_out in include/hppfcl_b200.h): the nearest of its environment
// pairs (hfb_env_distance's) and its self pairs (the template's), the environment first on ties -- what a planner's
// clearance(state) is, the smaller of MoveIt's distanceRobot and distanceSelf.
int hfb_env_distance_configs(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* handles_a, const hfb_transform* tfs_a,
                             size_t links_per_config, size_t n_self_pairs, const uint32_t* self_pairs, size_t first_config,
                             size_t num_configs, const hfb_distance_request* req, double max_distance,
                             const hfb_configs_distance_out* out) {
  if (!ctx || !env || !req || !configs_distance_ok(out, max_distance) || (n_a && (!handles_a || !tfs_a)) ||
      (n_self_pairs && !self_pairs))
    return HFB_ERR_INVALID_ARGUMENT;
  return env_call(ctx, env, Form::host, nullptr, n_a, handles_a, tfs_a,
                  EnvDistanceConfigs{req, max_distance, out, {links_per_config, n_self_pairs, self_pairs, first_config, num_configs}});
}

int hfb_env_distance_configs_device(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* d_handles_a,
                                    const hfb_transform* d_tfs_a, size_t links_per_config, size_t n_self_pairs,
                                    const uint32_t* self_pairs, size_t first_config, size_t num_configs,
                                    const hfb_distance_request* req, double max_distance,
                                    const hfb_configs_distance_out* d_out, void* stream) {
  if (!ctx || !env || !req || !configs_distance_ok(d_out, max_distance) || (n_a && (!d_handles_a || !d_tfs_a)) ||
      (n_self_pairs && !self_pairs))
    return HFB_ERR_INVALID_ARGUMENT;
  return env_call(ctx, env, Form::device, stream, n_a, d_handles_a, d_tfs_a,
                  EnvDistanceConfigs{req, max_distance, d_out, {links_per_config, n_self_pairs, self_pairs, first_config, num_configs}});
}
}  // extern "C"
