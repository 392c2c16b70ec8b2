// Device broadphase: scene boxes, uniform grid, pair sweep (design and the reference it stands in for:
// hfb_broadphase.cuh).  Everything stays on the device: the pair list feeds hfb_batch_*_objects_device directly.
#include <cfloat>

#include <cub/cub.cuh>

#include "hfb_broadphase.cuh"
#include "hfb_broadphase.h"

namespace hfb {

namespace {

constexpr unsigned kMaxCells = 2097152u;

// world-space box of one object (k_scene_aabbs, k_env_update)
__device__ __forceinline__ void scene_aabb(const double* local, uint32_t nshapes, uint32_t h, const hfb_transform& tf,
                                           double* o) {
  if (h >= nshapes) {  // no such geometry: an empty box that overlaps nothing
    for (int k = 0; k < 3; ++k) {
      o[k] = DBL_MAX;
      o[3 + k] = -DBL_MAX;
    }
    return;
  }
  const double* l = local + 6 * (size_t)h;
  if (!(l[0] <= l[3])) {  // node type without a local box (NaN / inverted marker)
    for (int k = 0; k < 3; ++k) {
      o[k] = DBL_MAX;
      o[3 + k] = -DBL_MAX;
    }
    return;
  }
  object_aabb(l, l + 3, tf, o);
}
__global__ void __launch_bounds__(256) k_scene_aabbs(const double* local, uint32_t nshapes, unsigned n,
                                                     const uint32_t* handles, const hfb_transform* tfs, double* out) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  scene_aabb(local, nshapes, handles[i], tfs[i], out + 6 * (size_t)i);
}
// hfb_env_update: m new poses scattered into the resident table (index idx[k] of B), and those m boxes recomputed
__global__ void __launch_bounds__(256) k_env_update(const double* local, uint32_t nshapes, unsigned m, const uint32_t* idx,
                                                    const hfb_transform* tfs_new, const uint32_t* handles,
                                                    hfb_transform* tfs, double* bb) {
  const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= m) return;
  const unsigned i = idx[k];
  const hfb_transform tf = tfs_new[k];
  tfs[i] = tf;
  scene_aabb(local, nshapes, handles[i], tf, bb + 6 * (size_t)i);
}

struct Bounds {  // centres' box and the largest extent
  double lo[3], hi[3], ext;
};
__device__ __forceinline__ void bounds_merge(Bounds& a, const Bounds& b) {
  for (int k = 0; k < 3; ++k) {
    a.lo[k] = b.lo[k] < a.lo[k] ? b.lo[k] : a.lo[k];
    a.hi[k] = b.hi[k] > a.hi[k] ? b.hi[k] : a.hi[k];
  }
  a.ext = b.ext > a.ext ? b.ext : a.ext;
}
__device__ __forceinline__ Bounds bounds_empty() {
  Bounds b;
  for (int k = 0; k < 3; ++k) {
    b.lo[k] = DBL_MAX;
    b.hi[k] = -DBL_MAX;
  }
  b.ext = 0;
  return b;
}
__device__ Bounds block_bounds(Bounds v) {
  __shared__ Bounds sh[8];
  for (int off = 16; off > 0; off >>= 1) {
    Bounds o;
    for (int k = 0; k < 3; ++k) {
      o.lo[k] = __shfl_xor_sync(0xffffffffu, v.lo[k], off);
      o.hi[k] = __shfl_xor_sync(0xffffffffu, v.hi[k], off);
    }
    o.ext = __shfl_xor_sync(0xffffffffu, v.ext, off);
    bounds_merge(v, o);
  }
  if ((threadIdx.x & 31u) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    v = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : bounds_empty();
    for (int off = 4; off > 0; off >>= 1) {
      Bounds o;
      for (int k = 0; k < 3; ++k) {
        o.lo[k] = __shfl_xor_sync(0xffffffffu, v.lo[k], off);
        o.hi[k] = __shfl_xor_sync(0xffffffffu, v.hi[k], off);
      }
      o.ext = __shfl_xor_sync(0xffffffffu, v.ext, off);
      bounds_merge(v, o);
    }
  }
  return v;  // valid in thread 0
}
__global__ void __launch_bounds__(256) k_bounds_partial(const double* bb, unsigned n, Bounds* part) {
  Bounds v = bounds_empty();
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double* b = bb + 6 * (size_t)i;
    if (aabb_empty(b) || aabb_unbounded(b)) continue;  // no box / a halfspace or plane: not in the grid
    Bounds o;
    for (int k = 0; k < 3; ++k) {
      o.lo[k] = o.hi[k] = 0.5 * (b[k] + b[3 + k]);
      const double e = b[3 + k] - b[k];
      o.ext = (k == 0 || e > o.ext) ? e : o.ext;
    }
    bounds_merge(v, o);
  }
  v = block_bounds(v);
  if (threadIdx.x == 0) part[blockIdx.x] = v;
}
// one block: final merge, then the grid (make_grid of hfb_broadphase.cuh) and the zeroed pair counter
__global__ void __launch_bounds__(256) k_make_grid(const Bounds* part, unsigned nparts, BroadGrid* grid, unsigned* n_pairs,
                                                   unsigned* n_unbounded) {
  Bounds v = bounds_empty();
  for (unsigned i = threadIdx.x; i < nparts; i += blockDim.x) bounds_merge(v, part[i]);
  v = block_bounds(v);
  if (threadIdx.x == 0) {
    BroadGrid g;
    if (!(v.lo[0] <= v.hi[0])) {  // no boxes at all
      for (int k = 0; k < 3; ++k) {
        v.lo[k] = v.hi[k] = 0;
      }
    }
    grid_fit(v.lo, v.hi, v.ext > 0 ? v.ext : 1.0, g);
    *grid = g;
    *n_pairs = 0u;
    *n_unbounded = 0u;
  }
}
// cell of every object; the unbounded ones (cell 0xfffffffe) are listed from the END of `order` backwards.
// max_ext (cross form only, else null): boxes wider than *max_ext are listed with the unbounded ones
__global__ void __launch_bounds__(256) k_cell_hist(const double* bb, unsigned n, const BroadGrid* grid, unsigned* cell,
                                                   unsigned* count, unsigned* order, unsigned* n_unbounded,
                                                   const double* max_ext) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* b = bb + 6 * (size_t)i;
  if (aabb_empty(b)) {
    cell[i] = 0xffffffffu;  // empty box: in no cell
    return;
  }
  if (aabb_unbounded(b) || (max_ext && box_extent(b) > *max_ext)) {
    cell[i] = 0xfffffffeu;
    order[n - 1u - atomicAdd(n_unbounded, 1u)] = i;
    return;
  }
  const unsigned c = grid_cell(*grid, b);
  cell[i] = c;
  atomicAdd(count + c, 1u);
}
__global__ void __launch_bounds__(256) k_cell_scatter(const unsigned* cell, unsigned n, const unsigned* start,
                                                      unsigned* cursor, unsigned* order) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || cell[i] >= 0xfffffffeu) return;
  order[start[cell[i]] + atomicAdd(cursor + cell[i], 1u)] = i;
}
// one object per thread: the 27 cells around its own, partners with a larger index
__global__ void __launch_bounds__(128) k_sweep(const double* bb, unsigned n, unsigned i_lo, const BroadGrid* grid,
                                               const unsigned* cell, const unsigned* start, const unsigned* order,
                                               uint32_t* first, uint32_t* second, unsigned capacity, unsigned* n_pairs) {
  // n: one past the last object this launch reports pairs for (as their smaller index); i_lo: the first one
  const unsigned i = i_lo + blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned lane = threadIdx.x & 31u;
  const BroadGrid g = *grid;
  const bool live = i < n && cell[i] < 0xfffffffeu;
  double mine[6] = {0, 0, 0, 0, 0, 0};
  int cx = 0, cy = 0, cz = 0;
  if (live) {
    for (int k = 0; k < 6; ++k) mine[k] = bb[6 * (size_t)i + k];
    const unsigned c = cell[i];
    cx = (int)(c % (unsigned)g.dim[0]);
    cy = (int)((c / (unsigned)g.dim[0]) % (unsigned)g.dim[1]);
    cz = (int)(c / ((unsigned)g.dim[0] * (unsigned)g.dim[1]));
  }
  for (int d = 0; d < 27; ++d) {
    const int x = cx + d % 3 - 1, y = cy + (d / 3) % 3 - 1, z = cz + d / 9 - 1;
    const bool in = live && x >= 0 && y >= 0 && z >= 0 && x < g.dim[0] && y < g.dim[1] && z < g.dim[2];
    unsigned q = 0, qe = 0;
    if (in) {
      const size_t nc = ((size_t)z * g.dim[1] + y) * g.dim[0] + x;
      q = start[nc];
      qe = start[nc + 1];
    }
    // the lanes of a warp walk their cells side by side; hits are appended with one counter bump per warp and round
    while (__any_sync(0xffffffffu, q < qe)) {
      bool hit = false;
      unsigned j = 0;
      if (q < qe) {
        j = order[q];
        ++q;
        hit = j > i && aabb_overlap(mine, bb + 6 * (size_t)j);
      }
      const unsigned m = __ballot_sync(0xffffffffu, hit);
      if (m) {
        unsigned base = 0;
        if (lane == (unsigned)(__ffs(m) - 1)) base = atomicAdd(n_pairs, (unsigned)__popc(m));
        base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
        const unsigned pos = base + (unsigned)__popc(m & ((1u << lane) - 1u));
        if (hit && pos < capacity) {
          first[pos] = i;
          second[pos] = j;
        }
      }
    }
  }
}

// the unbounded objects (halfspaces, planes) against every object: thread per object j, loop over the few unbounded u;
// the pair is this launch's when its smaller index lies in [i_lo, i_hi), a pair of two unbounded objects is reported
// from its smaller index only
__global__ void __launch_bounds__(128) k_sweep_unbounded(const double* bb, unsigned n, unsigned i_lo, unsigned i_hi,
                                                         const unsigned* cell, const unsigned* order, const unsigned* n_unbounded,
                                                         uint32_t* first, uint32_t* second, unsigned capacity, unsigned* n_pairs) {
  const unsigned nu = *n_unbounded;
  if (nu == 0) return;
  const unsigned lane = threadIdx.x & 31u;
  const unsigned j0 = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned jend = (n + 31u) & ~31u;  // (warp-uniform trip count for the ballots)
  for (unsigned j = j0; j < jend; j += gridDim.x * blockDim.x) {
    const bool jl = j < n && cell[j] != 0xffffffffu;
    double mine[6] = {0, 0, 0, 0, 0, 0};
    if (jl)
      for (int k = 0; k < 6; ++k) mine[k] = bb[6 * (size_t)j + k];
    for (unsigned q = 0; q < nu; ++q) {
      const unsigned u = order[n - 1u - q];
      const unsigned lo = u < j ? u : j, hi = u < j ? j : u;
      const bool hit = jl && j != u && !(cell[j] == 0xfffffffeu && j < u) && lo >= i_lo && lo < i_hi &&
                       aabb_overlap(mine, bb + 6 * (size_t)u);
      const unsigned m = __ballot_sync(0xffffffffu, hit);
      if (m) {
        unsigned base = 0;
        if (lane == (unsigned)(__ffs(m) - 1)) base = atomicAdd(n_pairs, (unsigned)__popc(m));
        base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
        const unsigned pos = base + (unsigned)__popc(m & ((1u << lane) - 1u));
        if (hit && pos < capacity) {
          first[pos] = lo;
          second[pos] = hi;
        }
      }
    }
  }
}

// ---- cross form (design: hfb_broadphase.cuh, broadphase_cross_pairs_host) -------------------------------------
struct CrossGrid {  // B's grid and its cell size (the largest extent a box in the grid may have)
  BroadGrid g;
  double cell;
};

// one warp's hits appended with one counter bump; every lane of the warp must call it
__device__ __forceinline__ void append_pair(bool hit, unsigned a, unsigned b, uint32_t* first, uint32_t* second,
                                            unsigned capacity, unsigned* n_pairs) {
  const unsigned m = __ballot_sync(0xffffffffu, hit);
  if (!m) return;
  const unsigned lane = threadIdx.x & 31u;
  unsigned base = 0;
  if (lane == (unsigned)(__ffs(m) - 1)) base = atomicAdd(n_pairs, (unsigned)__popc(m));
  base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
  const unsigned pos = base + (unsigned)__popc(m & ((1u << lane) - 1u));
  if (hit && pos < capacity) {
    first[pos] = a;
    second[pos] = b;
  }
}

// B's centres box and the log2 histogram of B's extents (bounded, non-empty boxes)
__global__ void __launch_bounds__(256) k_cross_bounds_partial(const double* bb, unsigned n, Bounds* part, unsigned* hist) {
  __shared__ unsigned sh_hist[kExtBins];
  for (unsigned k = threadIdx.x; k < (unsigned)kExtBins; k += blockDim.x) sh_hist[k] = 0;
  __syncthreads();
  Bounds v = bounds_empty();
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double* b = bb + 6 * (size_t)i;
    if (aabb_empty(b) || aabb_unbounded(b)) continue;
    Bounds o;
    for (int k = 0; k < 3; ++k) o.lo[k] = o.hi[k] = 0.5 * (b[k] + b[3 + k]);
    o.ext = 0;
    bounds_merge(v, o);
    atomicAdd(sh_hist + extent_bin(box_extent(b)), 1u);
  }
  v = block_bounds(v);  // (synchronises the block: the histogram is complete after it)
  if (threadIdx.x == 0) part[blockIdx.x] = v;
  for (unsigned k = threadIdx.x; k < (unsigned)kExtBins; k += blockDim.x)
    if (sh_hist[k]) atomicAdd(hist + k, sh_hist[k]);
}
// one block: final merge, the cell from the histogram, the grid, and the zeroed counters (pairs, B oversize, A brute)
__global__ void __launch_bounds__(256) k_cross_grid(const Bounds* part, unsigned nparts, const unsigned* hist, CrossGrid* cg,
                                                    unsigned* n_pairs, unsigned* counters) {
  Bounds v = bounds_empty();
  for (unsigned i = threadIdx.x; i < nparts; i += blockDim.x) bounds_merge(v, part[i]);
  v = block_bounds(v);
  if (threadIdx.x == 0) {
    unsigned total = 0;
    for (int k = 0; k < kExtBins; ++k) total += hist[k];
    if (!(v.lo[0] <= v.hi[0]))
      for (int k = 0; k < 3; ++k) v.lo[k] = v.hi[k] = 0;
    CrossGrid c;
    c.cell = cross_grid_fit(v.lo, v.hi, hist, total, c.g);
    *cg = c;
    *n_pairs = 0u;
    counters[0] = counters[1] = 0u;
  }
}
// one A object per thread, i in [a_lo, a_hi): the B objects in the grid rows its widened box covers, then B's oversize
// and unbounded ones (listed from the end of `order`); A objects that need the whole of B are listed in `brute`
__global__ void __launch_bounds__(128) k_cross_sweep(const double* ba, unsigned a_lo, unsigned a_hi, const double* bb,
                                                     unsigned nb, const CrossGrid* cgp, const unsigned* start,
                                                     const unsigned* order, unsigned* counters, unsigned* brute,
                                                     uint32_t* first, uint32_t* second, unsigned second_base,
                                                     unsigned capacity, unsigned* n_pairs) {
  const unsigned i = a_lo + blockIdx.x * blockDim.x + threadIdx.x;
  const CrossGrid cg = *cgp;
  bool live = i < a_hi && !aabb_empty(ba + 6 * (size_t)i);
  double mine[6] = {0, 0, 0, 0, 0, 0};
  int c0[3] = {0, 0, 0}, c1[3] = {-1, -1, -1};
  if (live) {
    for (int k = 0; k < 6; ++k) mine[k] = ba[6 * (size_t)i + k];
    if (aabb_unbounded(mine) || cross_query_cells(cg.g, cg.cell, mine, c0, c1) > kCrossScanRows) {
      brute[atomicAdd(counters + 1, 1u)] = i;
      live = false;
    }
  }
  // the lanes walk their rows side by side: a lane whose row is done fetches its next one
  int y = c0[1], z = c0[2];
  unsigned q = 0, qe = 0;
  bool more = live;
  while (__any_sync(0xffffffffu, more)) {
    bool hit = false;
    unsigned j = 0;
    if (more) {
      while (q >= qe) {
        if (z > c1[2]) {
          more = false;
          break;
        }
        const size_t row = ((size_t)z * cg.g.dim[1] + y) * cg.g.dim[0];
        q = start[row + c0[0]];
        qe = start[row + c1[0] + 1];
        if (++y > c1[1]) {
          y = c0[1];
          ++z;
        }
      }
      if (more) {
        j = order[q++];
        hit = aabb_overlap(mine, bb + 6 * (size_t)j);
      }
    }
    append_pair(hit, i, j + second_base, first, second, capacity, n_pairs);
  }
  const unsigned nover = counters[0];
  for (unsigned k = 0; k < nover; ++k) {
    const unsigned u = order[nb - 1u - k];
    append_pair(live && aabb_overlap(mine, bb + 6 * (size_t)u), i, u + second_base, first, second, capacity, n_pairs);
  }
}
// the A objects listed in `brute` against every B object: thread per B object j, loop over the (few) listed ones
__global__ void __launch_bounds__(128) k_cross_brute(const double* ba, const double* bb, unsigned nb, const unsigned* counters,
                                                     const unsigned* brute, uint32_t* first, uint32_t* second,
                                                     unsigned second_base, unsigned capacity, unsigned* n_pairs) {
  const unsigned nbr = counters[1];
  if (nbr == 0) return;
  const unsigned jend = (nb + 31u) & ~31u;  // (warp-uniform trip count for the ballots)
  for (unsigned j = blockIdx.x * blockDim.x + threadIdx.x; j < jend; j += gridDim.x * blockDim.x) {
    const bool jl = j < nb && !aabb_empty(bb + 6 * (size_t)j);
    double mine[6] = {0, 0, 0, 0, 0, 0};
    if (jl)
      for (int k = 0; k < 6; ++k) mine[k] = bb[6 * (size_t)j + k];
    for (unsigned q = 0; q < nbr; ++q) {
      const unsigned a = brute[q];
      append_pair(jl && aabb_overlap(ba + 6 * (size_t)a, mine), a, j + second_base, first, second, capacity, n_pairs);
    }
  }
}

// the resident environment's query: the A objects k_cross_sweep handles (in range, with a box, not on the brute list)
// against B's oversize and unbounded objects (the end of `order`), one thread per pair -- k_cross_sweep's own loop over
// that list is one serial chain per A object, which a few configurations against a list of about a thousand tables
// cannot hide
__global__ void __launch_bounds__(128) k_cross_oversize(const double* ba, unsigned a_lo, unsigned a_hi, const double* bb,
                                                        unsigned nb, const CrossGrid* cgp, const unsigned* order,
                                                        const unsigned* counters, uint32_t* first, uint32_t* second,
                                                        unsigned second_base, unsigned capacity, unsigned* n_pairs) {
  const unsigned na = a_hi - a_lo;
  const size_t total = (size_t)na * counters[0];
  const size_t tend = (total + 31u) & ~(size_t)31;  // (warp-uniform trip count for the ballots)
  const CrossGrid cg = *cgp;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < tend; t += (size_t)gridDim.x * blockDim.x) {
    bool hit = false;
    unsigned i = 0, u = 0;
    if (t < total) {
      i = a_lo + (unsigned)(t % na);
      u = order[nb - 1u - (unsigned)(t / na)];
      const double* a = ba + 6 * (size_t)i;
      int c0[3], c1[3];
      hit = !aabb_empty(a) && !aabb_unbounded(a) && cross_query_cells(cg.g, cg.cell, a, c0, c1) <= kCrossScanRows &&
            aabb_overlap(a, bb + 6 * (size_t)u);
    }
    append_pair(hit, i, u + second_base, first, second, capacity, n_pairs);
  }
}

// the self pairs of configurations [g0, g0 + total / P) (config_pair): one thread per (configuration, template pair),
// appended to the same counter as whatever ran before on it
__global__ void __launch_bounds__(128) k_config_pairs(const double* bb, unsigned links, const uint32_t* tpl, unsigned n_tpl,
                                                      unsigned g0, size_t total, uint32_t* first, uint32_t* second,
                                                      unsigned capacity, unsigned* n_pairs) {
  const size_t tend = (total + 31u) & ~(size_t)31;  // (warp-uniform trip count for the ballots)
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < tend; t += (size_t)gridDim.x * blockDim.x) {
    bool hit = false;
    uint32_t a = 0, b = 0;
    if (t < total) hit = config_pair(bb, links, tpl, n_tpl, g0, t, &a, &b);
    append_pair(hit, a, b, first, second, capacity, n_pairs);
  }
}

// k_config_pairs with each pair's template entry in `entry` at its position in the list (hfb_env_collide_motions' tie
// order)
__global__ void __launch_bounds__(128) k_config_entry_pairs(const double* bb, unsigned links, const uint32_t* tpl,
                                                            unsigned n_tpl, unsigned g0, size_t total, uint32_t* first,
                                                            uint32_t* second, uint32_t* entry, unsigned capacity,
                                                            unsigned* n_pairs) {
  const size_t tend = (total + 31u) & ~(size_t)31;  // (warp-uniform trip count for the ballots)
  const unsigned lane = threadIdx.x & 31u;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < tend; t += (size_t)gridDim.x * blockDim.x) {
    bool hit = false;
    uint32_t a = 0, b = 0;
    if (t < total) hit = config_pair(bb, links, tpl, n_tpl, g0, t, &a, &b);
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (!m) continue;
    unsigned base = 0;
    if (lane == (unsigned)(__ffs(m) - 1)) base = atomicAdd(n_pairs, (unsigned)__popc(m));
    base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
    const unsigned pos = base + (unsigned)__popc(m & ((1u << lane) - 1u));
    if (hit && pos < capacity) {
      first[pos] = a;
      second[pos] = b;
      entry[pos] = (uint32_t)(t % n_tpl);
    }
  }
}

// ---- hfb_env_distance's rounds (BpDistState in hfb_broadphase.h) -------------------------------------------------
// order-preserving key of a double: keys compare as the values do, -0 and +0 share one key (NaN is never keyed)
__device__ __forceinline__ unsigned long long dist_key(double d) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(d == 0.0 ? 0.0 : d);
  return (b >> 63) ? ~b : b | 0x8000000000000000ull;
}
// the value of a key; the initial keys ~0 and 0 come back as NaN, which no comparison takes
__device__ __forceinline__ double key_value(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? k & 0x7fffffffffffffffull : ~k));
}
__device__ __forceinline__ double dist_radius(double cell, int round, double maxd) {
  const double r = ldexp(cell, 3 * round);
  return r < maxd ? r : maxd;
}
// box a widened by r on every side, rounded outward: a B box that does not overlap it is more than r away from a
__device__ __forceinline__ void dist_inflate(const double* a, double r, double* o) {
  for (int k = 0; k < 3; ++k) {
    o[k] = __dsub_rd(a[k], r);
    o[3 + k] = __dadd_ru(a[3 + k], r);
  }
}
// the widened box overlaps every (non-empty) box of B: it reaches past the smallest maximum and the largest minimum
__device__ __forceinline__ bool dist_covers(const double* a, double r, const unsigned long long* reach) {
  double o[6];
  dist_inflate(a, r, o);
  for (int k = 0; k < 3; ++k)
    if (o[k] > key_value(reach[k]) || o[3 + k] < key_value(reach[3 + k])) return false;
  return true;
}
__device__ __forceinline__ bool dist_eligible(double d, uint32_t status, double maxd) {
  return ((status >> 16) & 0xffu) != HFB_PATH_UNSUPPORTED && d <= maxd;  // (NaN: never)
}

// a fresh record and no best for every A object; the ones in [a_lo, a_hi) open, against all of B in round 0 when
// their box cannot bound a distance (no box, or a coordinate that is not finite)
__global__ void __launch_bounds__(256) k_dist_init(const double* ba, unsigned n_a, unsigned a_lo, unsigned a_hi,
                                                   BpDistState st) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_a) return;
  uint8_t s = 0;
  if (i >= a_lo && i < a_hi) {
    const double* b = ba + 6 * (size_t)i;
    bool whole = aabb_empty(b);
    for (int k = 0; k < 6; ++k) whole = whole || !isfinite(b[k]);
    s = whole ? 2 : 1;
  }
  st.state[i] = s;
  st.key[i] = ~0ull;
  st.nearest[i] = -1;
  hfb_distance_result r;  // DistanceResult's initial values (collision_data.h:1090-1096)
  r.min_distance = DBL_MAX;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  for (int k = 0; k < 3; ++k) r.p1[k] = r.p2[k] = r.normal[k] = nan;
  r.b1 = r.b2 = -1;
  r.status = r.iterations = 0;
  st.rec[i] = r;
}
// B's reach (reach[k]: smallest maximum, reach[3 + k]: largest minimum along axis k; NaN coordinates left out, as they
// never fail an overlap test)
__global__ void __launch_bounds__(256) k_dist_reach(const double* bb, unsigned nb, unsigned long long* reach) {
  unsigned long long v[6] = {~0ull, ~0ull, ~0ull, 0ull, 0ull, 0ull};
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < nb; i += gridDim.x * blockDim.x) {
    const double* b = bb + 6 * (size_t)i;
    if (aabb_empty(b)) continue;
    for (int k = 0; k < 3; ++k) {
      if (b[3 + k] == b[3 + k]) v[k] = min(v[k], dist_key(b[3 + k]));
      if (b[k] == b[k]) v[3 + k] = max(v[3 + k], dist_key(b[k]));
    }
  }
  for (int off = 16; off > 0; off >>= 1)
    for (int k = 0; k < 6; ++k) {
      const unsigned long long o = __shfl_xor_sync(0xffffffffu, v[k], off);
      v[k] = k < 3 ? min(v[k], o) : max(v[k], o);
    }
  if ((threadIdx.x & 31u) == 0)
    for (int k = 0; k < 3; ++k) {
      atomicMin(reach + k, v[k]);
      atomicMax(reach + 3 + k, v[3 + k]);
    }
}
__global__ void __launch_bounds__(256) k_dist_boxes(const double* ba, unsigned a_lo, unsigned a_hi, const CrossGrid* cgp,
                                                    double maxd, int round, BpDistState st, double* bq, unsigned* n_open) {
  const unsigned i = a_lo + blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a_hi) return;
  const double cell = cgp->cell;
  const double* a = ba + 6 * (size_t)i;
  uint8_t s = st.state[i];
  if (round > 0 && s == 2) s = 0;  // it ran against all of B
  if (round > 0 && s == 1) {
    const double r = dist_radius(cell, round - 1, maxd);
    if (st.key[i] <= dist_key(r) || r >= maxd || dist_covers(a, r, st.reach)) s = 0;
  }
  st.state[i] = s;
  double* o = bq + 6 * (size_t)i;
  if (s == 0) {
    for (int k = 0; k < 3; ++k) {
      o[k] = DBL_MAX;
      o[3 + k] = -DBL_MAX;
    }
    return;
  }
  st.prev[i] = st.key[i];
  st.jround[i] = 0xffffffffu;
  if (s == 2)
    for (int k = 0; k < 3; ++k) {
      o[k] = -INFINITY;
      o[3 + k] = INFINITY;
    }
  else
    dist_inflate(a, dist_radius(cell, round, maxd), o);
  atomicAdd(n_open, 1u);
}
__global__ void __launch_bounds__(256) k_dist_filter(const uint32_t* pf, const uint32_t* ps, const unsigned* n_raw,
                                                     unsigned cap, const double* ba, const double* bb, unsigned second_base,
                                                     const CrossGrid* cgp, double maxd, int round, uint32_t* kf, uint32_t* ks,
                                                     unsigned* n_kept) {
  const unsigned n = *n_raw < cap ? *n_raw : cap;
  const unsigned nend = (n + 31u) & ~31u;  // (warp-uniform trip count for the ballots)
  const double r = round > 0 ? dist_radius(cgp->cell, round - 1, maxd) : 0.0;
  for (unsigned t = blockIdx.x * blockDim.x + threadIdx.x; t < nend; t += gridDim.x * blockDim.x) {
    bool keep = false;
    unsigned i = 0, j = 0;
    if (t < n) {
      i = pf[t];
      j = ps[t];
      keep = true;
      if (round > 0) {  // (an object open in this round was open in the one before)
        double o[6];
        dist_inflate(ba + 6 * (size_t)i, r, o);
        keep = !aabb_overlap(o, bb + 6 * (size_t)(j - second_base));
      }
    }
    append_pair(keep, i, j, kf, ks, cap, n_kept);
  }
}
// three passes over a round's records: the smallest key per A object, the lowest index in B at that key, then the
// winner against the best of the rounds before (strictly better, or equal with a lower index)
__global__ void __launch_bounds__(256) k_dist_min(const hfb_distance_result* r, const uint32_t* pf, unsigned n, double maxd,
                                                  unsigned long long* key, unsigned* n_unsupported) {
  const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
  bool unsup = false;
  if (p < n) {
    const double d = r[p].min_distance;
    const uint32_t status = r[p].status;
    unsup = ((status >> 16) & 0xffu) == HFB_PATH_UNSUPPORTED;
    if (dist_eligible(d, status, maxd)) atomicMin(key + pf[p], dist_key(d));
  }
  const unsigned m = __ballot_sync(0xffffffffu, unsup);
  if (m && (threadIdx.x & 31u) == 0) atomicAdd(n_unsupported, (unsigned)__popc(m));
}
__global__ void __launch_bounds__(256) k_dist_argmin(const hfb_distance_result* r, const uint32_t* pf, const uint32_t* ps,
                                                     unsigned n, unsigned second_base, double maxd, BpDistState st) {
  const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const double d = r[p].min_distance;
  const unsigned i = pf[p];
  if (dist_eligible(d, r[p].status, maxd) && dist_key(d) == st.key[i]) atomicMin(st.jround + i, ps[p] - second_base);
}
__global__ void __launch_bounds__(256) k_dist_take(const hfb_distance_result* r, const uint32_t* pf, const uint32_t* ps,
                                                   unsigned n, unsigned second_base, double maxd, BpDistState st) {
  const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const double d = r[p].min_distance;
  const unsigned i = pf[p], j = ps[p] - second_base;
  if (!dist_eligible(d, r[p].status, maxd) || dist_key(d) != st.key[i] || j != st.jround[i]) return;
  // (one pair per A object gets here; nearest -1 compares as the largest index)
  if (st.key[i] < st.prev[i] || (uint32_t)st.nearest[i] > j) {
    st.nearest[i] = (int32_t)j;
    st.rec[i] = r[p];
  }
}

// ---- hfb_env_distance_configs (BpConfigDist in hfb_broadphase.h) --------------------------------------------------
// the self pairs config_dist_pair runs, one thread per (configuration, template entry), each with its template entry in
// `entry` at its position in the list (the reduction's tie order)
__global__ void __launch_bounds__(128) k_config_dist_pairs(const double* bb, unsigned links, const uint32_t* tpl,
                                                           unsigned n_tpl, unsigned g0, size_t total, double maxd,
                                                           uint32_t* first, uint32_t* second, uint32_t* entry,
                                                           unsigned capacity, unsigned* n_pairs) {
  const size_t tend = (total + 31u) & ~(size_t)31;  // (warp-uniform trip count for the ballots)
  const unsigned lane = threadIdx.x & 31u;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < tend; t += (size_t)gridDim.x * blockDim.x) {
    bool hit = false;
    uint32_t a = 0, b = 0;
    if (t < total) hit = config_dist_pair(bb, links, tpl, n_tpl, g0, t, maxd, &a, &b);
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (!m) continue;
    unsigned base = 0;
    if (lane == (unsigned)(__ffs(m) - 1)) base = atomicAdd(n_pairs, (unsigned)__popc(m));
    base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
    const unsigned pos = base + (unsigned)__popc(m & ((1u << lane) - 1u));
    if (hit && pos < capacity) {
      first[pos] = a;
      second[pos] = b;
      entry[pos] = (uint32_t)(t % n_tpl);
    }
  }
}
__global__ void __launch_bounds__(256) k_cfg_init(unsigned n, BpConfigDist cs) {
  const unsigned g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n) return;
  cs.key[g] = ~0ull;
  cs.ord[g] = ~0ull;
  cs.kind[g] = -1;
  cs.first[g] = cs.second[g] = 0xffffffffu;
  hfb_distance_result r;  // DistanceResult's initial values, as k_dist_init writes them
  r.min_distance = DBL_MAX;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  for (int k = 0; k < 3; ++k) r.p1[k] = r.p2[k] = r.normal[k] = nan;
  r.b1 = r.b2 = -1;
  r.status = r.iterations = 0;
  cs.rec[g] = r;
}
// the items of one chunk's reduction: t < n_links is link a_lo + t with the best its rounds left (ordinal: the link
// index within its configuration), the rest are self records (ordinal L + template entry); false when not eligible
struct CfgItems {
  unsigned a_lo, n_links, links, n_self;
  const hfb_distance_result* r;
  const uint32_t *pf, *ps, *pk;
  double maxd;
};
__device__ __forceinline__ bool cfg_item(const BpDistState& st, const CfgItems& it, size_t t, unsigned* g,
                                         unsigned long long* key, unsigned long long* ord) {
  if (t < it.n_links) {
    const unsigned i = it.a_lo + (unsigned)t;
    *g = i / it.links;
    *ord = i - *g * it.links;
    *key = st.key[i];
    return *key != ~0ull;
  }
  const unsigned p = (unsigned)(t - it.n_links);
  *g = it.pf[p] / it.links;
  *ord = (unsigned long long)it.links + it.pk[p];
  const double d = it.r[p].min_distance;
  *key = dist_key(d);
  return dist_eligible(d, it.r[p].status, it.maxd);
}
// three passes as k_dist_min / k_dist_argmin / k_dist_take: the smallest key per configuration, the lowest ordinal at
// that key, then the gather of the winner
__global__ void __launch_bounds__(256) k_cfg_min(BpDistState st, CfgItems it, BpConfigDist cs, unsigned* n_unsupported) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool unsup = false;
  if (t < (size_t)it.n_links + it.n_self) {
    unsigned g;
    unsigned long long key, ord;
    if (cfg_item(st, it, t, &g, &key, &ord)) atomicMin(cs.key + g, key);
    unsup = t >= it.n_links && ((it.r[t - it.n_links].status >> 16) & 0xffu) == HFB_PATH_UNSUPPORTED;
  }
  const unsigned m = __ballot_sync(0xffffffffu, unsup);
  if (m && (threadIdx.x & 31u) == 0) atomicAdd(n_unsupported, (unsigned)__popc(m));
}
__global__ void __launch_bounds__(256) k_cfg_argmin(BpDistState st, CfgItems it, BpConfigDist cs) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (size_t)it.n_links + it.n_self) return;
  unsigned g;
  unsigned long long key, ord;
  if (cfg_item(st, it, t, &g, &key, &ord) && key == cs.key[g]) atomicMin(cs.ord + g, ord);
}
__global__ void __launch_bounds__(256) k_cfg_take(BpDistState st, CfgItems it, BpConfigDist cs) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (size_t)it.n_links + it.n_self) return;
  unsigned g;
  unsigned long long key, ord;
  if (!cfg_item(st, it, t, &g, &key, &ord) || key != cs.key[g] || ord != cs.ord[g]) return;
  // (ordinals are unique within a configuration: one item per configuration gets here)
  if (t < it.n_links) {
    const unsigned i = it.a_lo + (unsigned)t;
    cs.kind[g] = 0;
    cs.first[g] = i;
    cs.second[g] = (uint32_t)st.nearest[i];
    cs.rec[g] = st.rec[i];
  } else {
    const unsigned p = (unsigned)(t - it.n_links);
    cs.kind[g] = 1;
    cs.first[g] = it.pf[p];
    cs.second[g] = it.ps[p];
    cs.rec[g] = it.r[p];
  }
}

// ---- hfb_env_collide_motions (BpMotions in hfb_broadphase.h) -------------------------------------------------------
// no witness: first_invalid -1, kind -1, first = second = UINT32_MAX, CollisionResult::clear()'s record
// (collision_data.h:483-489)
__global__ void __launch_bounds__(256) k_mot_init(unsigned n, BpMotions ms) {
  const unsigned m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n) return;
  if (ms.sample) {
    ms.sample[m] = 0xffffffffu;
    ms.ord[m] = ~0ull;
  }
  if (ms.first_invalid) ms.first_invalid[m] = -1;
  if (ms.kind) ms.kind[m] = -1;
  if (ms.first) ms.first[m] = 0xffffffffu;
  if (ms.second) ms.second[m] = 0xffffffffu;
  if (ms.rec) {
    hfb_contact r;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    r.distance = nan;
    for (int k = 0; k < 3; ++k) r.p1[k] = r.p2[k] = r.normal[k] = r.pos[k] = nan;
    r.distance_lower_bound = DBL_MAX;
    r.b1 = r.b2 = -1;
    r.status = r.num_contacts = r.iterations = r._pad = 0;
    ms.rec[m] = r;
  }
}
// the colliding candidates of one reduction; the motion of configuration g is the last motion of the range that starts
// at or before it (an empty motion starts where the next one does)
struct MotItems {
  const hfb_contact* r;
  const uint32_t *pf, *ps, *pk;
  unsigned n, split, links, n_b, second_base;
};
__device__ __forceinline__ bool mot_item(const BpMotions& ms, const MotItems& it, unsigned p, unsigned* m, unsigned* k) {
  if (p >= it.n || it.r[p].num_contacts == 0) return false;
  const unsigned g = it.pf[p] / it.links;
  unsigned lo = ms.m0, hi = ms.m1;  // off[lo] <= g < off[hi]
  while (hi - lo > 1) {
    const unsigned mid = lo + (hi - lo) / 2;
    if (ms.off[mid] <= g) lo = mid;
    else hi = mid;
  }
  *m = lo;
  *k = g - ms.off[lo];
  return true;
}
__device__ __forceinline__ unsigned long long mot_ord(const MotItems& it, unsigned p) {
  if (p < it.split) {
    const unsigned i = it.pf[p] % it.links;
    return (unsigned long long)i * it.n_b + (it.ps[p] - it.second_base);
  }
  return (unsigned long long)it.links * it.n_b + it.pk[p];
}
// three passes as k_cfg_min / k_cfg_argmin / k_cfg_take: the smallest colliding sample per motion (and the colliding
// candidates of each kind counted), the lowest ordinal at that sample, then the gather of the winner
__global__ void __launch_bounds__(256) k_mot_min(BpMotions ms, MotItems it, unsigned* n_colliding) {
  const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned m, k;
  const bool hit = mot_item(ms, it, p, &m, &k);
  if (hit) atomicMin(ms.sample + m, k);
  const unsigned me = __ballot_sync(0xffffffffu, hit && p < it.split), mself = __ballot_sync(0xffffffffu, hit && p >= it.split);
  if ((threadIdx.x & 31u) == 0) {
    if (me) atomicAdd(n_colliding, (unsigned)__popc(me));
    if (mself) atomicAdd(n_colliding + 1, (unsigned)__popc(mself));
  }
}
__global__ void __launch_bounds__(256) k_mot_argmin(BpMotions ms, MotItems it) {
  const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned m, k;
  if (mot_item(ms, it, p, &m, &k) && k == ms.sample[m]) atomicMin(ms.ord + m, mot_ord(it, p));
}
__global__ void __launch_bounds__(256) k_mot_take(BpMotions ms, MotItems it) {
  const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned m, k;
  if (!mot_item(ms, it, p, &m, &k) || k != ms.sample[m] || mot_ord(it, p) != ms.ord[m]) return;
  // (ordinals are unique within a configuration: one candidate per motion gets here)
  const bool env = p < it.split;
  if (ms.kind) ms.kind[m] = env ? 0 : 1;
  if (ms.first) ms.first[m] = it.pf[p];
  if (ms.second) ms.second[m] = env ? it.ps[p] - it.second_base : it.ps[p];
  if (ms.rec) ms.rec[m] = it.r[p];
}
__global__ void __launch_bounds__(256) k_mot_final(BpMotions ms) {
  const unsigned m = ms.m0 + blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= ms.m1) return;
  const unsigned k = ms.sample[m];
  ms.first_invalid[m] = k == 0xffffffffu ? -1 : (int32_t)k;
}

// ---- hfb_env_certify_motions (BpCertify in hfb_broadphase.h) -------------------------------------------------------
// one thread per A object of the range: its sides, and its box widened by its reach (the only place that knows where
// the motions end; every later pass reads the sides)
__global__ void __launch_bounds__(256) k_sweep_sides(const double* bb, const double* sweep, unsigned a_lo, unsigned a_hi,
                                                     BpCertify c, double* wbb) {
  const unsigned i = a_lo + blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a_hi) return;
  const unsigned m = motion_of(c.off, c.m0, c.m1, i / c.links);
  double r, l;
  sweep_sides(sweep, i, c.links, c.off[m], c.off[m + 1], &r, &l);
  c.sides[2 * (size_t)i] = r;
  c.sides[2 * (size_t)i + 1] = l;
  const double* b = bb + 6 * (size_t)i;
  double o[6];
  if (aabb_empty(b)) {
    for (int k = 0; k < 6; ++k) o[k] = b[k];
  } else {
    dist_inflate(b, sweep_reach(r, l), o);
  }
  for (int k = 0; k < 6; ++k) wbb[6 * (size_t)i + k] = o[k];
}
// the self candidates (sweep_pair): one thread per (configuration, template pair), as k_config_pairs
__global__ void __launch_bounds__(128) k_sweep_pairs(const double* bb, BpCertify c, const uint32_t* tpl, unsigned n_tpl,
                                                     size_t total, uint32_t* first, uint32_t* second, unsigned capacity,
                                                     unsigned* n_pairs) {
  const size_t tend = (total + 31u) & ~(size_t)31;  // (warp-uniform trip count for the ballots)
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < tend; t += (size_t)gridDim.x * blockDim.x) {
    bool hit = false;
    uint32_t a = 0, b = 0;
    if (t < total) hit = sweep_pair(bb, c.sides, c.links, tpl, n_tpl, c.g0, t, &a, &b);
    append_pair(hit, a, b, first, second, capacity, n_pairs);
  }
}
// per configuration of the range: a side passes until a pair fails it, and exists when every link has it; per motion:
// no colliding sample, no uncertified segment
__global__ void __launch_bounds__(256) k_cert_init(BpCertify c, unsigned n_motions) {
  const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < c.ng) {
    const double* s = c.sides + 2 * (size_t)(c.g0 + t) * c.links;
    bool r = true, l = true;
    for (unsigned i = 0; i < c.links; ++i) {
      r = r && s[2 * i] == s[2 * i];  // (NaN: no side)
      l = l && s[2 * i + 1] == s[2 * i + 1];
    }
    c.pass[2 * (size_t)t] = r;
    c.pass[2 * (size_t)t + 1] = l;
  }
  if (t < n_motions) c.sample[t] = c.unc[t] = 0xffffffffu;
}
// the candidates of one collide() pass; the environment pairs' boxes are A's and B's unwidened ones
struct CertItems {
  const hfb_contact* r;
  const uint32_t *pf, *ps;
  const double *ba, *bb_b;
  unsigned n, split, second_base;
};
// one thread per record: the pair's two thresholds from the sides clear its sample's flags unless the record clears
// them (no contact, supported, 2 * lower bound above the threshold; NaN never does); a contact of a pair whose
// unwidened boxes overlap makes its sample collide
__global__ void __launch_bounds__(256) k_cert_pairs(BpCertify c, CertItems it, unsigned* n_unsupported) {
  const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
  bool unsup = false;
  if (p < it.n) {
    const hfb_contact& rec = it.r[p];
    const bool env = p < it.split;
    const uint32_t a = it.pf[p], b = env ? it.ps[p] - it.second_base : it.ps[p];
    double sr = c.sides[2 * (size_t)a], sl = c.sides[2 * (size_t)a + 1];
    if (!env) {
      sr = add_ru(sr, c.sides[2 * (size_t)b]);
      sl = add_ru(sl, c.sides[2 * (size_t)b + 1]);
    }
    unsup = ((rec.status >> 16) & 0xffu) == HFB_PATH_UNSUPPORTED;
    const bool clear = rec.num_contacts == 0 && !unsup;
    const double d2 = 2.0 * rec.distance_lower_bound;
    const unsigned g = a / c.links;
    uint8_t* f = c.pass + 2 * (size_t)(g - c.g0);
    if (!(clear && d2 > sr)) f[0] = 0;
    if (!(clear && d2 > sl)) f[1] = 0;
    if (rec.num_contacts > 0 && aabb_overlap(it.ba + 6 * (size_t)a, (env ? it.bb_b : it.ba) + 6 * (size_t)b)) {
      const unsigned m = motion_of(c.off, c.m0, c.m1, g);
      atomicMin(c.sample + m, g - c.off[m]);
    }
  }
  const unsigned mu = __ballot_sync(0xffffffffu, unsup);
  if ((threadIdx.x & 31u) == 0 && mu) atomicAdd(n_unsupported, (unsigned)__popc(mu));
}
// per configuration of the range: certified when it has a successor in its motion (its right side exists), its right
// side passes and its successor's left side passes; a motion's first segment that is not, and their count
__global__ void __launch_bounds__(256) k_cert_final(BpCertify c, unsigned* n_uncertified) {
  const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
  bool unc = false;
  if (t < c.ng) {
    const unsigned g = c.g0 + t, m = motion_of(c.off, c.m0, c.m1, g);
    const bool seg = g + 1 < c.off[m + 1];
    const bool cert = seg && c.pass[2 * (size_t)t] && c.pass[2 * (size_t)t + 3];
    if (c.certified) c.certified[t] = cert;
    unc = seg && !cert;
    if (unc) atomicMin(c.unc + m, g - c.off[m]);
  }
  const unsigned mu = __ballot_sync(0xffffffffu, unc);
  if ((threadIdx.x & 31u) == 0 && mu) atomicAdd(n_uncertified, (unsigned)__popc(mu));
}
__global__ void __launch_bounds__(256) k_cert_motions(BpCertify c) {
  const unsigned m = c.m0 + blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= c.m1) return;
  const unsigned k = c.sample[m], u = c.unc[m];
  if (c.first_invalid) c.first_invalid[m] = k == 0xffffffffu ? -1 : (int32_t)k;
  if (c.first_uncertified) c.first_uncertified[m] = u == 0xffffffffu ? -1 : (int32_t)u;
}

size_t up256(size_t b) { return (b + 255) & ~(size_t)255; }
struct Scratch {
  Bounds* part;
  BroadGrid* grid;
  unsigned* n_unbounded;
  unsigned* cell;
  unsigned* order;
  unsigned* count;   // kMaxCells + 1 (count, then exclusive scan in place via `start`)
  unsigned* start;   // kMaxCells + 1
  unsigned* cursor;  // kMaxCells
  void* cub_tmp;
  size_t cub_bytes;
};
constexpr unsigned kParts = 592;
size_t cub_scan_bytes() {
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, b, (unsigned*)nullptr, (unsigned*)nullptr, (int)(kMaxCells + 1));
  return b;
}
Scratch carve(void* p, size_t n) {
  unsigned char* c = static_cast<unsigned char*>(p);
  Scratch s;
  s.part = reinterpret_cast<Bounds*>(c); c += up256(kParts * sizeof(Bounds));
  s.grid = reinterpret_cast<BroadGrid*>(c); c += up256(sizeof(BroadGrid));
  s.n_unbounded = reinterpret_cast<unsigned*>(c); c += 256;
  s.cell = reinterpret_cast<unsigned*>(c); c += up256(n * 4);
  s.order = reinterpret_cast<unsigned*>(c); c += up256(n * 4);
  s.count = reinterpret_cast<unsigned*>(c); c += up256((size_t)(kMaxCells + 1) * 4);
  s.start = reinterpret_cast<unsigned*>(c); c += up256((size_t)(kMaxCells + 1) * 4);
  s.cursor = reinterpret_cast<unsigned*>(c); c += up256((size_t)kMaxCells * 4);
  s.cub_tmp = c;
  s.cub_bytes = cub_scan_bytes();
  return s;
}

}  // namespace

int bp_scene_aabbs_launch(const double* d_local_aabbs, uint32_t nshapes, size_t n, const uint32_t* d_handles,
                          const hfb_transform* d_tfs, double* d_aabbs, cudaStream_t s) {
  if (n == 0) return 0;
  k_scene_aabbs<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(d_local_aabbs, nshapes, (unsigned)n, d_handles, d_tfs, d_aabbs);
  return (int)cudaGetLastError();
}

size_t bp_scratch_bytes(size_t n) {
  return up256(kParts * sizeof(Bounds)) + up256(sizeof(BroadGrid)) + 256 + 2 * up256(n * 4) +
         2 * up256((size_t)(kMaxCells + 1) * 4) + up256((size_t)kMaxCells * 4) + up256(cub_scan_bytes()) + 256;
}

int bp_pairs_launch(size_t n, const double* d_aabbs, size_t i_lo, size_t i_hi, uint32_t* d_first, uint32_t* d_second,
                    size_t capacity, unsigned* d_n_pairs, void* scratch, int num_sms, cudaStream_t s, int* launches) {
  if (num_sms < 1) num_sms = 1;
  Scratch w = carve(scratch, n);
  const unsigned nn = (unsigned)n;
  unsigned pb = (nn + 255) / 256;
  if (pb > kParts) pb = kParts;
  if (pb == 0) pb = 1;
  cudaError_t e;
  k_bounds_partial<<<pb, 256, 0, s>>>(d_aabbs, nn, w.part);
  k_make_grid<<<1, 256, 0, s>>>(w.part, pb, w.grid, d_n_pairs, w.n_unbounded);
  *launches += 2;
  if (n < 2) return (int)cudaGetLastError();
  // the number of cells is only known on the device: counters are cleared and scanned for the maximum
  if ((e = cudaMemsetAsync(w.count, 0, (size_t)(kMaxCells + 1) * 4, s)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(w.cursor, 0, (size_t)kMaxCells * 4, s)) != cudaSuccess) return (int)e;
  k_cell_hist<<<(nn + 255) / 256, 256, 0, s>>>(d_aabbs, nn, w.grid, w.cell, w.count, w.order, w.n_unbounded, nullptr);
  size_t tb = w.cub_bytes;
  if ((e = cub::DeviceScan::ExclusiveSum(w.cub_tmp, tb, w.count, w.start, (int)(kMaxCells + 1), s)) != cudaSuccess) return (int)e;
  k_cell_scatter<<<(nn + 255) / 256, 256, 0, s>>>(w.cell, nn, w.start, w.cursor, w.order);
  if (i_hi > n) i_hi = n;
  if (i_lo < i_hi)
    k_sweep<<<(unsigned)((i_hi - i_lo + 127) / 128), 128, 0, s>>>(d_aabbs, (unsigned)i_hi, (unsigned)i_lo, w.grid, w.cell, w.start,
                                                                 w.order, d_first, d_second,
                                                                 (unsigned)(capacity > 0xffffffffull ? 0xffffffffull : capacity),
                                                                 d_n_pairs);
  if (i_lo < i_hi) {
    unsigned ub = (nn + 127) / 128;
    if (ub > (unsigned)num_sms * 8u) ub = (unsigned)num_sms * 8u;
    k_sweep_unbounded<<<ub ? ub : 1u, 128, 0, s>>>(d_aabbs, nn, (unsigned)i_lo, (unsigned)i_hi, w.cell, w.order, w.n_unbounded, d_first,
                                                   d_second, (unsigned)(capacity > 0xffffffffull ? 0xffffffffull : capacity), d_n_pairs);
  }
  *launches += 5;
  return (int)cudaGetLastError();
}

// the self form's scratch for B, then the extent histogram and the list of A objects tested against all of B
size_t bp_cross_scratch_bytes(size_t n_a, size_t n_b) {
  return bp_scratch_bytes(n_b) + up256((size_t)kExtBins * 4) + up256(n_a * 4);
}

namespace {
// the grid over B in two steps: its bounds, cell and dims (clearing *d_n_pairs and both counters), then B's objects
// binned into `order` / `start` (the oversize and unbounded ones listed from the end of `order`)
int cross_grid_fit(size_t n_b, const double* d_aabbs_b, const BpCrossGrid& g, unsigned* d_n_pairs, void* scratch,
                   cudaStream_t s, int* launches) {
  Scratch w = carve(scratch, n_b);
  unsigned* hist = reinterpret_cast<unsigned*>(static_cast<unsigned char*>(scratch) + bp_scratch_bytes(n_b));
  const unsigned nb = (unsigned)n_b;
  unsigned pb = (nb + 255) / 256;
  if (pb > kParts) pb = kParts;
  if (pb == 0) pb = 1;
  cudaError_t e;
  if ((e = cudaMemsetAsync(hist, 0, (size_t)kExtBins * 4, s)) != cudaSuccess) return (int)e;
  k_cross_bounds_partial<<<pb, 256, 0, s>>>(d_aabbs_b, nb, w.part, hist);
  k_cross_grid<<<1, 256, 0, s>>>(w.part, pb, hist, static_cast<CrossGrid*>(g.grid), d_n_pairs, g.counters);
  *launches += 2;
  return (int)cudaGetLastError();
}
int cross_grid_bin(size_t n_b, const double* d_aabbs_b, const BpCrossGrid& g, void* scratch, cudaStream_t s, int* launches) {
  Scratch w = carve(scratch, n_b);
  CrossGrid* cg = static_cast<CrossGrid*>(g.grid);
  const unsigned nb = (unsigned)n_b;
  cudaError_t e;
  if ((e = cudaMemsetAsync(w.count, 0, (size_t)(kMaxCells + 1) * 4, s)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(w.cursor, 0, (size_t)kMaxCells * 4, s)) != cudaSuccess) return (int)e;
  k_cell_hist<<<(nb + 255) / 256, 256, 0, s>>>(d_aabbs_b, nb, &cg->g, w.cell, w.count, g.order, g.counters, &cg->cell);
  size_t tb = w.cub_bytes;
  if ((e = cub::DeviceScan::ExclusiveSum(w.cub_tmp, tb, w.count, g.start, (int)(kMaxCells + 1), s)) != cudaSuccess) return (int)e;
  k_cell_scatter<<<(nb + 255) / 256, 256, 0, s>>>(w.cell, nb, g.start, w.cursor, g.order);
  *launches += 3;
  return (int)cudaGetLastError();
}
}  // namespace

size_t bp_cross_grid_bytes(size_t n_b) { return 512 + up256(n_b * 4) + up256((size_t)(kMaxCells + 1) * 4); }

BpCrossGrid bp_cross_grid_carve(void* p, size_t n_b) {
  unsigned char* c = static_cast<unsigned char*>(p);
  BpCrossGrid g;
  g.grid = c;
  g.counters = reinterpret_cast<unsigned*>(c + 256);
  g.order = reinterpret_cast<unsigned*>(c + 512);
  g.start = reinterpret_cast<unsigned*>(c + 512 + up256(n_b * 4));
  return g;
}

int bp_cross_build_launch(size_t n_b, const double* d_aabbs_b, const BpCrossGrid& g, void* scratch, cudaStream_t s,
                          int* launches) {
  // (k_cross_grid clears a pair counter: the one of the next query is cleared by bp_cross_query_reset)
  if (int e = cross_grid_fit(n_b, d_aabbs_b, g, g.counters + 2, scratch, s, launches)) return e;
  return n_b ? cross_grid_bin(n_b, d_aabbs_b, g, scratch, s, launches) : 0;
}

namespace {
// the grid rows of every A object in [a_lo, a_hi) (k_cross_sweep) and the A objects that need all of B (k_cross_brute);
// counters[0]: the length of B's oversize list k_cross_sweep walks, counters[1]: the length of A's brute list
int cross_sweep(size_t a_lo, size_t a_hi, const double* d_aabbs_a, size_t n_b, const double* d_aabbs_b, const BpCrossGrid& g,
                unsigned* counters, uint32_t* d_first, uint32_t* d_second, uint32_t second_base, unsigned cap,
                unsigned* d_n_pairs, void* scratch, int num_sms, cudaStream_t s, int* launches) {
  unsigned* brute = reinterpret_cast<unsigned*>(static_cast<unsigned char*>(scratch) + bp_scratch_bytes(n_b) +
                                                up256((size_t)kExtBins * 4));
  const unsigned nb = (unsigned)n_b;
  k_cross_sweep<<<(unsigned)((a_hi - a_lo + 127) / 128), 128, 0, s>>>(d_aabbs_a, (unsigned)a_lo, (unsigned)a_hi, d_aabbs_b, nb,
                                                                      static_cast<const CrossGrid*>(g.grid), g.start, g.order,
                                                                      counters, brute, d_first, d_second, second_base, cap,
                                                                      d_n_pairs);
  unsigned ub = (nb + 127) / 128;
  if (ub > (unsigned)num_sms * 8u) ub = (unsigned)num_sms * 8u;
  k_cross_brute<<<ub, 128, 0, s>>>(d_aabbs_a, d_aabbs_b, nb, counters, brute, d_first, d_second, second_base, cap, d_n_pairs);
  *launches += 2;
  return (int)cudaGetLastError();
}
}  // namespace

// A query against a built grid reads its counters from g.counters + 2: [2] stays 0 (k_cross_grid cleared it at the
// build), so k_cross_sweep leaves B's oversize list to k_cross_oversize, which reads its length from [0]; [3] is A's
// brute list
int bp_cross_query_reset(const BpCrossGrid& g, unsigned* d_n_pairs, cudaStream_t s) {
  cudaError_t e;
  if ((e = cudaMemsetAsync(d_n_pairs, 0, sizeof(unsigned), s)) != cudaSuccess) return (int)e;
  return (int)cudaMemsetAsync(g.counters + 3, 0, sizeof(unsigned), s);  // A's brute list; B's oversize count stays
}

int bp_cross_query_launch(size_t n_a, const double* d_aabbs_a, size_t a_lo, size_t a_hi, size_t n_b, const double* d_aabbs_b,
                          const BpCrossGrid& g, uint32_t* d_first, uint32_t* d_second, uint32_t second_base, size_t capacity,
                          unsigned* d_n_pairs, void* scratch, int num_sms, cudaStream_t s, int* launches) {
  if (num_sms < 1) num_sms = 1;
  if (a_hi > n_a) a_hi = n_a;
  if (n_b == 0 || a_lo >= a_hi) return 0;
  const unsigned cap = (unsigned)(capacity > 0xffffffffull ? 0xffffffffull : capacity);
  if (int e = cross_sweep(a_lo, a_hi, d_aabbs_a, n_b, d_aabbs_b, g, g.counters + 2, d_first, d_second, second_base, cap,
                          d_n_pairs, scratch, num_sms, s, launches))
    return e;
  // (grid-stride: the length of the list is only known on the device)
  size_t ob = ((a_hi - a_lo) * n_b + 127) / 128;
  if (ob > (size_t)num_sms * 16u) ob = (size_t)num_sms * 16u;
  k_cross_oversize<<<(unsigned)ob, 128, 0, s>>>(d_aabbs_a, (unsigned)a_lo, (unsigned)a_hi, d_aabbs_b, (unsigned)n_b,
                                                static_cast<const CrossGrid*>(g.grid), g.order, g.counters, d_first, d_second,
                                                second_base, cap, d_n_pairs);
  *launches += 1;
  return (int)cudaGetLastError();
}

int bp_cross_pairs_launch(size_t n_a, const double* d_aabbs_a, size_t a_lo, size_t a_hi, size_t n_b, const double* d_aabbs_b,
                          uint32_t* d_first, uint32_t* d_second, uint32_t second_base, size_t capacity, unsigned* d_n_pairs,
                          void* scratch, int num_sms, cudaStream_t s, int* launches) {
  if (num_sms < 1) num_sms = 1;
  // the grid in the self form's slots of the scratch: grid (256 bytes), counters ([0]: B oversize + unbounded, [1]: A
  // brute), order, start
  Scratch w = carve(scratch, n_b);
  BpCrossGrid g;
  g.grid = w.grid;
  g.counters = w.n_unbounded;
  g.order = w.order;
  g.start = w.start;
  if (int e = cross_grid_fit(n_b, d_aabbs_b, g, d_n_pairs, scratch, s, launches)) return e;
  if (a_hi > n_a) a_hi = n_a;
  if (n_b == 0 || a_lo >= a_hi) return 0;
  if (int e = cross_grid_bin(n_b, d_aabbs_b, g, scratch, s, launches)) return e;
  return cross_sweep(a_lo, a_hi, d_aabbs_a, n_b, d_aabbs_b, g, g.counters, d_first, d_second, second_base,
                     (unsigned)(capacity > 0xffffffffull ? 0xffffffffull : capacity), d_n_pairs, scratch, num_sms, s, launches);
}

int bp_config_pairs_launch(const double* d_aabbs, size_t links, const uint32_t* d_tpl, size_t n_tpl, size_t g0,
                           size_t num_configs, uint32_t* d_first, uint32_t* d_second, size_t capacity, unsigned* d_n_pairs,
                           int num_sms, cudaStream_t s, int* launches, uint32_t* d_entry) {
  const size_t total = num_configs * n_tpl;
  if (total == 0) return 0;
  if (num_sms < 1) num_sms = 1;
  size_t nb = (total + 127) / 128;
  if (nb > (size_t)num_sms * 16u) nb = (size_t)num_sms * 16u;
  if (d_entry) {
    k_config_entry_pairs<<<(unsigned)nb, 128, 0, s>>>(d_aabbs, (unsigned)links, d_tpl, (unsigned)n_tpl, (unsigned)g0, total,
                                                      d_first, d_second, d_entry,
                                                      (unsigned)(capacity > 0xffffffffull ? 0xffffffffull : capacity),
                                                      d_n_pairs);
    *launches += 1;
    return (int)cudaGetLastError();
  }
  k_config_pairs<<<(unsigned)nb, 128, 0, s>>>(d_aabbs, (unsigned)links, d_tpl, (unsigned)n_tpl, (unsigned)g0, total, d_first,
                                              d_second, (unsigned)(capacity > 0xffffffffull ? 0xffffffffull : capacity),
                                              d_n_pairs);
  *launches += 1;
  return (int)cudaGetLastError();
}

size_t bp_dist_state_bytes(size_t n_a) { return 2 * up256(n_a * 8) + 2 * up256(n_a * 4) + up256(n_a) + n_a * 96; }

BpDistState bp_dist_state_carve(void* p, size_t n_a, const unsigned long long* reach) {
  unsigned char* c = static_cast<unsigned char*>(p);
  BpDistState st;
  st.reach = reach;
  st.key = reinterpret_cast<unsigned long long*>(c); c += up256(n_a * 8);
  st.prev = reinterpret_cast<unsigned long long*>(c); c += up256(n_a * 8);
  st.nearest = reinterpret_cast<int32_t*>(c); c += up256(n_a * 4);
  st.jround = reinterpret_cast<uint32_t*>(c); c += up256(n_a * 4);
  st.state = c; c += up256(n_a);
  st.rec = reinterpret_cast<hfb_distance_result*>(c);
  return st;
}

int bp_dist_reach_launch(size_t n_b, const double* d_bb, unsigned long long* d_reach, int num_sms, cudaStream_t s,
                         int* launches) {
  cudaError_t e;
  if ((e = cudaMemsetAsync(d_reach, 0xff, 24, s)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(d_reach + 3, 0, 24, s)) != cudaSuccess) return (int)e;
  if (n_b == 0) return 0;
  if (num_sms < 1) num_sms = 1;
  size_t nb = (n_b + 255) / 256;
  if (nb > (size_t)num_sms * 4u) nb = (size_t)num_sms * 4u;
  k_dist_reach<<<(unsigned)nb, 256, 0, s>>>(d_bb, (unsigned)n_b, d_reach);
  *launches += 1;
  return (int)cudaGetLastError();
}

int bp_dist_init_launch(size_t n_a, const double* d_ba, size_t a_lo, size_t a_hi, const BpDistState& st, cudaStream_t s,
                        int* launches) {
  if (n_a == 0) return 0;
  k_dist_init<<<(unsigned)((n_a + 255) / 256), 256, 0, s>>>(d_ba, (unsigned)n_a, (unsigned)a_lo, (unsigned)a_hi, st);
  *launches += 1;
  return (int)cudaGetLastError();
}

int bp_dist_boxes_launch(const double* d_ba, size_t a_lo, size_t a_hi, const BpCrossGrid& g, double max_distance, int round,
                         const BpDistState& st, double* d_bq, unsigned* d_n_open, cudaStream_t s, int* launches) {
  cudaError_t e;
  if ((e = cudaMemsetAsync(d_n_open, 0, sizeof(unsigned), s)) != cudaSuccess) return (int)e;
  if (a_lo >= a_hi) return 0;
  k_dist_boxes<<<(unsigned)((a_hi - a_lo + 255) / 256), 256, 0, s>>>(d_ba, (unsigned)a_lo, (unsigned)a_hi,
                                                                     static_cast<const CrossGrid*>(g.grid), max_distance, round,
                                                                     st, d_bq, d_n_open);
  *launches += 1;
  return (int)cudaGetLastError();
}

int bp_dist_filter_launch(const uint32_t* d_first, const uint32_t* d_second, const unsigned* d_n_raw, size_t capacity,
                          const double* d_ba, const double* d_bb, uint32_t second_base, const BpCrossGrid& g,
                          double max_distance, int round, uint32_t* d_kept_first, uint32_t* d_kept_second,
                          unsigned* d_n_kept, int num_sms, cudaStream_t s, int* launches) {
  cudaError_t e;
  if ((e = cudaMemsetAsync(d_n_kept, 0, sizeof(unsigned), s)) != cudaSuccess) return (int)e;
  if (num_sms < 1) num_sms = 1;
  const unsigned cap = (unsigned)(capacity > 0xffffffffull ? 0xffffffffull : capacity);
  size_t nb = (capacity + 255) / 256;  // (grid-stride: the count is only known on the device)
  if (nb > (size_t)num_sms * 8u) nb = (size_t)num_sms * 8u;
  k_dist_filter<<<(unsigned)(nb ? nb : 1), 256, 0, s>>>(d_first, d_second, d_n_raw, cap, d_ba, d_bb, second_base,
                                                        static_cast<const CrossGrid*>(g.grid), max_distance, round,
                                                        d_kept_first, d_kept_second, d_n_kept);
  *launches += 1;
  return (int)cudaGetLastError();
}

int bp_dist_reduce_launch(const hfb_distance_result* d_recs, const uint32_t* d_first, const uint32_t* d_second, size_t n,
                          uint32_t second_base, double max_distance, const BpDistState& st, unsigned* d_n_unsupported,
                          cudaStream_t s, int* launches) {
  if (n == 0) return 0;
  const unsigned nb = (unsigned)((n + 255) / 256);
  k_dist_min<<<nb, 256, 0, s>>>(d_recs, d_first, (unsigned)n, max_distance, st.key, d_n_unsupported);
  k_dist_argmin<<<nb, 256, 0, s>>>(d_recs, d_first, d_second, (unsigned)n, second_base, max_distance, st);
  k_dist_take<<<nb, 256, 0, s>>>(d_recs, d_first, d_second, (unsigned)n, second_base, max_distance, st);
  *launches += 3;
  return (int)cudaGetLastError();
}

size_t bp_config_dist_bytes(size_t n_configs) { return 2 * up256(n_configs * 8) + 2 * up256(n_configs * 4) + up256(n_configs) + n_configs * 96; }

BpConfigDist bp_config_dist_carve(void* p, size_t n_configs) {
  unsigned char* c = static_cast<unsigned char*>(p);
  BpConfigDist cs;
  cs.key = reinterpret_cast<unsigned long long*>(c); c += up256(n_configs * 8);
  cs.ord = reinterpret_cast<unsigned long long*>(c); c += up256(n_configs * 8);
  cs.first = reinterpret_cast<uint32_t*>(c); c += up256(n_configs * 4);
  cs.second = reinterpret_cast<uint32_t*>(c); c += up256(n_configs * 4);
  cs.kind = reinterpret_cast<int8_t*>(c); c += up256(n_configs);
  cs.rec = reinterpret_cast<hfb_distance_result*>(c);
  return cs;
}

int bp_config_dist_init_launch(size_t n_configs, const BpConfigDist& cs, cudaStream_t s, int* launches) {
  if (n_configs == 0) return 0;
  k_cfg_init<<<(unsigned)((n_configs + 255) / 256), 256, 0, s>>>((unsigned)n_configs, cs);
  *launches += 1;
  return (int)cudaGetLastError();
}

int bp_config_dist_pairs_launch(const double* d_aabbs, size_t links, const uint32_t* d_tpl, size_t n_tpl, size_t g0,
                                size_t num_configs, double max_distance, uint32_t* d_first, uint32_t* d_second,
                                uint32_t* d_entry, size_t capacity, unsigned* d_n_pairs, int num_sms, cudaStream_t s,
                                int* launches) {
  cudaError_t e;
  if ((e = cudaMemsetAsync(d_n_pairs, 0, sizeof(unsigned), s)) != cudaSuccess) return (int)e;
  const size_t total = num_configs * n_tpl;
  if (total == 0) return 0;
  if (num_sms < 1) num_sms = 1;
  size_t nb = (total + 127) / 128;
  if (nb > (size_t)num_sms * 16u) nb = (size_t)num_sms * 16u;
  k_config_dist_pairs<<<(unsigned)nb, 128, 0, s>>>(d_aabbs, (unsigned)links, d_tpl, (unsigned)n_tpl, (unsigned)g0, total,
                                                   max_distance, d_first, d_second, d_entry,
                                                   (unsigned)(capacity > 0xffffffffull ? 0xffffffffull : capacity),
                                                   d_n_pairs);
  *launches += 1;
  return (int)cudaGetLastError();
}

int bp_config_dist_reduce_launch(const BpDistState& st, size_t a_lo, size_t a_hi, size_t links,
                                 const hfb_distance_result* d_recs, const uint32_t* d_first, const uint32_t* d_second,
                                 const uint32_t* d_entry, size_t n_self, double max_distance, const BpConfigDist& cs,
                                 unsigned* d_n_unsupported, cudaStream_t s, int* launches) {
  const CfgItems it{(unsigned)a_lo, (unsigned)(a_hi - a_lo), (unsigned)links, (unsigned)n_self, d_recs, d_first, d_second,
                    d_entry, max_distance};
  const size_t n = (a_hi - a_lo) + n_self;
  if (n == 0) return 0;
  const unsigned nb = (unsigned)((n + 255) / 256);
  k_cfg_min<<<nb, 256, 0, s>>>(st, it, cs, d_n_unsupported);
  k_cfg_argmin<<<nb, 256, 0, s>>>(st, it, cs);
  k_cfg_take<<<nb, 256, 0, s>>>(st, it, cs);
  *launches += 3;
  return (int)cudaGetLastError();
}

size_t bp_motions_bytes(size_t n, bool staged) {
  return up256(n * 4) + up256(n * 8) + (staged ? 3 * up256(n * 4) + up256(n) + n * sizeof(hfb_contact) : 0);
}

BpMotions bp_motions_carve(void* p, size_t n, bool staged) {
  unsigned char* c = static_cast<unsigned char*>(p);
  BpMotions ms{};
  ms.sample = reinterpret_cast<unsigned*>(c); c += up256(n * 4);
  ms.ord = reinterpret_cast<unsigned long long*>(c); c += up256(n * 8);
  if (!staged) return ms;
  ms.first_invalid = reinterpret_cast<int32_t*>(c); c += up256(n * 4);
  ms.first = reinterpret_cast<uint32_t*>(c); c += up256(n * 4);
  ms.second = reinterpret_cast<uint32_t*>(c); c += up256(n * 4);
  ms.kind = reinterpret_cast<int8_t*>(c); c += up256(n);
  ms.rec = reinterpret_cast<hfb_contact*>(c);
  return ms;
}

int bp_motions_init_launch(size_t n, const BpMotions& ms, cudaStream_t s, int* launches) {
  if (n == 0) return 0;
  k_mot_init<<<(unsigned)((n + 255) / 256), 256, 0, s>>>((unsigned)n, ms);
  *launches += 1;
  return (int)cudaGetLastError();
}

int bp_motions_reduce_launch(const hfb_contact* d_recs, const uint32_t* d_first, const uint32_t* d_second,
                             const uint32_t* d_entry, size_t n, size_t split, size_t links, size_t n_b,
                             uint32_t second_base, bool witness, const BpMotions& ms, unsigned* d_n_colliding,
                             cudaStream_t s, int* launches) {
  if (n == 0) return 0;
  const MotItems it{d_recs, d_first, d_second, d_entry, (unsigned)n, (unsigned)split, (unsigned)links, (unsigned)n_b,
                    second_base};
  const unsigned nb = (unsigned)((n + 255) / 256);
  k_mot_min<<<nb, 256, 0, s>>>(ms, it, d_n_colliding);
  *launches += 1;
  if (witness) {
    k_mot_argmin<<<nb, 256, 0, s>>>(ms, it);
    k_mot_take<<<nb, 256, 0, s>>>(ms, it);
    *launches += 2;
  }
  return (int)cudaGetLastError();
}

int bp_motions_final_launch(const BpMotions& ms, cudaStream_t s, int* launches) {
  const unsigned n = ms.m1 - ms.m0;
  if (n == 0 || !ms.first_invalid) return 0;
  k_mot_final<<<(n + 255) / 256, 256, 0, s>>>(ms);
  *launches += 1;
  return (int)cudaGetLastError();
}

size_t bp_certify_bytes(size_t n, bool staged) { return (staged ? 4 : 2) * up256(n * 4); }

BpCertify bp_certify_carve(void* p, size_t n, bool staged) {
  unsigned char* c = static_cast<unsigned char*>(p);
  BpCertify cs{};
  cs.sample = reinterpret_cast<unsigned*>(c); c += up256(n * 4);
  cs.unc = reinterpret_cast<unsigned*>(c); c += up256(n * 4);
  if (!staged) return cs;
  cs.first_invalid = reinterpret_cast<int32_t*>(c); c += up256(n * 4);
  cs.first_uncertified = reinterpret_cast<int32_t*>(c);
  return cs;
}

int bp_sweep_sides_launch(const double* d_bb, const double* d_sweep, size_t a_lo, size_t a_hi, const BpCertify& c,
                          double* d_wbb, cudaStream_t s, int* launches) {
  if (a_hi <= a_lo) return 0;
  k_sweep_sides<<<(unsigned)((a_hi - a_lo + 255) / 256), 256, 0, s>>>(d_bb, d_sweep, (unsigned)a_lo, (unsigned)a_hi, c,
                                                                      d_wbb);
  *launches += 1;
  return (int)cudaGetLastError();
}

int bp_sweep_pairs_launch(const double* d_bb, const BpCertify& c, const uint32_t* d_tpl, size_t n_tpl, uint32_t* d_first,
                          uint32_t* d_second, size_t capacity, unsigned* d_n_pairs, int num_sms, cudaStream_t s,
                          int* launches) {
  const size_t total = (size_t)c.ng * n_tpl;
  if (total == 0) return 0;
  if (num_sms < 1) num_sms = 1;
  size_t nb = (total + 127) / 128;
  if (nb > (size_t)num_sms * 16u) nb = (size_t)num_sms * 16u;
  k_sweep_pairs<<<(unsigned)nb, 128, 0, s>>>(d_bb, c, d_tpl, (unsigned)n_tpl, total, d_first, d_second,
                                             (unsigned)(capacity > 0xffffffffull ? 0xffffffffull : capacity), d_n_pairs);
  *launches += 1;
  return (int)cudaGetLastError();
}

int bp_certify_launch(const hfb_contact* d_recs, const uint32_t* d_first, const uint32_t* d_second, size_t n, size_t split,
                      uint32_t second_base, const double* d_ba, const double* d_bb_b, const BpCertify& c,
                      unsigned* d_counts, cudaStream_t s, int* launches) {
  const unsigned n_motions = c.m1;  // (the state of motions [0, m1) is set: the range's binary search reads no other)
  const unsigned n_init = c.ng > n_motions ? c.ng : n_motions;
  if (n_init == 0) return 0;
  k_cert_init<<<(n_init + 255) / 256, 256, 0, s>>>(c, n_motions);
  *launches += 1;
  if (n) {
    const CertItems it{d_recs, d_first, d_second, d_ba, d_bb_b, (unsigned)n, (unsigned)split, second_base};
    k_cert_pairs<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(c, it, d_counts);
    *launches += 1;
  }
  if (c.ng) {
    k_cert_final<<<(c.ng + 255) / 256, 256, 0, s>>>(c, d_counts + 1);
    *launches += 1;
  }
  if (c.m1 > c.m0) {
    k_cert_motions<<<(c.m1 - c.m0 + 255) / 256, 256, 0, s>>>(c);
    *launches += 1;
  }
  return (int)cudaGetLastError();
}

int bp_env_update_launch(const double* d_local_aabbs, uint32_t nshapes, size_t m, const uint32_t* d_idx,
                         const hfb_transform* d_tfs_new, const uint32_t* d_handles, hfb_transform* d_tfs, double* d_aabbs,
                         cudaStream_t s) {
  if (m == 0) return 0;
  k_env_update<<<(unsigned)((m + 255) / 256), 256, 0, s>>>(d_local_aabbs, nshapes, (unsigned)m, d_idx, d_tfs_new, d_handles,
                                                           d_tfs, d_aabbs);
  return (int)cudaGetLastError();
}

}  // namespace hfb
