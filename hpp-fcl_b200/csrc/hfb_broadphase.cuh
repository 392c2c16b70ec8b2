// Broadphase feed of the batched narrow phase (BASELINE config 5, SURVEY 8(f1)): world-space AABBs of a scene's
// objects and the pairs whose AABBs overlap -- what a BroadPhaseCollisionManager hands to its collision callback.
//
// Replaces, for this path only:
//   computeLocalAABB of the shapes / BVHModel            src/shape/geometric_shapes.cpp:145-260, src/BVH/BVH_model.cpp
//       (computeBV<AABB, S> with the identity transform: src/shape/geometric_shapes_utility.cpp:264-420)
//   CollisionObject::computeAABB                          include/hpp/fcl/collision_object.h:258-278
//   AABB::overlap                                         include/hpp/fcl/BV/AABB.h:111-118
//   DynamicAABBTreeCollisionManager::collide(callback)    src/broadphase/broadphase_dynamic_AABB_tree.cpp:336-407,716-721
//       -- the SET of pairs it reports (every pair of objects with overlapping AABBs, once); the order is the
//       manager's own business in the reference as well (its managers disagree among themselves).
// Design: no tree.  A uniform grid whose cell is as large as the largest AABB: objects are bucketed by the cell of
// their centre, so a partner can only sit in the 27 cells around -- a counting sort and one sweep, the same three
// steps on the host (here) and on the device (hfb_broadphase.cu).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

#include "hfb_arena.cuh"

namespace hfb {

struct LocalAabb {  // CollisionGeometry::aabb_local
  double mn[3], mx[3];
};

// aabb_local of a shape record (computeLocalAABB); false for node types without one here
inline bool shape_local_aabb(const HostArena& A, const hfb_shape& s, LocalAabb& b) {
  double h[3];
  switch (s.type) {
    case HFB_GEOM_BOX: h[0] = s.p[0]; h[1] = s.p[1]; h[2] = s.p[2]; break;            // half sides
    case HFB_GEOM_SPHERE: h[0] = h[1] = h[2] = s.p[0]; break;
    case HFB_GEOM_ELLIPSOID: h[0] = s.p[0]; h[1] = s.p[1]; h[2] = s.p[2]; break;
    case HFB_GEOM_CAPSULE: h[0] = h[1] = s.p[0]; h[2] = s.p[1] + s.p[0]; break;      // 0.5 * lz + radius
    case HFB_GEOM_CONE:
    case HFB_GEOM_CYLINDER: h[0] = h[1] = s.p[0]; h[2] = s.p[1]; break;
    case HFB_GEOM_CONVEX:
    case HFB_GEOM_TRIANGLE: {
      if (s.data >= A.cvx.size()) return false;
      const ConvexDesc& d = A.cvx[s.data];
      const uint32_t nv = s.type == HFB_GEOM_TRIANGLE ? 3u : d.nv;
      for (int k = 0; k < 3; ++k) {
        b.mn[k] = DBL_MAX;
        b.mx[k] = -DBL_MAX;
        for (uint32_t i = 0; i < nv; ++i) {
          const double v = A.pool[d.off + (size_t)k * d.vpad + i];
          b.mn[k] = v < b.mn[k] ? v : b.mn[k];
          b.mx[k] = v > b.mx[k] ? v : b.mx[k];
        }
      }
      h[0] = -1;
    } break;
    case HFB_BV_OBB:
    case HFB_BV_OBBRSS: {
      if (s.data >= A.bvh_desc.size()) return false;
      const BvhDesc& d = A.bvh_desc[s.data];
      for (int k = 0; k < 3; ++k) {
        b.mn[k] = DBL_MAX;
        b.mx[k] = -DBL_MAX;
      }
      for (uint32_t i = 0; i < d.num_verts; ++i)
        for (int k = 0; k < 3; ++k) {
          const double v = A.bvh_verts[3 * ((size_t)d.vert_off + i) + k];
          b.mn[k] = v < b.mn[k] ? v : b.mn[k];
          b.mx[k] = v > b.mx[k] ? v : b.mx[k];
        }
      h[0] = -1;
    } break;
    case HFB_GEOM_PLANE:
    case HFB_GEOM_HALFSPACE: {
      // computeBV<AABB, Halfspace / Plane> with the identity pose (geometric_shapes_utility.cpp:391-456): everything,
      // except along an axis the normal is exactly aligned with.  transform() builds a new Halfspace / Plane, whose
      // constructor normalises (n, d) once more (unitNormalTest)
      if (s.data >= A.pool.size()) return false;
      double n[3] = {s.p[0], s.p[1], s.p[2]};
      double d = A.pool[s.data] + ((n[0] * 0.0 + n[1] * 0.0) + n[2] * 0.0);
      const double l = sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]);
      if (l > 0) {
        const double inv_l = 1.0 / l;
        for (int k = 0; k < 3; ++k) n[k] *= inv_l;
        d *= inv_l;
      } else {
        n[0] = 1;
        n[1] = n[2] = 0;
        d = 0;
      }
      for (int k = 0; k < 3; ++k) {
        b.mn[k] = -DBL_MAX;
        b.mx[k] = DBL_MAX;
      }
      int axis = -1;
      if (n[1] == 0.0 && n[2] == 0.0) axis = 0;
      else if (n[0] == 0.0 && n[2] == 0.0) axis = 1;
      else if (n[0] == 0.0 && n[1] == 0.0) axis = 2;
      if (axis >= 0) {
        if (s.type == HFB_GEOM_HALFSPACE) {
          if (n[axis] < 0) b.mn[axis] = -d;
          else if (n[axis] > 0) b.mx[axis] = d;
        } else {
          if (n[axis] < 0) b.mn[axis] = b.mx[axis] = -d;
          else if (n[axis] > 0) b.mn[axis] = b.mx[axis] = d;
        }
      }
      h[0] = -1;
    } break;
    default: return false;
  }
  if (h[0] >= 0)
    for (int k = 0; k < 3; ++k) {
      b.mn[k] = -h[k];
      b.mx[k] = h[k];
    }
  if (s.ssr > 0)  // the swept-sphere radius inflates the local box (geometric_shapes.cpp:147-151)
    for (int k = 0; k < 3; ++k) {
      b.mn[k] -= s.ssr;
      b.mx[k] += s.ssr;
    }
  return true;
}

// CollisionObject::computeAABB: the box around the rotated local box, translated.  `out`: min xyz, max xyz
HFB_HD void object_aabb(const double* lmn, const double* lmx, const hfb_transform& tf, double* out) {
  // Matrix3f::isIdentity(): |R - I| <= 1e-12 element-wise (Eigen's fuzzy test against the identity's norm of 1)
  bool ident = true;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      const double v = tf.R[c * 3 + r] - (r == c ? 1.0 : 0.0);
      if (fabs(v) > 1e-12) ident = false;
    }
  if (ident) {
    for (int k = 0; k < 3; ++k) {
      out[k] = lmn[k] + tf.T[k];
      out[3 + k] = lmx[k] + tf.T[k];
    }
    return;
  }
  for (int k = 0; k < 3; ++k) {
    double a[3], b[3];
    for (int j = 0; j < 3; ++j) {
      const double r = tf.R[j * 3 + k];  // R(k, j), column-major storage
      const double lo = r * lmn[j], hi = r * lmx[j];
      a[j] = lo < hi ? lo : hi;
      b[j] = lo < hi ? hi : lo;
    }
    out[k] = tf.T[k] + ((a[0] + a[1]) + a[2]);
    out[3 + k] = tf.T[k] + ((b[0] + b[1]) + b[2]);
  }
}

HFB_HD bool aabb_overlap(const double* a, const double* b) {  // AABB::overlap: closed intervals
  if (a[0] > b[3] || a[1] > b[4] || a[2] > b[5]) return false;
  if (a[3] < b[0] || a[4] < b[1] || a[5] < b[2]) return false;
  return true;
}

// A box that reaches past this (a Halfspace or Plane: +-DBL_MAX, or +-inf once rotated) is "unbounded": it takes no part
// in the grid -- a cell as large as the largest box would be the whole scene -- and is tested against every object.
#define HFB_BP_UNBOUNDED 1e300
HFB_HD bool aabb_unbounded(const double* b) {
  for (int k = 0; k < 6; ++k)
    if (!(b[k] > -HFB_BP_UNBOUNDED && b[k] < HFB_BP_UNBOUNDED)) return true;
  return false;
}
// the marker hfb_scene_aabbs writes for an object without a box (no such geometry, node type without aabb_local)
HFB_HD bool aabb_empty(const double* b) { return b[0] == DBL_MAX && b[3] == -DBL_MAX; }

// grid geometry shared by the host and device pair finders
struct BroadGrid {
  double origin[3];
  double inv_cell;
  int dim[3];
};
HFB_HD int grid_coord(const BroadGrid& g, double c, int k) {
  // clamped before the conversion: a query box of the cross form may lie far outside the grid
  const double v = floor((c - g.origin[k]) * g.inv_cell);
  return !(v >= 0) ? 0 : (v >= g.dim[k] ? g.dim[k] - 1 : (int)v);
}
HFB_HD unsigned grid_cell(const BroadGrid& g, const double* bb) {
  const int x = grid_coord(g, 0.5 * (bb[0] + bb[3]), 0), y = grid_coord(g, 0.5 * (bb[1] + bb[4]), 1),
            z = grid_coord(g, 0.5 * (bb[2] + bb[5]), 2);
  return (unsigned)((z * g.dim[1] + y) * g.dim[0] + x);
}
// the grid over the centres' box [lo, hi] with cells of at least `cell`, grown until it has at most 2^21 cells;
// returns the cell size used
HFB_HD double grid_fit(const double* lo, const double* hi, double cell, BroadGrid& g) {
  double dim[3];
  for (;;) {
    // counted in double: a cell far below the span must grow, not wrap the int dimensions
    double cells = 1;
    for (int k = 0; k < 3; ++k) {
      dim[k] = floor((hi[k] - lo[k]) / cell) + 1;
      cells *= dim[k];
    }
    if (cells <= 2097152.0) break;
    cell *= 1.26;  // halves the number of cells
  }
  for (int k = 0; k < 3; ++k) g.dim[k] = (int)dim[k];
  for (int k = 0; k < 3; ++k) g.origin[k] = lo[k];
  g.inv_cell = 1.0 / cell;
  return cell;
}

// a grid for these boxes: cell = the largest box extent (so partners sit in adjacent cells), at most ~2^21 cells
inline BroadGrid make_grid(size_t n, const double* bb) {
  BroadGrid g;
  double lo[3] = {DBL_MAX, DBL_MAX, DBL_MAX}, hi[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX}, ext = 0;
  for (size_t i = 0; i < n; ++i) {
    if (aabb_empty(bb + 6 * i) || aabb_unbounded(bb + 6 * i)) continue;
    for (int k = 0; k < 3; ++k) {
      const double c = 0.5 * (bb[6 * i + k] + bb[6 * i + 3 + k]), e = bb[6 * i + 3 + k] - bb[6 * i + k];
      lo[k] = c < lo[k] ? c : lo[k];
      hi[k] = c > hi[k] ? c : hi[k];
      ext = e > ext ? e : ext;
    }
  }
  if (!(lo[0] <= hi[0])) lo[0] = lo[1] = lo[2] = hi[0] = hi[1] = hi[2] = 0;  // nothing bounded
  grid_fit(lo, hi, ext > 0 ? ext : 1.0, g);
  return g;
}

// every pair i < j with overlapping boxes, in no particular order; returns their number (all of them are counted,
// at most `capacity` stored)
inline size_t broadphase_pairs_host(size_t n, const double* bb, uint32_t* first, uint32_t* second, size_t capacity) {
  if (n < 2) return 0;
  const BroadGrid g = make_grid(n, bb);
  const size_t ncell = (size_t)g.dim[0] * g.dim[1] * g.dim[2];
  std::vector<uint32_t> cell(n), start(ncell + 1, 0), order(n), unbounded;
  for (size_t i = 0; i < n; ++i) {
    if (aabb_empty(bb + 6 * i)) {
      cell[i] = 0xffffffffu;
    } else if (aabb_unbounded(bb + 6 * i)) {
      cell[i] = 0xfffffffeu;
      unbounded.push_back((uint32_t)i);
    } else {
      cell[i] = grid_cell(g, bb + 6 * i);
      ++start[cell[i] + 1];
    }
  }
  for (size_t c = 0; c < ncell; ++c) start[c + 1] += start[c];
  {
    std::vector<uint32_t> cur(start.begin(), start.end() - 1);
    for (size_t i = 0; i < n; ++i)
      if (cell[i] < 0xfffffffeu) order[cur[cell[i]]++] = (uint32_t)i;
  }
  size_t count = 0;
  // the unbounded objects against everything (a pair of two of them once)
  for (uint32_t u : unbounded)
    for (size_t j = 0; j < n; ++j) {
      if (j == u || cell[j] == 0xffffffffu || (cell[j] == 0xfffffffeu && j < u)) continue;
      if (!aabb_overlap(bb + 6 * (size_t)u, bb + 6 * j)) continue;
      if (count < capacity) {
        first[count] = u < j ? u : (uint32_t)j;
        second[count] = u < j ? (uint32_t)j : u;
      }
      ++count;
    }
  for (size_t i = 0; i < n; ++i) {
    if (cell[i] >= 0xfffffffeu) continue;
    const unsigned c = cell[i];
    const int cx = (int)(c % (unsigned)g.dim[0]), cy = (int)((c / (unsigned)g.dim[0]) % (unsigned)g.dim[1]),
              cz = (int)(c / ((unsigned)g.dim[0] * (unsigned)g.dim[1]));
    for (int dz = -1; dz <= 1; ++dz)
      for (int dy = -1; dy <= 1; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
          const int x = cx + dx, y = cy + dy, z = cz + dz;
          if (x < 0 || y < 0 || z < 0 || x >= g.dim[0] || y >= g.dim[1] || z >= g.dim[2]) continue;
          const size_t nc = ((size_t)z * g.dim[1] + y) * g.dim[0] + x;
          for (uint32_t q = start[nc]; q < start[nc + 1]; ++q) {
            const uint32_t j = order[q];
            if (j <= i) continue;
            if (!aabb_overlap(bb + 6 * i, bb + 6 * (size_t)j)) continue;
            if (count < capacity) {
              first[count] = (uint32_t)i;
              second[count] = j;
            }
            ++count;
          }
        }
  }
  return count;
}

// ---- cross form: every (i in A, j in B) with overlapping boxes --------------------------------------------------
// BroadPhaseCollisionManager::collide(other, callback) (broadphase_collision_manager.h:94-118; the set of
// NaiveCollisionManager::collide(other), src/broadphase/broadphase_bruteforce.cpp:150-170).  The grid is built over B
// only, so the sizes of A's boxes never shape it.  Its cell is not B's largest extent (one wall among small objects
// would put the whole environment in a handful of cells) but the power of two at or above the extents of 95 % of
// B's bounded boxes (a log2 histogram of the extents).  B boxes wider than the final cell ("oversize") stay out of the
// grid with B's unbounded ones and are tested against every A object.  A B box in the grid has its centre within
// half a cell of any box it overlaps, so an A box looks up the cells its box covers widened by half a cell; the cells
// of one grid row are contiguous in the sorted order, so a lookup walks one index range per row.  A boxes that are
// unbounded or whose lookup spans more than kCrossScanRows rows are tested against every B object instead.  The
// pairs are partitioned by (A grid / A brute) x (B grid / B oversize), so each is reported once.
constexpr int kExtBins = 128;
constexpr int kCrossScanRows = 256;

HFB_HD double box_extent(const double* b) {
  double e = b[3] - b[0];
  e = b[4] - b[1] > e ? b[4] - b[1] : e;
  return b[5] - b[2] > e ? b[5] - b[2] : e;
}
// histogram bin of an extent: bin b >= 1 holds [2^(b-64), 2^(b-63)), bin 0 the empty extents
HFB_HD int extent_bin(double e) {
  if (!(e > 0)) return 0;
  const int b = ilogb(e) + 64;
  return b < 1 ? 1 : (b >= kExtBins ? kExtBins - 1 : b);
}
// the cell the cross form starts from: the top of the bin that holds the 95th percentile of the extents.  Boxes of
// zero extent (points) fit any cell: when they make up the percentile, the first non-empty bin above them sets the
// cell, and with nothing but points the self form's fallback of 1 does
HFB_HD double cross_cell(const unsigned* hist, unsigned total) {
  if (total == 0) return 1.0;
  const unsigned want = total - total / 20u;
  unsigned cum = 0;
  int b = 0;
  for (; b < kExtBins - 1; ++b) {
    cum += hist[b];
    if (cum >= want) break;
  }
  if (b == 0)
    for (b = 1; b < kExtBins && hist[b] == 0; ++b) {
    }
  return b < kExtBins ? ldexp(1.0, b - 63) : 1.0;
}
// B's grid over its centres' box [lo, hi]: the cell from the histogram, no finer than the largest span / 2^21 (a
// finer one has more than 2^21 cells along that axis alone, so grid_fit would only grow it step by step)
HFB_HD double cross_grid_fit(const double* lo, const double* hi, const unsigned* hist, unsigned total, BroadGrid& g) {
  double cell = cross_cell(hist, total), span = 0;
  for (int k = 0; k < 3; ++k) span = hi[k] - lo[k] > span ? hi[k] - lo[k] : span;
  cell = cell > span * 0x1p-21 ? cell : span * 0x1p-21;
  return grid_fit(lo, hi, cell, g);
}
// the grid cells an A box looks up: its box widened by half a cell, plus a margin that covers the rounding of the
// centres (the grid coordinate is monotonic in the position, so a margin is all it takes)
HFB_HD int cross_query_cells(const BroadGrid& g, double cell, const double* a, int* c0, int* c1) {
  for (int k = 0; k < 3; ++k) {
    const double m = 0.5 * cell * (1.0 + 1e-6) + 1e-12 * fmax(fabs(a[k]), fabs(a[3 + k]));
    c0[k] = grid_coord(g, a[k] - m, k);
    c1[k] = grid_coord(g, a[3 + k] + m, k);
  }
  return (c1[1] - c0[1] + 1) * (c1[2] - c0[2] + 1);  // rows
}

// the cross set in no particular order, (index in A, index in B); returns its size (all pairs are counted, at most
// `capacity` stored)
inline size_t broadphase_cross_pairs_host(size_t na, const double* ba, size_t nb, const double* bb, uint32_t* first,
                                          uint32_t* second, size_t capacity) {
  if (na == 0 || nb == 0) return 0;
  double lo[3] = {DBL_MAX, DBL_MAX, DBL_MAX}, hi[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX};
  unsigned hist[kExtBins] = {0}, total = 0;
  for (size_t j = 0; j < nb; ++j) {
    const double* b = bb + 6 * j;
    if (aabb_empty(b) || aabb_unbounded(b)) continue;
    for (int k = 0; k < 3; ++k) {
      const double c = 0.5 * (b[k] + b[3 + k]);
      lo[k] = c < lo[k] ? c : lo[k];
      hi[k] = c > hi[k] ? c : hi[k];
    }
    ++hist[extent_bin(box_extent(b))];
    ++total;
  }
  if (!(lo[0] <= hi[0])) lo[0] = lo[1] = lo[2] = hi[0] = hi[1] = hi[2] = 0;
  BroadGrid g;
  const double cell = cross_grid_fit(lo, hi, hist, total, g);
  const size_t ncell = (size_t)g.dim[0] * g.dim[1] * g.dim[2];
  std::vector<uint32_t> cell_of(nb), start(ncell + 1, 0), order(nb), over, brute;
  for (size_t j = 0; j < nb; ++j) {
    const double* b = bb + 6 * j;
    if (aabb_empty(b)) {
      cell_of[j] = 0xffffffffu;
    } else if (aabb_unbounded(b) || box_extent(b) > cell) {
      cell_of[j] = 0xfffffffeu;
      over.push_back((uint32_t)j);
    } else {
      cell_of[j] = grid_cell(g, b);
      ++start[cell_of[j] + 1];
    }
  }
  for (size_t c = 0; c < ncell; ++c) start[c + 1] += start[c];
  {
    std::vector<uint32_t> cur(start.begin(), start.end() - 1);
    for (size_t j = 0; j < nb; ++j)
      if (cell_of[j] < 0xfffffffeu) order[cur[cell_of[j]]++] = (uint32_t)j;
  }
  size_t count = 0;
  auto emit = [&](size_t i, uint32_t j) {
    if (count < capacity) {
      first[count] = (uint32_t)i;
      second[count] = j;
    }
    ++count;
  };
  for (size_t i = 0; i < na; ++i) {
    const double* a = ba + 6 * i;
    if (aabb_empty(a)) continue;
    int c0[3], c1[3];
    if (aabb_unbounded(a) || cross_query_cells(g, cell, a, c0, c1) > kCrossScanRows) {
      brute.push_back((uint32_t)i);
      continue;
    }
    for (int z = c0[2]; z <= c1[2]; ++z)
      for (int y = c0[1]; y <= c1[1]; ++y) {
        const size_t row = ((size_t)z * g.dim[1] + y) * g.dim[0];
        for (uint32_t q = start[row + c0[0]]; q < start[row + c1[0] + 1]; ++q)
          if (aabb_overlap(a, bb + 6 * (size_t)order[q])) emit(i, order[q]);
      }
    for (uint32_t j : over)
      if (aabb_overlap(a, bb + 6 * (size_t)j)) emit(i, j);
  }
  for (uint32_t i : brute)
    for (size_t j = 0; j < nb; ++j)
      if (cell_of[j] != 0xffffffffu && aabb_overlap(ba + 6 * (size_t)i, bb + 6 * j)) emit(i, (uint32_t)j);
  return count;
}

// ---- self pairs within configurations: a robot checked against itself, one configuration at a time ----------------
// Set A holds configurations of L links each, configuration-major (object g*L + i is link i of configuration g).  A
// template of P link pairs (i, j) -- an SRDF's enabled pairs, the collision pairs of a Pinocchio GeometryModel -- names
// the pairs each configuration checks.  The candidates of configuration g are the template's pairs whose boxes
// overlap: the set DynamicAABBTreeCollisionManager::collide(callback) over g's L objects hands to a callback that keeps
// only the template's pairs (broadphase_collision_manager.h:104-106), with o1 = g*L + i and o2 = g*L + j.  No grid: a
// configuration has a few hundred pairs at most, each a test of two boxes.

// the template's conditions; null when it meets them
inline const char* config_template_error(size_t links, size_t n_pairs, const uint32_t* tpl) {
  std::vector<uint64_t> keys(n_pairs);
  for (size_t k = 0; k < n_pairs; ++k) {
    const uint32_t i = tpl[2 * k], j = tpl[2 * k + 1];
    if (i >= links || j >= links) return "self-pair template: link index out of range";
    if (i == j) return "self-pair template: a link paired with itself";
    keys[k] = i < j ? (uint64_t)i << 32 | j : (uint64_t)j << 32 | i;
  }
  std::sort(keys.begin(), keys.end());
  if (std::adjacent_find(keys.begin(), keys.end()) != keys.end()) return "self-pair template: a pair listed twice";
  return nullptr;
}
// a set A of n_a objects as configurations of `links` objects each, the range [g0, g0 + ng) of them and the template of
// n_tpl self pairs; null when they meet the conditions
inline const char* config_range_error(size_t n_a, size_t links, size_t g0, size_t ng, size_t n_tpl, const uint32_t* tpl) {
  if (links == 0 || n_a % links) return "n_a is not a multiple of links_per_config";
  if (g0 > n_a / links || ng > n_a / links - g0) return "configuration range past the end";
  if (n_tpl > 0xffffffffull) return "self-pair template too large";
  return config_template_error(links, n_tpl, tpl);
}
// the n_motions + 1 offsets of n_motions runs of configurations: from 0 on, not decreasing, at most INT32_MAX samples
// per motion; null when they meet these.  That off[n_motions] is the number of configurations is the caller's check.
inline const char* motion_offsets_error(size_t n_motions, const uint32_t* off) {
  if (n_motions > 0xffffffffull) return "too many motions";
  if (off[0] != 0) return "motion offsets do not start at 0";
  for (size_t m = 0; m < n_motions; ++m) {
    if (off[m + 1] < off[m]) return "motion offsets decrease";
    if (off[m + 1] - off[m] > 0x7fffffffu) return "a motion has more than INT32_MAX samples";
  }
  return nullptr;
}
// self pair t of the configurations from g0 on: configuration g0 + t / P, template entry t % P -> (*a, *b), object
// indices in A; true when both objects have a box and the boxes overlap (AABB::overlap, closed intervals)
HFB_HD bool config_pair(const double* bb, uint32_t links, const uint32_t* tpl, uint32_t n_pairs, uint32_t g0, size_t t,
                        uint32_t* a, uint32_t* b) {
  const size_t g = g0 + t / n_pairs, k = t % n_pairs;
  *a = (uint32_t)(g * links + tpl[2 * k]);
  *b = (uint32_t)(g * links + tpl[2 * k + 1]);
  const double* x = bb + 6 * (size_t)*a;
  const double* y = bb + 6 * (size_t)*b;
  return !aabb_empty(x) && !aabb_empty(y) && aabb_overlap(x, y);
}
// the self pairs of configurations [g0, g0 + num_configs), configuration by configuration in template order; returns
// their number (all of them are counted, at most `capacity` stored)
inline size_t broadphase_config_pairs_host(const double* bb, uint32_t links, const uint32_t* tpl, uint32_t n_pairs,
                                           uint32_t g0, size_t num_configs, uint32_t* first, uint32_t* second,
                                           size_t capacity) {
  size_t count = 0;
  for (size_t t = 0; t < num_configs * n_pairs; ++t) {
    uint32_t a, b;
    if (!config_pair(bb, links, tpl, n_pairs, g0, t, &a, &b)) continue;
    if (count < capacity) {
      first[count] = a;
      second[count] = b;
    }
    ++count;
  }
  return count;
}

// ---- self pairs within configurations for distance: the pairs whose distance() must run --------------------------
// a - r rounded down and a + r rounded up (r >= 0): __dsub_rd / __dadd_ru on the device.  On the host the nearest sum
// and its exact rounding error (TwoSum, no multiplication, so no contraction can change it) give the same value: one
// step outward when the error lies outward.  An overflow to +-inf already lies outward (its error is NaN).
HFB_HD double sub_rd(double a, double r) {
#ifdef __CUDA_ARCH__
  return __dsub_rd(a, r);
#else
  const double s = a - r, z = s - a, e = (a - (s - z)) - (r + z);
  return e < 0 ? nextafter(s, -INFINITY) : s;
#endif
}
HFB_HD double add_ru(double a, double r) {
#ifdef __CUDA_ARCH__
  return __dadd_ru(a, r);
#else
  const double s = a + r, z = s - a, e = (a - (s - z)) + (r - z);
  return e > 0 ? nextafter(s, INFINITY) : s;
#endif
}
// self pair t as in config_pair; true when its distance() runs: unless both boxes exist and are finite and link j's box
// does not overlap link i's box widened by max_distance, rounded outward (the test k_dist_filter applies with
// dist_inflate) -- then the box gap, and so the distance, exceeds max_distance.  At max_distance = inf all run.
HFB_HD bool config_dist_pair(const double* bb, uint32_t links, const uint32_t* tpl, uint32_t n_pairs, uint32_t g0, size_t t,
                             double maxd, uint32_t* a, uint32_t* b) {
  const size_t g = g0 + t / n_pairs, k = t % n_pairs;
  *a = (uint32_t)(g * links + tpl[2 * k]);
  *b = (uint32_t)(g * links + tpl[2 * k + 1]);
  const double* x = bb + 6 * (size_t)*a;
  const double* y = bb + 6 * (size_t)*b;
  if (aabb_empty(x) || aabb_empty(y)) return true;
  for (int c = 0; c < 6; ++c)
    if (!isfinite(x[c]) || !isfinite(y[c])) return true;
  double o[6];
  for (int c = 0; c < 3; ++c) {
    o[c] = sub_rd(x[c], maxd);
    o[3 + c] = add_ru(x[3 + c], maxd);
  }
  return aabb_overlap(o, y);
}
// the pairs config_dist_pair runs for configurations [g0, g0 + num_configs), configuration by configuration in template
// order; returns their number (all of them are counted, at most `capacity` stored)
inline size_t broadphase_config_distance_pairs_host(const double* bb, uint32_t links, const uint32_t* tpl, uint32_t n_pairs,
                                                    uint32_t g0, size_t num_configs, double maxd, uint32_t* first,
                                                    uint32_t* second, size_t capacity) {
  size_t count = 0;
  for (size_t t = 0; t < num_configs * n_pairs; ++t) {
    uint32_t a, b;
    if (!config_dist_pair(bb, links, tpl, n_pairs, g0, t, maxd, &a, &b)) continue;
    if (count < capacity) {
      first[count] = a;
      second[count] = b;
    }
    ++count;
  }
  return count;
}

// ---- hfb_env_certify_motions: the sides of a sample and the candidates they widen -------------------------------
// A side of sample g is the segment to g + 1 (right) or from g - 1 (left) of its motion; an object's side is the
// caller's sweep bound of its link on that segment, NaN when the segment does not exist or the bound is not finite and
// >= 0.  A NaN side widens nothing and fails every threshold test (a comparison with NaN is false).
HFB_HD double sweep_side(double s) { return s >= 0 && s <= DBL_MAX ? s : NAN; }
// s / 2 rounded up: exact but for subnormals
HFB_HD double half_ru(double s) {
#ifdef __CUDA_ARCH__
  return __dmul_ru(s, 0.5);
#else
  const double h = s * 0.5;
  return h + h < s ? nextafter(h, INFINITY) : h;
#endif
}
// the widening of a link or pair whose side thresholds are r and l: half the larger one that is not NaN, rounded up;
// 0 when both are NaN.  A pair whose boxes are more than this apart is farther apart than half of either threshold.
HFB_HD double sweep_reach(double r, double l) {
  double s = 0;
  if (r > s) s = r;
  if (l > s) s = l;
  return half_ru(s);
}
// the motion of configuration g among motions [m0, m1): the last one starting at or before it (off[m0] <= g <
// off[m1]; an empty motion starts where the next one does)
HFB_HD unsigned motion_of(const uint32_t* off, unsigned m0, unsigned m1, size_t g) {
  unsigned lo = m0, hi = m1;
  while (hi - lo > 1) {
    const unsigned mid = lo + (hi - lo) / 2;
    if (off[mid] <= g) lo = mid;
    else hi = mid;
  }
  return lo;
}
// the right and left sides of A object i = g * links + link, whose configuration g lies in the motion [g_lo, g_hi)
HFB_HD void sweep_sides(const double* sweep, size_t i, size_t links, size_t g_lo, size_t g_hi, double* r, double* l) {
  const size_t g = i / links;
  *r = g + 1 < g_hi ? sweep_side(sweep[i]) : NAN;
  *l = g > g_lo ? sweep_side(sweep[i - links]) : NAN;
}
// self pair t (config_pair's numbering), `sides` the right and left side of every A object: true when its collide()
// runs for certification -- both links have a box, and config_dist_pair holds with the pair's reach (sweep_reach of
// the sums of its links' sides, rounded up) in place of max_distance.  A pair it skips has a box gap larger than half
// of either threshold.
HFB_HD bool sweep_pair(const double* bb, const double* sides, uint32_t links, const uint32_t* tpl, uint32_t n_pairs,
                       uint32_t g0, size_t t, uint32_t* a, uint32_t* b) {
  const size_t g = g0 + t / n_pairs, k = t % n_pairs;
  const size_t i = g * links + tpl[2 * k], j = g * links + tpl[2 * k + 1];
  *a = (uint32_t)i;
  *b = (uint32_t)j;
  if (aabb_empty(bb + 6 * i) || aabb_empty(bb + 6 * j)) return false;
  const double w = sweep_reach(add_ru(sides[2 * i], sides[2 * j]), add_ru(sides[2 * i + 1], sides[2 * j + 1]));
  return config_dist_pair(bb, links, tpl, n_pairs, g0, t, w, a, b);
}

}  // namespace hfb
