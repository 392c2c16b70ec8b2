// Shape records, the lane-group cooperation policy and the per-shape support
// functions  argmax_{x in shape} <dir, x>  (swept-sphere radius excluded).
//
// Replaces details::getShapeSupport<NoSweptSphere>
//   (src/narrowphase/support_functions.cpp:111-437) and
//   details::getSupportTpl / MinkowskiDiff::set
//   (src/narrowphase/minkowski_difference.cpp:47-63, 78-285).
// ConvexBase: the reference switches to a neighbour hill-climb above 32 vertices
// (:425-437); here the argmax is always exhaustive and split over the G lanes
// that own the pair (strict '>' + lowest index on ties == the linear scan of
// :401-421, and equal to the hill-climb result whenever the maximum is unique).
#pragma once
#include "../../include/hppfcl_b200.h"
#include "hfb_math.cuh"

namespace hfb {

#define HFB_DUMMY_PRECISION 1e-12  // Eigen::NumTraits<double>::dummy_precision()
// Box support "inflate" (support_functions.cpp:146): function-local static fixed by
// the first direction a process queries; (-1,0,0) with the default guess => 1+1e-10.
#define HFB_BOX_INFLATE (1 + 1e-10)
#define HFB_INFLATE (1 + 1e-10)

// ---- lane-group policy: G lanes of a warp own one pair ---------------------
// Four primitives -- lane(), mask(), shfl_xor(), sync() -- carry everything the pair code does across lanes;
// argmax() and the two reductions of hfb_epa.cuh are written on top of them.  On the device they are the warp
// intrinsics.  tests/emu (HFB_LANE_SIM) supplies host versions in which the G lanes of a group are G threads
// meeting at barriers, so that the cooperative paths run -- and race -- on the CPU as well.
#if !defined(__CUDACC__) && defined(HFB_LANE_SIM)
namespace lanesim {  // defined by the test harness
int lane();
void sync();
double shfl_xor(double v, int off);
int shfl_xor(int v, int off);
const void* peer_workspace(int lane);  // the EPA workspace lane `lane` of this group registered (private copies)
void trace_bvh_state(int state);       // the phase a lane of the BVH walk waits for, once per scheduling round
}  // namespace lanesim
#endif
template <int G>
struct Coop {
#if defined(__CUDACC__)
  static __device__ __forceinline__ int lane() { return (int)(threadIdx.x & (G - 1)); }
  static __device__ __forceinline__ unsigned mask() {
    if (G == 32) return 0xffffffffu;
    unsigned wl = threadIdx.x & 31u;
    return (((1u << (G & 31)) - 1u)) << (wl & ~(unsigned)(G - 1));  // (G & 31: no over-wide shift in the dead G == 32 copy)
  }
  static __device__ __forceinline__ double shfl_xor(double v, int off) { return __shfl_xor_sync(mask(), v, off); }
  static __device__ __forceinline__ int shfl_xor(int v, int off) { return __shfl_xor_sync(mask(), v, off); }
  static __device__ __forceinline__ void sync() { __syncwarp(mask()); }
#define HFB_COOP_FN static __device__ __forceinline__
#elif defined(HFB_LANE_SIM)
  static int lane() { return lanesim::lane(); }
  static unsigned mask() { return 0u; }
  static double shfl_xor(double v, int off) { return lanesim::shfl_xor(v, off); }
  static int shfl_xor(int v, int off) { return lanesim::shfl_xor(v, off); }
  static void sync() { lanesim::sync(); }
#define HFB_COOP_FN static inline
#endif
#if defined(__CUDACC__) || defined(HFB_LANE_SIM)
  // group-wide argmax; ties -> lowest index; result broadcast to every lane
  HFB_COOP_FN void argmax(double& v, int& idx) {
#pragma unroll
    for (int off = G / 2; off > 0; off >>= 1) {
      double ov = shfl_xor(v, off);
      int oi = shfl_xor(idx, off);
      if (ov > v || (ov == v && oi < idx)) {
        v = ov;
        idx = oi;
      }
    }
  }
#undef HFB_COOP_FN
#endif
};
template <>
struct Coop<1> {
  static HFB_HD int lane() { return 0; }
  static HFB_HD unsigned mask() { return 0xffffffffu; }
  static HFB_HD double shfl_xor(double v, int) { return v; }
  static HFB_HD int shfl_xor(int v, int) { return v; }
  static HFB_HD void argmax(double&, int&) {}
  static HFB_HD void sync() {}
};

// ---- device-side shape record ----------------------------------------------
struct ShapeD {
  int type;          // HFB_GEOM_*
  double p0, p1, p2; // see hfb_shape
  double ssr;
  // CONVEX: SoA vertex arrays (global or shared memory) and count
  const double* cx;
  const double* cy;
  const double* cz;
  int nv;
  v3 center;         // aabb_local.center() (BoundingVolumeGuess)
  // TRIANGLE: vertices by value (possibly pre-transformed, narrowphase.h:327-329)
  v3 ta, tb, tc;
};

// capability mask of a kernel instantiation: which shape classes it may meet
// CAP_INLINE_PRIM: expand the primitive supports in place (the BVH walk: a call inside the leaf test
// costs more in spills than the duplicate code costs in instruction fetch)
// CAP_PLANE: the Plane / Halfspace closed forms (only the kernels their pair classes are binned to)
enum { CAP_PRIM = 1, CAP_CONVEX = 2, CAP_TRI = 4, CAP_INLINE_PRIM = 8, CAP_PLANE = 16 };

HFB_HD v3 prim_support_inl(int type, double p0, double p1, double p2, v3 dir) {
  v3 r = mk(0, 0, 0);
  struct { int type; double p0, p1, p2; } s = {type, p0, p1, p2};
  {
    switch (s.type) {
      case HFB_GEOM_BOX: {  // :141-157
        r.x = ((dir.x > HFB_DUMMY_PRECISION) ? s.p0 : 0.0) +
              ((dir.x < -HFB_DUMMY_PRECISION) ? (-HFB_BOX_INFLATE * s.p0) : 0.0);
        r.y = ((dir.y > HFB_DUMMY_PRECISION) ? s.p1 : 0.0) +
              ((dir.y < -HFB_DUMMY_PRECISION) ? (-HFB_BOX_INFLATE * s.p1) : 0.0);
        r.z = ((dir.z > HFB_DUMMY_PRECISION) ? s.p2 : 0.0) +
              ((dir.z < -HFB_DUMMY_PRECISION) ? (-HFB_BOX_INFLATE * s.p2) : 0.0);
      } break;
      case HFB_GEOM_SPHERE:  // :164-176 (radius lives in the swept-sphere radius)
        break;
      case HFB_GEOM_CAPSULE:  // :206-222
        if (dir.z > HFB_DUMMY_PRECISION) r.z = s.p1;
        else if (dir.z < -HFB_DUMMY_PRECISION) r.z = -s.p1;
        break;
      case HFB_GEOM_ELLIPSOID: {  // :183-199
        double a2 = s.p0 * s.p0, b2 = s.p1 * s.p1, c2 = s.p2 * s.p2;
        v3 v = mk(a2 * dir.x, b2 * dir.y, c2 * dir.z);
        double d = sqrt(dot(v, dir));
        r = v / d;
      } break;
      case HFB_GEOM_CYLINDER: {  // :281-317
        double half_h = s.p1, rad = s.p0;
        const bool aligned = fabs(dir.x) <= HFB_DUMMY_PRECISION && fabs(dir.y) <= HFB_DUMMY_PRECISION;
        if (aligned) half_h *= HFB_INFLATE;
        if (dir.z > HFB_DUMMY_PRECISION) r.z = half_h;
        else if (dir.z < -HFB_DUMMY_PRECISION) r.z = -half_h;
        else { r.z = 0; rad *= HFB_INFLATE; }
        if (!aligned) {
          double z = dir.x * dir.x + dir.y * dir.y;
          double nx = dir.x, ny = dir.y;
          if (z > 0) { double q = sqrt(z); nx = dir.x / q; ny = dir.y / q; }
          r.x = nx * rad;
          r.y = ny * rad;
        }
      } break;
      case HFB_GEOM_CONE: {  // :229-274
        double h = s.p1, rad0 = s.p0;
        if (fabs(dir.x) <= HFB_DUMMY_PRECISION && fabs(dir.y) <= HFB_DUMMY_PRECISION) {
          r.z = (dir.z > HFB_DUMMY_PRECISION) ? h : (-HFB_INFLATE * h);
        } else {
          double zdist = dir.x * dir.x + dir.y * dir.y;
          double len = zdist + dir.z * dir.z;
          zdist = sqrt(zdist);
          bool apex = false;
          if (!(dir.z <= 0)) {
            len = sqrt(len);
            double sin_a = rad0 / sqrt(rad0 * rad0 + 4 * h * h);
            apex = dir.z > len * sin_a;
          }
          if (apex) {
            r = mk(0, 0, h);
          } else {
            double rad = rad0 / zdist;
            r = mk(rad * dir.x, rad * dir.y, -h);
          }
        }
      } break;
      default:
        break;
    }
  }
  return r;
}
// primitive supports, out of line on the device: one copy of this code serves both operands of
// the Minkowski difference (inlined twice it dominated the GJK loop's instruction footprint and the
// kernel stalled on instruction fetch)
HFB_HD_NOINLINE v3 prim_support(int type, double p0, double p1, double p2, v3 dir) {
  return prim_support_inl(type, p0, p1, p2, dir);
}

template <int G, int CAPS>
HFB_HD v3 shape_support(const ShapeD& s, v3 dir, int& hint) {
  v3 r = mk(0, 0, 0);
  if ((CAPS & CAP_CONVEX) && s.type == HFB_GEOM_CONVEX) {
    // exhaustive argmax, striped over the group's lanes.  It must equal the serial scan (start from vertex 0,
    // move on strictly greater) for EVERY input, including a NaN direction -- GJK does produce one now and
    // then (0/0 in the projection of a degenerate simplex) and carries on: the serial scan then keeps
    // vertex 0, because vertex 0 is taken unconditionally and nothing compares greater than NaN, while
    // elsewhere a NaN never wins.  So a NaN at index 0 is made the winner (+inf, index -1 < every index),
    // a NaN at the head of another lane's stripe is skipped, and no NaN reaches the cross-lane reduction
    // (where it would leave the lanes of a group with different answers).
    double best = -(double)INFINITY;
    int bi = 0x7fffffff;
    int i = Coop<G>::lane();
    // head of the lane's stripe: its first dot that is a number -- or the NaN at vertex 0
    for (; i < s.nv; i += G) {
      const double d = (s.cx[i] * dir.x + s.cy[i] * dir.y) + s.cz[i] * dir.z;
      if (d == d) {
        best = d;
        bi = i;
        i += G;
        break;
      }
      if (i == 0) {
        best = (double)INFINITY;
        bi = -1;
        i += G;
        break;
      }
    }
    // the rest: a NaN never passes '>' (a plain loop the compiler unrolls, as before the NaN rule)
#pragma unroll 4
    for (; i < s.nv; i += G) {
      const double d = (s.cx[i] * dir.x + s.cy[i] * dir.y) + s.cz[i] * dir.z;
      if (d > best) {
        best = d;
        bi = i;
      }
    }
    Coop<G>::argmax(best, bi);
    if (bi < 0) bi = 0;
    hint = bi;
    return mk(s.cx[bi], s.cy[bi], s.cz[bi]);
  }
  if ((CAPS & CAP_TRI) && s.type == HFB_GEOM_TRIANGLE) {  // :111-134
    double dota = dot(dir, s.ta), dotb = dot(dir, s.tb), dotc = dot(dir, s.tc);
    if (dota > dotb) {
      r = (dotc > dota) ? s.tc : s.ta;
    } else {
      r = (dotc > dotb) ? s.tc : s.tb;
    }
    return r;
  }
  if (CAPS & CAP_PRIM) {
    if (CAPS & CAP_INLINE_PRIM) return prim_support_inl(s.type, s.p0, s.p1, s.p2, dir);
    return prim_support(s.type, s.p0, s.p1, s.p2, dir);
  }
  return r;
}

// ---- MinkowskiDiff (minkowski_difference.h:57-186) --------------------------
struct MinkD {
  m3 oR1;   // R0^T R1
  v3 ot1;   // R0^T (t1 - t0)
  double ssr0, ssr1;  // swept_sphere_radius[2] incl. sphere/capsule radii (:103-125,182-201)
  bool identity;
  bool normalize_support_direction;  // both ConvexBase (:261-266)
};

HFB_HD void mink_radii(const ShapeD& s0, const ShapeD& s1, MinkD& md) {
  md.ssr0 = s0.ssr;
  if (s0.type == HFB_GEOM_SPHERE || s0.type == HFB_GEOM_CAPSULE) md.ssr0 += s0.p0;
  md.ssr1 = s1.ssr;
  if (s1.type == HFB_GEOM_SPHERE || s1.type == HFB_GEOM_CAPSULE) md.ssr1 += s1.p0;
  md.normalize_support_direction = (s0.type == HFB_GEOM_CONVEX) && (s1.type == HFB_GEOM_CONVEX);
}
// MinkowskiDiff::set(shape0, shape1, tf0, tf1)  (.cpp:269-285)
HFB_HD void mink_set(const ShapeD& s0, const ShapeD& s1, const xf& tf0, const xf& tf1, MinkD& md) {
  md.oR1 = mtmulm(tf0.R, tf1.R);
  md.ot1 = mtmul(tf0.R, tf1.T - tf0.T);
  md.identity = is_identity(md.oR1, HFB_DUMMY_PRECISION) && is_zero(md.ot1, HFB_DUMMY_PRECISION);
  mink_radii(s0, s1, md);
}
// MinkowskiDiff::set(shape0, shape1)  (.cpp:293-305)
HFB_HD void mink_set_identity(const ShapeD& s0, const ShapeD& s1, MinkD& md) {
  md.oR1.r0 = mk(1, 0, 0);
  md.oR1.r1 = mk(0, 1, 0);
  md.oR1.r2 = mk(0, 0, 1);
  md.ot1 = mk(0, 0, 0);
  md.identity = true;
  mink_radii(s0, s1, md);
}

// getSupportTpl (.cpp:47-63): support0 along dir, support1 along -oR1^T dir
template <int G, int CAPS>
HFB_HD void mink_support(const ShapeD& s0, const ShapeD& s1, const MinkD& md, v3 dir, v3& w0, v3& w1,
                         int& hint0, int& hint1) {
  w0 = shape_support<G, CAPS>(s0, dir, hint0);
  if (md.identity) {
    w1 = shape_support<G, CAPS>(s1, -dir, hint1);
  } else {
    w1 = shape_support<G, CAPS>(s1, -mtmul(md.oR1, dir), hint1);
    w1 = mmul(md.oR1, w1) + md.ot1;
  }
}
// The same, with what a pair's iterations never write -- the relative pose oR1 / ot1 and the shapes' parameters --
// read from `mr` (the GJK passes keep them in a per-thread store in shared memory, SlotStore in hfb_gjkpass.cu).  The
// pose is read once before the second support call and once after it, so that it is not live across the call.
template <int G, int CAPS, class Mink>
HFB_HD void mink_support(const ShapeD& s0, const ShapeD& s1, const MinkD& md, v3 dir, v3& w0, v3& w1,
                         int& hint0, int& hint1, const Mink& mr) {
  w0 = shape_support<G, CAPS>(mr.shape0(s0), dir, hint0);
  if (md.identity) {
    w1 = shape_support<G, CAPS>(mr.shape1(s1), -dir, hint1);
  } else {
    w1 = shape_support<G, CAPS>(mr.shape1(s1), -mtmul(mr.oR1(), dir), hint1);
    w1 = mmul(mr.oR1(), w1) + mr.ot1();
  }
}

}  // namespace hfb
