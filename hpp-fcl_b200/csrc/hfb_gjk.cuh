// GJK for one shape pair, register-resident, branch-uniform across the lanes
// that own the pair.
//
// Replaces details::GJK::evaluate / checkConvergence / project{Line,Triangle,
// Tetrahedra}Origin / getWitnessPointsAndNormal (src/narrowphase/gjk.cpp:94-1010)
// and Project::project{Triangle,Tetrahedra}Origin (src/intersect.cpp:570-705).
//
// Design differences from the reference (same arithmetic, different structure):
//  * the simplex is held BY VALUE in vertex order (no store_v/free_v pointer
//    pool, gjk.cpp:195-200): slot identity has no numerical meaning, only the
//    order of simplex.vertex[] does, and that order is reproduced exactly;
//  * projectTetrahedraOrigin's 24-leaf decision tree (:656-1005) is evaluated as
//    twelve sign predicates + a region decode, then ONE update per region class
//    (point / segment / triangle), which keeps the warp on a single path.
#pragma once
#include "hfb_shapes.cuh"

namespace hfb {

struct SV {  // GJK::SimplexV (gjk.h:55-61)
  v3 w0, w1, w;
};
// A vertex whose support points w0 / w1 are kept in slot `slot` of a per-thread store outside the registers (the GJK
// passes, hfb_gjkpass.cu): the iterations only read w.
struct SVSlot {
  v3 w;
  int slot;
};

struct GjkParams {  // per-batch constants (GJKSolver::set, narrowphase.h:162-244)
  double tolerance;
  double distance_upper_bound;
  unsigned max_iterations;
  int variant;
  int criterion;
  int criterion_type;
};

template <class V>
struct GjkStateT {
  V s0, s1, s2, s3;  // simplex.vertex[0..3]
  int rank;
  v3 ray;
  double distance;
  int status;
  int hint0, hint1;
  unsigned iterations;
};
using GjkState = GjkStateT<SV>;

template <class V>
HFB_HD V pick(const GjkStateT<V>& g, int i) { return i == 0 ? g.s0 : (i == 1 ? g.s1 : (i == 2 ? g.s2 : g.s3)); }
template <class V>
HFB_HD void put(GjkStateT<V>& g, int i, const V& v) {
  if (i == 0) g.s0 = v;
  else if (i == 1) g.s1 = v;
  else if (i == 2) g.s2 = v;
  else g.s3 = v;
}

// GJK::getSupport (gjk.h:163-167)
template <int G, int CAPS>
HFB_HD SV gjk_support(const ShapeD& a, const ShapeD& b, const MinkD& md, v3 d, int& h0, int& h1) {
  SV sv;
  mink_support<G, CAPS>(a, b, md, d, sv.w0, sv.w1, h0, h1);
  sv.w = sv.w0 - sv.w1;
  return sv;
}
// the same, with the pose and the shapes' parameters read from `mr` (see mink_support)
template <int G, int CAPS, class Mink>
HFB_HD SV gjk_support(const ShapeD& a, const ShapeD& b, const MinkD& md, v3 d, int& h0, int& h1, const Mink& mr) {
  SV sv;
  mink_support<G, CAPS>(a, b, md, d, sv.w0, sv.w1, h0, h1, mr);
  sv.w = sv.w0 - sv.w1;
  return sv;
}

// Where gjk_step appends a support point and the witness points read them back: InRegs keeps the whole SV in the
// simplex (every caller but the GJK passes, which keep w0 / w1 in a per-thread store of their own, SlotStore in
// hfb_gjkpass.cu).  append puts `nv` at simplex.vertex[g.rank] and returns its w; support_points gives a vertex's
// w0 / w1; inline_projections: closest_points_inl inlines the triangle projection of a rank-3 simplex, and the segment
// projections it calls, instead of calling them out of line (in a kernel held to few registers an out-of-line call
// saves and restores registers in local memory).  The tetrahedron projection is always called out of line: GJK's
// witness points never reach it (a rank-4 simplex encloses the origin, which is a collision), and inlined it would
// add ~20 KB of code.  support: GJK::getSupport with the pose and the shapes' parameters of the MinkD and the shape
// records (the passes read them from their store); ssr, upper_bound: the sum of the radii and the early-stop bound
// gjk_begin put in the loop state.
struct InRegs {
  using V = SV;
  static constexpr bool inline_projections = false;
  template <int G, int CAPS>
  HFB_HD SV support(const ShapeD& a, const ShapeD& b, const MinkD& md, v3 d, int& h0, int& h1) const {
    return gjk_support<G, CAPS>(a, b, md, d, h0, h1);
  }
  template <class Loop>
  HFB_HD double ssr(const Loop& L) const {
    return L.ssr;
  }
  template <class Loop>
  HFB_HD double upper_bound(const Loop& L, const GjkParams&) const {
    return L.upper_bound;
  }
  HFB_HD v3 append(GjkState& g, const SV& nv) const {
    put(g, g.rank, nv);
    return nv.w;
  }
  HFB_HD void support_points(const SV& v, v3& w0, v3& w1) const {
    w0 = v.w0;
    w1 = v.w1;
  }
};

// region codes of the simplex projections
enum { RG_A = 0, RG_AB, RG_AC, RG_AD, RG_ABC, RG_ACD, RG_ADB, RG_INSIDE };

// originToSegment (:502-515): ray = ((AX.X) A + t X) / |AX|^2
HFB_HD v3 ray_segment(v3 A, v3 X, v3 AX, double t) {
  v3 r = dot(AX, X) * A + t * X;
  return r / sqn(AX);
}
// originToTriangle (:517-541), ABCdotAO != 0
HFB_HD v3 ray_triangle(v3 N, double NdotAO) { return (-NdotAO / sqn(N)) * N; }

// The new ray as a projection leaves it.  With DEFER (the default variant's GJK passes) a segment's or a face's ray is
// not formed by the projection but left in `r`: ray_segment(A, X, X - A, t) (every segment's AX is X - A, the same
// operation on the same values) or ray_triangle(N = A, NdotAO = t), which gjk_step evaluates after the projection of
// every rank, so that a warp whose lanes project simplices of different ranks runs each formula, and its divisions,
// once.  Without DEFER the projection forms the ray itself (the other kernels: carrying the inputs costs them more in
// registers than it saves).  A vertex or a zero ray is always set in g.ray at once.
enum { RAY_SET = 0, RAY_SEGMENT, RAY_TRIANGLE };
struct RayOf {
  int kind;
  v3 A, X;
  double t;
};
template <bool DEFER, class V>
HFB_HD void ray_of_segment(GjkStateT<V>& g, RayOf& r, v3 A, v3 X, double t) {
  if (!DEFER) {
    g.ray = ray_segment(A, X, X - A, t);
    return;
  }
  r.kind = RAY_SEGMENT;
  r.A = A;
  r.X = X;
  r.t = t;
}
template <bool DEFER, class V>
HFB_HD void ray_of_triangle(GjkStateT<V>& g, RayOf& r, v3 N, double NdotAO) {
  if (!DEFER) {
    g.ray = ray_triangle(N, NdotAO);
    return;
  }
  r.kind = RAY_TRIANGLE;
  r.A = N;
  r.t = NdotAO;
}

// The projections read only w of each vertex and move whole vertices (V: SV or SVSlot).
// projectLineOrigin (:543-569). A = newest = s1, B = s0.
template <bool DEFER, class V>
HFB_HD bool project_line(GjkStateT<V>& g, RayOf& r) {
  const v3 A = g.s1.w, B = g.s0.w;
  const v3 AB = B - A;
  const double d = dot(AB, -A);
  if (d == 0) {
    g.ray = A;
    g.s0 = g.s1;
    g.rank = 1;
    return is_zero(A, HFB_DUMMY_PRECISION);
  } else if (d < 0) {
    g.ray = A;
    g.s0 = g.s1;
    g.rank = 1;
  } else {
    ray_of_segment<DEFER>(g, r, A, B, d);  // next = [b, a]: order unchanged
  }
  return false;
}

// projectTriangleOrigin (:571-611). A = s2, B = s1, C = s0.
template <bool DEFER, class V>
HFB_HD bool project_triangle(GjkStateT<V>& g, RayOf& r) {
  const v3 A = g.s2.w, B = g.s1.w, C = g.s0.w;
  const v3 AB = B - A, AC = C - A, ABC = cross(AB, AC);
  int region;
  double t = 0;
  const double edgeAC2o = dot(cross(ABC, AC), -A);
  if (edgeAC2o >= 0) {
    const double towardsC = dot(AC, -A);
    if (towardsC >= 0) {
      region = RG_AC;
      t = towardsC;
    } else {
      const double towardsB = dot(AB, -A);
      if (towardsB < 0) region = RG_A;
      else { region = RG_AB; t = towardsB; }
    }
  } else {
    const double edgeAB2o = dot(cross(AB, ABC), -A);
    if (edgeAB2o >= 0) {
      const double towardsB = dot(AB, -A);
      if (towardsB < 0) region = RG_A;
      else { region = RG_AB; t = towardsB; }
    } else {
      region = RG_ABC;
    }
  }
  switch (region) {
    case RG_AC:
    case RG_AB: {  // AC: next = [c, a]; AB: next = [b, a]
      const bool ac = region == RG_AC;
      ray_of_segment<DEFER>(g, r, A, ac ? C : B, t);
      if (!ac) g.s0 = g.s1;
      g.s1 = g.s2;
      g.rank = 2;
      return false;
    }
    case RG_A:
      g.ray = A;
      g.s0 = g.s2;
      g.rank = 1;
      return false;
    default: {  // originToTriangle(a, b, c, ABC, ABC.dot(-A))
      const double dAO = dot(ABC, -A);
      if (dAO == 0) {  // next = [c, b, a]
        g.ray = mk(0, 0, 0);
        return true;
      }
      if (!(dAO > 0)) {  // next = [b, c, a]
        V tmp = g.s0;
        g.s0 = g.s1;
        g.s1 = tmp;
      }
      ray_of_triangle<DEFER>(g, r, ABC, dAO);
      return false;
    }
  }
}

// projectTetrahedraOrigin (:613-1010). A = s3, B = s2, C = s1, D = s0.
template <bool DEFER, class V>
HFB_HD bool project_tetra(GjkStateT<V>& g, RayOf& r) {
  const v3 A = g.s3.w, B = g.s2.w, C = g.s1.w, D = g.s0.w;
  const double aa = sqn(A);
  const double da = dot(D, A), db = dot(D, B), dc = dot(D, C), dd = dot(D, D);
  const double da_aa = da - aa;
  const double ca = dot(C, A), cb = dot(C, B), cc = dot(C, C);
  const double cd = dc;
  const double ca_aa = ca - aa;
  const double ba = dot(B, A), bb = dot(B, B);
  const double bc = cb, bd = db;
  const double ba_aa = ba - aa, ba_ca = ba - ca, ca_da = ca - da, da_ba = da - ba;
  const v3 a_cross_b = cross(A, B);
  const v3 a_cross_c = cross(A, C);
  const double D_axb = dot(D, a_cross_b);
  const double C_axb = dot(C, a_cross_b);
  const double D_axc = dot(D, a_cross_c);

  // the twelve predicates (names as in the reference's generated comments)
  const bool a10 = ba_aa <= 0;
  const bool a11 = ca_aa <= 0;
  const bool a12 = da_aa <= 0;
  const bool a3 = -D_axb <= 0;
  const bool a1 = C_axb <= 0;
  const bool a2 = D_axc <= 0;
  const bool a9 = ba * da_ba + bd * ba_aa - bb * da_aa <= 0;
  const bool a8 = da * da_ba + dd * ba_aa - db * da_aa <= 0;
  const bool a4 = ba * ba_ca + bb * ca_aa - bc * ba_aa <= 0;
  const bool a5 = ca * ba_ca + cb * ca_aa - cc * ba_aa <= 0;
  const bool a6 = ca * ca_da + cc * da_aa - cd * ca_aa <= 0;
  const bool a7 = da * ca_da + dc * da_aa - dd * ca_aa <= 0;

  // region decode: same truth table as the reference's nested ifs
  int region;
  if (a10) {
    if (a3) {
      if (a9) {
        if (a12) region = a4 ? RG_ABC : RG_AB;
        else region = a4 ? (a5 ? (a6 ? RG_ACD : RG_AC) : RG_ABC) : RG_AB;
      } else {
        region = a8 ? RG_ADB : (a6 ? (a7 ? RG_AD : RG_ACD) : (a7 ? RG_AD : RG_AC));
      }
    } else {
      if (a1) region = a4 ? (a5 ? (a6 ? RG_ACD : RG_AC) : RG_ABC) : RG_AB;
      else region = a2 ? (a6 ? (a7 ? RG_AD : RG_ACD) : (a11 ? RG_AC : RG_AD)) : RG_INSIDE;
    }
  } else {
    if (a11) {
      if (a2) {
        if (a12) region = a6 ? (a7 ? (a8 ? RG_ADB : RG_AD) : RG_ACD) : (a5 ? RG_AC : RG_ABC);
        else region = a5 ? (a6 ? RG_ACD : RG_AC) : (a1 ? RG_ABC : RG_ACD);
      } else {
        if (a1) region = a5 ? RG_AC : RG_ABC;
        else region = a3 ? (a8 ? RG_ADB : RG_AD) : RG_INSIDE;
      }
    } else {
      if (a12) {
        if (a3) region = a7 ? (a8 ? RG_ADB : RG_AD) : (a2 ? RG_ACD : RG_ADB);
        else region = a2 ? (a7 ? RG_AD : RG_ACD) : RG_INSIDE;
      } else {
        region = RG_A;
      }
    }
  }

  if (region == RG_INSIDE) {  // next = [d, c, b, a]: unchanged
    g.ray = mk(0, 0, 0);
    return true;
  }
  if (region == RG_A) {
    g.ray = A;
    g.s0 = g.s3;
    g.rank = 1;
    return false;
  }
  if (region <= RG_AD) {  // segment A-X, next = [x, a]
    const bool isB = region == RG_AB, isC = region == RG_AC;
    const v3 X = isB ? B : (isC ? C : D);
    const double t = isB ? -ba_aa : (isC ? -ca_aa : -da_aa);
    ray_of_segment<DEFER>(g, r, A, X, t);
    const V sx = isB ? g.s2 : (isC ? g.s1 : g.s0);
    g.s0 = sx;
    g.s1 = g.s3;
    g.rank = 2;
    return false;
  }
  // triangle A-X-Y: originToTriangle(a, x, y, (X-A)x(Y-A), dAO)
  //   ABC: x=b y=c dAO=-C.(AxB) ; ACD: x=c y=d dAO=-D.(AxC) ; ADB: x=d y=b dAO=+D.(AxB)
  const bool tABC = region == RG_ABC, tACD = region == RG_ACD;
  const v3 X = tABC ? B : (tACD ? C : D);
  const v3 Y = tABC ? C : (tACD ? D : B);
  const V sx = tABC ? g.s2 : (tACD ? g.s1 : g.s0);
  const V sy = tABC ? g.s1 : (tACD ? g.s0 : g.s2);
  const double dAO = tABC ? -C_axb : (tACD ? -D_axc : D_axb);
  const v3 N = cross(X - A, Y - A);
  g.rank = 3;
  g.s2 = g.s3;
  if (dAO == 0) {  // next = [y, x, a]; ray = 0.  (return value ignored by the caller
    g.s0 = sy;     // in the reference; rl == 0 then reports Collision, gjk.cpp:354)
    g.s1 = sx;
    g.ray = mk(0, 0, 0);
    return false;
  }
  if (dAO > 0) {  // next = [y, x, a]
    g.s0 = sy;
    g.s1 = sx;
  } else {        // next = [x, y, a]
    g.s0 = sx;
    g.s1 = sy;
  }
  ray_of_triangle<DEFER>(g, r, N, dAO);
  return false;
}

// GJK::checkConvergence (:372-425)
HFB_HD bool gjk_converged(const GjkParams& P, v3 ray, v3 w, double rl, double& alpha, double omega) {
  const double tol = P.tolerance;
  if (P.criterion == HFB_CRIT_DEFAULT) {
    alpha = fmax(alpha, omega);
    const double diff = rl - alpha;
    return ((diff - (tol + tol * rl)) <= 0);
  }
  double diff;
  if (P.criterion == HFB_CRIT_DUALITY_GAP) {
    diff = 2 * dot(ray, ray - w);
  } else {
    alpha = fmax(alpha, omega);
    diff = rl * rl - alpha * alpha;
  }
  if (P.criterion_type == HFB_CRIT_ABSOLUTE) return ((diff - tol) <= 0);
  return (((diff / tol * rl) - tol * rl) <= 0);
}

// GJK::evaluate (:188-370)
// GJK::evaluate (gjk.cpp:188-370) as set-up + one-iteration steps, so that a kernel can interleave the
// iterations of different pairs (a lane whose pair is done takes the next pair instead of idling until
// the slowest pair of its warp converges).  gjk_evaluate below is the plain loop over the same pieces.
struct GjkLoop {  // what the do-while of the reference carries from one iteration to the next
  double alpha, rl;
  double ssr, upper_bound;
  int variant;
  v3 w, dir;
};

template <class V>
HFB_HD void gjk_begin(const MinkD& md, const GjkParams& P, v3 guess, int hint0, int hint1, GjkStateT<V>& g,
                      GjkLoop& L) {
  L.alpha = 0;
  g.iterations = 0;
  L.ssr = md.ssr0 + md.ssr1;
  L.upper_bound = P.distance_upper_bound + L.ssr;
  const double tol = P.tolerance;
  g.status = HFB_GJK_NO_COLLISION;
  g.distance = 0.0;
  g.rank = 0;
  g.hint0 = hint0;
  g.hint1 = hint1;

  L.rl = nrm(guess);
  if (L.rl < tol) {
    g.ray = mk(-1, 0, 0);
    L.rl = 1;
  } else {
    g.ray = guess;
  }
  L.variant = P.variant;
  L.w = g.ray;
  L.dir = g.ray;
}

// one pass through the body of the do-while; returns whether the loop goes on.  `st` appends the new support point
// and gives the relative pose and the shapes' parameters to the support calls (InRegs, or the passes' SlotStore; its
// vertex type is the simplex's).  MOMENTUM false: the caller guarantees L.variant is HFB_GJK_DEFAULT, so L.w and L.dir are written
// before they are read in every step and are not live from one step to the next.
template <int G, int CAPS, class Store = InRegs, bool MOMENTUM = true>
HFB_HD bool gjk_step(const ShapeD& sa, const ShapeD& sb, const MinkD& md, const GjkParams& P,
                     GjkStateT<typename Store::V>& g, GjkLoop& L, const Store& st = Store()) {
  const double tol = P.tolerance;
  // check A (:228-243)
  if (L.rl < tol) {
    g.status = HFB_GJK_COLLISION;
    g.distance = L.rl;
    return false;
  }
  // support direction (:246-278)
  if (!MOMENTUM || L.variant == HFB_GJK_DEFAULT) {
    L.dir = g.ray;
  } else if (L.variant == HFB_GJK_NESTEROV) {
    if (md.normalize_support_direction) {
      const double momentum = ((double)g.iterations + 2) / ((double)g.iterations + 3);
      const v3 y = momentum * g.ray + (1 - momentum) * L.w;
      const double y_norm = nrm(y);
      L.dir = momentum * L.dir / nrm(L.dir) + (1 - momentum) * y / y_norm;
    } else {
      const double momentum = ((double)g.iterations + 1) / ((double)g.iterations + 3);
      const v3 y = momentum * g.ray + (1 - momentum) * L.w;
      L.dir = momentum * L.dir + (1 - momentum) * y;
    }
  } else {  // Polyak
    const double momentum = 1 / ((double)g.iterations + 1);
    L.dir = momentum * L.dir + (1 - momentum) * g.ray;
  }

  // appendVertex(curr_simplex, -dir, support_hint) (:281)
  const SV nv = st.template support<G, CAPS>(sa, sb, md, -L.dir, g.hint0, g.hint1);
  L.w = st.append(g, nv);
  g.rank += 1;

  // check B (:288-293).  Without momentum L.dir is g.ray, and L.rl already holds nrm(g.ray), the same operation on the
  // same value: gjk_begin sets it with the ray, the end of every step that goes on recomputes it, and the passes'
  // load_running restores it with the ray.
  const double omega = dot(L.dir, L.w) / (MOMENTUM ? nrm(L.dir) : L.rl);
  if (omega > st.upper_bound(L, P)) {
    g.distance = omega - st.ssr(L);
    g.status = HFB_GJK_NO_COLLISION_EARLY_STOPPED;
    return false;
  }

  // drop the momentum when the Frank-Wolfe duality gap closes (:296-304)
  if (MOMENTUM && L.variant != HFB_GJK_DEFAULT) {
    const double fw_gap = 2 * dot(g.ray, g.ray - L.w);
    if (fw_gap - tol <= 0) {
      g.rank -= 1;  // removeVertex
      L.variant = HFB_GJK_DEFAULT;
      return true;  // `continue`: does not advance `iterations`
    }
  }

  // check C (:308-326)
  const bool cv = gjk_converged(P, g.ray, L.w, L.rl, L.alpha, omega);
  if (g.iterations > 0 && cv) {
    g.rank -= 1;  // removeVertex
    if (MOMENTUM && L.variant != HFB_GJK_DEFAULT) {
      L.variant = HFB_GJK_DEFAULT;
      return true;  // `continue`
    }
    g.distance = L.rl - st.ssr(L);
    g.status = (g.distance < tol) ? HFB_GJK_COLLISION_WITH_PENETRATION : HFB_GJK_NO_COLLISION;
    return false;
  }

  // simplex sub-solve (:330-350)
  bool inside;
  RayOf r;
  r.kind = RAY_SET;
  if (g.rank == 1) {
    g.ray = L.w;
    inside = false;
  } else if (g.rank == 2) {
    inside = project_line<!MOMENTUM>(g, r);
  } else if (g.rank == 3) {
    inside = project_triangle<!MOMENTUM>(g, r);
  } else {
    inside = project_tetra<!MOMENTUM>(g, r);
  }
  if constexpr (!MOMENTUM) {
    if (r.kind == RAY_SEGMENT) g.ray = ray_segment(r.A, r.X, r.X - r.A, r.t);
    else if (r.kind == RAY_TRIANGLE) g.ray = ray_triangle(r.A, r.t);
  }
  L.rl = nrm(g.ray);
  if (inside || L.rl == 0) {
    g.status = HFB_GJK_COLLISION;
    g.distance = L.rl;
    return false;
  }
  g.iterations += 1;
  if (!(g.iterations < P.max_iterations)) g.status = HFB_GJK_FAILED;
  return g.status == HFB_GJK_NO_COLLISION;
}

template <int G, int CAPS>
HFB_HD void gjk_evaluate(const ShapeD& sa, const ShapeD& sb, const MinkD& md, const GjkParams& P,
                         v3 guess, int hint0, int hint1, GjkState& g) {
  GjkLoop L;
  gjk_begin(md, P, guess, hint0, hint1, g, L);
  while (gjk_step<G, CAPS>(sa, sb, md, P, g, L)) {
  }
}

// ---- Project::*Origin (src/intersect.cpp:570-705), parameterization only ----
struct Param4 {
  double p0, p1, p2, p3;
  double sqr_distance;
  unsigned encode;
};
HFB_HD void pset(Param4& r, int i, double v) {
  if (i == 0) r.p0 = v;
  else if (i == 1) r.p1 = v;
  else if (i == 2) r.p2 = v;
  else r.p3 = v;
}
// The segment and triangle projections are called out of line (one copy per kernel) or, in their _inl form with INL
// set, inlined together with the projections they call (see InRegs::inline_projections).
HFB_HD Param4 proj_line_origin_inl(v3 a, v3 b) {
  Param4 res;
  res.p0 = res.p1 = res.p2 = res.p3 = 0;
  res.sqr_distance = -1;
  res.encode = 0;
  const v3 d = b - a;
  const double l = sqn(d);
  if (l > 0) {
    const double t = -dot(a, d);
    res.p1 = (t >= l) ? 1 : ((t <= 0) ? 0 : (t / l));
    res.p0 = 1 - res.p1;
    if (t >= l) {
      res.sqr_distance = sqn(b);
      res.encode = 2;
    } else if (t <= 0) {
      res.sqr_distance = sqn(a);
      res.encode = 1;
    } else {
      res.sqr_distance = sqn(a + d * res.p1);
      res.encode = 3;
    }
  }
  return res;
}
HFB_HD_NOINLINE Param4 proj_line_origin(v3 a, v3 b) { return proj_line_origin_inl(a, b); }
template <bool INL>
HFB_HD Param4 proj_triangle_origin_inl(v3 a, v3 b, v3 c) {
  Param4 res;
  res.p0 = res.p1 = res.p2 = res.p3 = 0;
  res.sqr_distance = -1;
  res.encode = 0;
  const v3 dl0 = a - b, dl1 = b - c, dl2 = c - a;
  const v3 n = cross(dl0, dl1);
  const double l = sqn(n);
  if (l > 0) {
    double mindist = -1;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const v3 vi = i == 0 ? a : (i == 1 ? b : c);
      const v3 dli = i == 0 ? dl0 : (i == 1 ? dl1 : dl2);
      if (dot(vi, cross(dli, n)) > 0) {
        const int j = i == 2 ? 0 : i + 1;
        const v3 vj = j == 0 ? a : (j == 1 ? b : c);
        const Param4 rl = INL ? proj_line_origin_inl(vi, vj) : proj_line_origin(vi, vj);
        if (mindist < 0 || rl.sqr_distance < mindist) {
          mindist = rl.sqr_distance;
          res.encode = (unsigned)(((rl.encode & 1) ? 1 << i : 0) + ((rl.encode & 2) ? 1 << j : 0));
          pset(res, i, rl.p0);
          pset(res, j, rl.p1);
          pset(res, j == 2 ? 0 : j + 1, 0);
        }
      }
    }
    if (mindist < 0) {
      const double d = dot(a, n);
      const double s = sqrt(l);
      const v3 o_to_project = n * (d / l);
      mindist = sqn(o_to_project);
      res.encode = 7;
      res.p0 = nrm(cross(dl1, b - o_to_project)) / s;
      res.p1 = nrm(cross(dl2, c - o_to_project)) / s;
      res.p2 = 1 - res.p0 - res.p1;
    }
    res.sqr_distance = mindist;
  }
  return res;
}
HFB_HD_NOINLINE Param4 proj_triangle_origin(v3 a, v3 b, v3 c) { return proj_triangle_origin_inl<false>(a, b, c); }
HFB_HD_NOINLINE Param4 proj_tetra_origin(v3 a, v3 b, v3 c, v3 d) {
  Param4 res;
  res.p0 = res.p1 = res.p2 = res.p3 = 0;
  res.sqr_distance = -1;
  res.encode = 0;
  const v3 dl0 = a - d, dl1 = b - d, dl2 = c - d;
  const double vl = triple(dl0, dl1, dl2);
  const bool ng = (vl * dot(a, cross(b - c, a - b))) <= 0;
  if (ng && fabs(vl) > 0) {
    double mindist = -1;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const int j = i == 2 ? 0 : i + 1;
      const v3 dli = i == 0 ? dl0 : (i == 1 ? dl1 : dl2);
      const v3 dlj = j == 0 ? dl0 : (j == 1 ? dl1 : dl2);
      const double s = vl * dot(d, cross(dli, dlj));
      if (s > 0) {
        const v3 vi = i == 0 ? a : (i == 1 ? b : c);
        const v3 vj = j == 0 ? a : (j == 1 ? b : c);
        const Param4 rt = proj_triangle_origin(vi, vj, d);
        if (mindist < 0 || rt.sqr_distance < mindist) {
          mindist = rt.sqr_distance;
          res.encode = (unsigned)((rt.encode & 1 ? 1 << i : 0) + (rt.encode & 2 ? 1 << j : 0) +
                                  (rt.encode & 4 ? 8 : 0));
          pset(res, i, rt.p0);
          pset(res, j, rt.p1);
          pset(res, j == 2 ? 0 : j + 1, 0);
          res.p3 = rt.p2;
        }
      }
    }
    if (mindist < 0) {
      mindist = 0;
      res.encode = 15;
      res.p0 = triple(c, b, d) / vl;
      res.p1 = triple(a, c, d) / vl;
      res.p2 = triple(b, a, d) / vl;
      res.p3 = 1 - (res.p0 + res.p1 + res.p2);
    }
    res.sqr_distance = mindist;
  } else if (!ng) {
    res = proj_triangle_origin(a, b, c);
    res.p3 = 0;
  }
  return res;
}

// details::getClosestPoints (gjk.cpp:94-151) on a by-value simplex.  Most kernels call it out of line (closest_points);
// one that inlines it keeps the simplex in registers (passed by reference to the call, it goes to local memory).  The
// weights come from w alone; `st` hands each vertex's w0 / w1 to the sums (InRegs, or the passes' SlotStore).
template <class Store = InRegs>
HFB_HD void closest_points_inl(const typename Store::V& v0, const typename Store::V& v1, const typename Store::V& v2,
                               const typename Store::V& v3_, int rank, v3& w0, v3& w1, const Store& st = Store()) {
  if (rank == 1) {
    st.support_points(v0, w0, w1);
    return;
  }
  if (rank == 2) {
    const v3 a = v0.w, b = v1.w;
    const v3 N = b - a;
    double la = dot(N, -a);
    if (la <= 0) {
      st.support_points(v0, w0, w1);
    } else {
      double lb = sqn(N);
      if (la > lb) {
        st.support_points(v1, w0, w1);
      } else {
        lb = la / lb;
        la = 1 - lb;
        v3 a0, a1, b0, b1;
        st.support_points(v0, a0, a1);
        st.support_points(v1, b0, b1);
        w0 = la * a0 + lb * b0;
        w1 = la * a1 + lb * b1;
      }
    }
    return;
  }
  Param4 pr;
  if (rank == 3)
    pr = Store::inline_projections ? proj_triangle_origin_inl<true>(v0.w, v1.w, v2.w) : proj_triangle_origin(v0.w, v1.w, v2.w);
  else pr = proj_tetra_origin(v0.w, v1.w, v2.w, v3_.w);
  // w0 = 0; w0 += p_i * vs[i].w0 ...
  v3 s0, s1;
  st.support_points(v0, s0, s1);
  w0 = mk(0, 0, 0) + pr.p0 * s0;
  w1 = mk(0, 0, 0) + pr.p0 * s1;
  st.support_points(v1, s0, s1);
  w0 = w0 + pr.p1 * s0;
  w1 = w1 + pr.p1 * s1;
  st.support_points(v2, s0, s1);
  w0 = w0 + pr.p2 * s0;
  w1 = w1 + pr.p2 * s1;
  if (rank == 4) {
    st.support_points(v3_, s0, s1);
    w0 = w0 + pr.p3 * s0;
    w1 = w1 + pr.p3 * s1;
  }
}
HFB_HD_NOINLINE void closest_points(const SV& v0, const SV& v1, const SV& v2, const SV& v3_, int rank, v3& w0,
                                   v3& w1) {
  closest_points_inl(v0, v1, v2, v3_, rank, w0, w1);
}

// details::inflate (gjk.cpp:158-173)
HFB_HD void inflate(const MinkD& md, v3 normal, v3& w0, v3& w1) {
  if (md.ssr0 > 0) w0 = w0 + md.ssr0 * normal;
  if (md.ssr1 > 0) w1 = w1 - md.ssr1 * normal;
}

// GJK::getWitnessPointsAndNormal (gjk.cpp:177-186); INL: closest_points inlined (a Store other than InRegs needs it)
template <bool INL = false, class Store = InRegs>
HFB_HD void gjk_witness(const GjkStateT<typename Store::V>& g, const MinkD& md, v3& w0, v3& w1, v3& normal,
                        const Store& st = Store()) {
  if constexpr (INL) closest_points_inl(g.s0, g.s1, g.s2, g.s3, g.rank, w0, w1, st);
  else closest_points(g.s0, g.s1, g.s2, g.s3, g.rank, w0, w1);
  if (nrm(w1 - w0) > HFB_DUMMY_PRECISION) normal = unit(w1 - w0);
  else normal = -unit(g.ray);
  inflate(md, normal, w0, w1);
}

}  // namespace hfb
