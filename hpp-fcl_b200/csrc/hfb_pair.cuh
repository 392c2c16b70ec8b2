// One narrow-phase query (one shape pair): dispatch, solver status machine,
// witness extraction and the distance()/collide() epilogues.
//
// Replaces, per pair:
//   distance()/collide() dispatch          src/distance.cpp:60-109, src/collision.cpp:69-130
//   ShapeShapeDistancer/Collider::run      include/hpp/fcl/internal/shape_shape_func.h:51-82,132-164
//   GJKSolver::shapeDistance (+TriangleP)  include/hpp/fcl/narrowphase/narrowphase.h:308-348
//   GJKSolver::runGJKAndEPA + extractors   narrowphase.h:420-723
//   ShapeShapeDistance<TriangleP,TriangleP> src/distance/triangle_triangle.cpp:47-104
// The query is split in two phases so that the rare, long EPA runs can be
// compacted into their own kernel: phase 1 = closed form or GJK (+ extraction
// when GJK suffices); phase 2 = EPA (+ extraction) for pairs phase 1 flags.
#pragma once
#include "hfb_closed.cuh"
#include "hfb_epa.cuh"

namespace hfb {

struct SolverP {  // GJKSolver::set (narrowphase.h:162-190, 214-244), uniform per batch
  GjkParams gjk;
  EpaParams epa;
  int initial_guess;
  bool compute_penetration;  // enable_signed_distance / (enable_contact || margin < 0)
};

struct PairIn {
  ShapeD s1, s2;
  xf tf1, tf2;
  v3 cached_guess;  // QueryRequest::cached_gjk_guess (default (1,0,0))
  int hint0, hint1; // QueryRequest::cached_support_func_guess
};

struct PairOut {
  double distance;
  v3 p1, p2, normal;
  v3 cached_guess;
  int hint0, hint1;
  unsigned status;      // gjk | epa << 8 | path << 16
  unsigned iterations;  // gjk | epa << 16
};

HFB_HD bool type_known(int t) {
  return t == HFB_GEOM_BOX || t == HFB_GEOM_SPHERE || t == HFB_GEOM_CAPSULE || t == HFB_GEOM_CONE ||
         t == HFB_GEOM_CYLINDER || t == HFB_GEOM_CONVEX || t == HFB_GEOM_TRIANGLE ||
         t == HFB_GEOM_ELLIPSOID || t == HFB_GEOM_PLANE || t == HFB_GEOM_HALFSPACE;
}

// the closed-form specialisation table (shape_shape_func.h:281-306)
HFB_HD bool is_closed_form(int t1, int t2) {
  if (is_plane_type(t1) || is_plane_type(t2)) return true;  // src/distance/*_halfspace.cpp, *_plane.cpp
  if (t1 == HFB_GEOM_SPHERE)
    return t2 == HFB_GEOM_SPHERE || t2 == HFB_GEOM_CAPSULE || t2 == HFB_GEOM_CYLINDER ||
           t2 == HFB_GEOM_BOX || t2 == HFB_GEOM_TRIANGLE;
  if (t2 == HFB_GEOM_SPHERE)
    return t1 == HFB_GEOM_CAPSULE || t1 == HFB_GEOM_CYLINDER || t1 == HFB_GEOM_BOX ||
           t1 == HFB_GEOM_TRIANGLE;
  if (t1 == HFB_GEOM_CAPSULE && t2 == HFB_GEOM_CAPSULE) return true;
  return false;
}

// effective GJK operands after the TriangleP rewrites of shapeDistance
// (narrowphase.h:322-348): triangle always second, pre-transformed into the
// first shape's frame, identity relative transform.
struct GjkSetup {
  ShapeD a, b;
  xf tfa;        // frame the witness points are mapped back with
  MinkD md;
  bool swapped;  // results must be swapped back (p1<->p2, normal negated)
};

template <int CAPS>
HFB_HD void make_setup(const PairIn& in, GjkSetup& S) {
  const bool tri2 = (CAPS & CAP_TRI) && in.s2.type == HFB_GEOM_TRIANGLE;
  const bool tri1 = (CAPS & CAP_TRI) && in.s1.type == HFB_GEOM_TRIANGLE;
  if (tri2 || tri1) {
    const ShapeD& shp = tri2 ? in.s1 : in.s2;
    const ShapeD& tri = tri2 ? in.s2 : in.s1;
    const xf& tfs = tri2 ? in.tf1 : in.tf2;
    const xf& tft = tri2 ? in.tf2 : in.tf1;
    xf rel;  // tf_1M2 = tfs.inverseTimes(tft)  (transform.h:176-178)
    rel.R = mtmulm(tfs.R, tft.R);
    rel.T = mtmul(tfs.R, tft.T - tfs.T);
    S.a = shp;
    S.b = tri;
    S.b.ta = xform(rel, tri.ta);
    S.b.tb = xform(rel, tri.tb);
    S.b.tc = xform(rel, tri.tc);
    S.tfa = tfs;
    S.swapped = tri1 && !tri2;
    mink_set_identity(S.a, S.b, S.md);
  } else {
    S.a = in.s1;
    S.b = in.s2;
    S.tfa = in.tf1;
    S.swapped = false;
    mink_set(S.a, S.b, in.tf1, in.tf2, S.md);
  }
}

HFB_HD v3 initial_guess(const SolverP& P, const PairIn& in, const GjkSetup& S) {  // narrowphase.h:353-391
  if (P.initial_guess == HFB_GUESS_CACHED) return in.cached_guess;
  if (P.initial_guess == HFB_GUESS_BOUNDING_VOLUME)
    return S.a.center - (mmul(S.md.oR1, S.b.center) + S.md.ot1);
  return mk(1, 0, 0);
}

HFB_HD unsigned pack_status(int gjk, int epa, int path) {
  return ((unsigned)gjk & 0xffu) | (((unsigned)epa & 0xffu) << 8) | (((unsigned)path & 0xffu) << 16);
}

// the record of a pair no kernel can compute (the cached guess, hints and iterations are left as they are)
HFB_HD void set_unsupported(PairOut& o) {
  o.distance = DBL_MAX;
  o.p1 = o.p2 = o.normal = nan3();
  o.status = pack_status(0, 0, HFB_PATH_UNSUPPORTED);
}

// world-frame re-centring shared by the GJK and EPA extractors
// (narrowphase.h:632-635, 707-710)
HFB_HD void recentre(const xf& tfa, double distance, v3& p1, v3& p2, v3& normal) {
  const v3 p = xform(tfa, 0.5 * (p1 + p2));
  normal = mmul(tfa.R, normal);
  p1 = p - 0.5 * distance * normal;
  p2 = p + 0.5 * distance * normal;
}

HFB_HD void unswap(const GjkSetup& S, PairOut& o) {  // narrowphase.h:344-346
  if (S.swapped) {
    const v3 t = o.p1;
    o.p1 = o.p2;
    o.p2 = t;
    o.normal = -o.normal;
  }
}

// which code paths a kernel instantiation carries (the batch is binned by pair class first,
// so each kernel only needs its own path: smaller code, no divergence between classes)
enum { PATH_CLOSED = 1, PATH_GJKROUTE = 2, PATH_BOTH = 3 };

// the general GJK route of phase 1 in three pieces (set-up, iterations, extraction), so that the
// primitive-pair kernel can refill lanes between iterations; pair_phase1 chains them for everybody else
template <int CAPS, class V>
HFB_HD void pair_gjk_begin(const PairIn& in, const SolverP& P, GjkSetup& S, GjkLoop& L, GjkStateT<V>& g,
                           PairOut& o) {
  o.cached_guess = (P.initial_guess == HFB_GUESS_CACHED) ? in.cached_guess : mk(1, 0, 0);
  o.hint0 = in.hint0;
  o.hint1 = in.hint1;
  o.iterations = 0;
  make_setup<CAPS>(in, S);
  const v3 guess = initial_guess(P, in, S);
  gjk_begin(S.md, P.gjk, guess, in.hint0, in.hint1, g, L);
}
// returns true when EPA must still run (g holds GJK's final simplex); INL, st: see gjk_witness
template <bool INL = false, class Store = InRegs>
HFB_HD bool pair_gjk_end(const SolverP& P, const GjkSetup& S, GjkStateT<typename Store::V>& g, PairOut& o,
                         const Store& st = Store()) {
  o.iterations = g.iterations & 0xffffu;
  o.status = pack_status(g.status, HFB_EPA_DID_NOT_RUN, HFB_PATH_GJK);
  switch (g.status) {
    case HFB_GJK_FAILED:
    case HFB_GJK_NO_COLLISION:
    case HFB_GJK_COLLISION_WITH_PENETRATION: {  // GJKExtractWitnessPointsAndNormal :610-636
      o.cached_guess = g.ray;
      o.hint0 = g.hint0;
      o.hint1 = g.hint1;
      o.distance = g.distance;
      gjk_witness<INL>(g, S.md, o.p1, o.p2, o.normal, st);
      recentre(S.tfa, o.distance, o.p1, o.p2, o.normal);
      unswap(S, o);
    } break;
    case HFB_GJK_NO_COLLISION_EARLY_STOPPED:  // :589-608
      o.cached_guess = g.ray;
      o.hint0 = g.hint0;
      o.hint1 = g.hint1;
      o.distance = g.distance;
      o.p1 = o.p2 = o.normal = nan3();
      break;
    default:  // HFB_GJK_COLLISION
      if (!P.compute_penetration) {  // :638-656
        o.hint0 = g.hint0;
        o.hint1 = g.hint1;
        o.distance = g.distance;
        o.p1 = o.p2 = o.normal = nan3();
      } else {
        return true;
      }
  }
  return false;
}

// ---- phase 1 -----------------------------------------------------------------
// returns true when EPA must still run (g holds GJK's final simplex).
template <int G, int CAPS, int PATHS = PATH_BOTH>
HFB_HD bool pair_phase1(const PairIn& in, const SolverP& P, PairOut& o, GjkState& g) {
  const int t1 = in.s1.type, t2 = in.s2.type;
  o.cached_guess = (P.initial_guess == HFB_GUESS_CACHED) ? in.cached_guess : mk(1, 0, 0);
  o.hint0 = in.hint0;
  o.hint1 = in.hint1;
  o.iterations = 0;
  if (!type_known(t1) || !type_known(t2)) {
    set_unsupported(o);
    return false;
  }
  if (is_plane_type(t1) || is_plane_type(t2)) {
    // only the kernels the plane classes are binned to carry this code (CAP_PLANE); elsewhere such a pair cannot
    // arrive (k_bin_*; the mesh walks refuse plane partners in bvh_make_query)
    if ((CAPS & CAP_PLANE) && (PATHS & PATH_CLOSED)) {
      const Wit w = plane_family<G, CAPS>(in.s1, in.tf1, in.s2, in.tf2);
      o.distance = w.d;
      o.p1 = w.p1;
      o.p2 = w.p2;
      o.normal = w.n;
      o.status = pack_status(HFB_GJK_DID_NOT_RUN, HFB_EPA_DID_NOT_RUN, HFB_PATH_CLOSED_FORM);
    } else {
      set_unsupported(o);
    }
    return false;
  }
  if ((PATHS & PATH_CLOSED) && (CAPS & CAP_PRIM) && is_closed_form(t1, t2)) {
    Wit w;
    if (t1 == HFB_GEOM_SPHERE && t2 == HFB_GEOM_SPHERE) w = sphere_sphere(in.s1, in.tf1, in.s2, in.tf2);
    else if (t1 == HFB_GEOM_SPHERE && t2 == HFB_GEOM_CAPSULE) w = sphere_capsule(in.s1, in.tf1, in.s2, in.tf2);
    else if (t1 == HFB_GEOM_CAPSULE && t2 == HFB_GEOM_SPHERE) w = flip(sphere_capsule(in.s2, in.tf2, in.s1, in.tf1));
    else if (t1 == HFB_GEOM_SPHERE && t2 == HFB_GEOM_CYLINDER) w = sphere_cylinder(in.s1, in.tf1, in.s2, in.tf2);
    else if (t1 == HFB_GEOM_CYLINDER && t2 == HFB_GEOM_SPHERE) w = flip(sphere_cylinder(in.s2, in.tf2, in.s1, in.tf1));
    else if (t1 == HFB_GEOM_BOX && t2 == HFB_GEOM_SPHERE) w = box_sphere(in.s1, in.tf1, in.s2, in.tf2);
    else if (t1 == HFB_GEOM_SPHERE && t2 == HFB_GEOM_BOX) w = flip(box_sphere(in.s2, in.tf2, in.s1, in.tf1));
    else if ((CAPS & CAP_TRI) && t1 == HFB_GEOM_SPHERE && t2 == HFB_GEOM_TRIANGLE)
      w = sphere_triangle(in.s1, in.tf1, in.s2, in.tf2);
    else if ((CAPS & CAP_TRI) && t1 == HFB_GEOM_TRIANGLE && t2 == HFB_GEOM_SPHERE)
      w = flip(sphere_triangle(in.s2, in.tf2, in.s1, in.tf1));
    else w = capsule_capsule(in.s1, in.tf1, in.s2, in.tf2);
    o.distance = w.d;
    o.p1 = w.p1;
    o.p2 = w.p2;
    o.normal = w.n;
    o.status = pack_status(HFB_GJK_DID_NOT_RUN, HFB_EPA_DID_NOT_RUN, HFB_PATH_CLOSED_FORM);
    return false;
  }

  if (!(PATHS & PATH_GJKROUTE)) {  // mis-binned pair: cannot happen (k_bin_* and is_closed_form agree)
    set_unsupported(o);
    return false;
  }
  if ((CAPS & CAP_TRI) && t1 == HFB_GEOM_TRIANGLE && t2 == HFB_GEOM_TRIANGLE) {
    // triangle_triangle.cpp:47-104: world-frame triangles, GJK only
    ShapeD a = in.s1, b = in.s2;
    a.ta = xform(in.tf1, in.s1.ta);
    a.tb = xform(in.tf1, in.s1.tb);
    a.tc = xform(in.tf1, in.s1.tc);
    b.ta = xform(in.tf2, in.s2.ta);
    b.tb = xform(in.tf2, in.s2.tb);
    b.tc = xform(in.tf2, in.s2.tc);
    MinkD md;
    mink_set_identity(a, b, md);
    v3 guess;
    if (P.initial_guess == HFB_GUESS_CACHED) guess = in.cached_guess;
    else guess = (a.ta + a.tb + a.tc - b.ta - b.tb - b.tc) / 3;
    // this specialisation only calls gjk.reset(max_iterations, tolerance): variant, convergence
    // criterion and early-stop bound are those of a freshly constructed GJK (gjk.cpp:51-57), not the
    // request's (runGJKAndEPA, which copies them, is never reached)
    GjkParams pg = P.gjk;
    pg.distance_upper_bound = DBL_MAX;
    pg.variant = HFB_GJK_DEFAULT;
    pg.criterion = HFB_CRIT_DEFAULT;
    pg.criterion_type = HFB_CRIT_RELATIVE;
    gjk_evaluate<G, CAPS>(a, b, md, pg, guess, 0, 0, g);
    o.cached_guess = g.ray;
    o.hint0 = g.hint0;
    o.hint1 = g.hint1;
    gjk_witness(g, md, o.p1, o.p2, o.normal);
    o.distance = g.distance;
    if (g.status == HFB_GJK_COLLISION) {  // details::computePenetration (details.h:699-711)
      const v3 u = cross(a.tb - a.ta, a.tc - a.ta);
      o.normal = unit(u);
      const double d1 = dot(a.ta - b.ta, o.normal);
      const double d2 = dot(a.ta - b.tb, o.normal);
      const double d3 = dot(a.ta - b.tc, o.normal);
      o.distance = -fmax(d1, fmax(d2, d3));
    }
    o.status = pack_status(g.status, HFB_EPA_DID_NOT_RUN, HFB_PATH_CLOSED_FORM);
    o.iterations = 0;
    return false;
  }

  GjkSetup S;
  GjkLoop L;
  pair_gjk_begin<CAPS>(in, P, S, L, g, o);
  while (gjk_step<G, CAPS>(S.a, S.b, S.md, P.gjk, g, L)) {
  }
  return pair_gjk_end(P, S, g, o);
}

// ---- phase 2: EPA + EPAExtractWitnessPointsAndNormal (narrowphase.h:514-583, 658-723)
// what a run that outgrew a reduced-size workspace hands to its continuation in the full-size one
struct EpaResume {
  EpaState E;
  EpaLoop L;
};
// the result record of a finished EPA run (r) whose workspace is `ws` and side `sd`.  Of S it reads the radii, tfa and
// swapped.
template <class WS, class Side>
HFB_HD void pair_epa_result(const GjkSetup& S, unsigned gjk_iterations, const EpaResume& r, const WS* ws,
                            const Side& sd, PairOut& o) {
  o.iterations = (gjk_iterations & 0xffffu) | ((r.L.it & 0xffffu) << 16);
  o.status = pack_status(HFB_GJK_COLLISION, r.E.status, HFB_PATH_GJK);
  if (r.E.status == HFB_EPA_FALLBACK) {  // EPAFailedExtract... :713-723
    o.cached_guess = mk(1, 0, 0);
    o.hint0 = o.hint1 = 0;
    o.distance = -DBL_MAX;
    o.p1 = o.p2 = o.normal = nan3();
    return;
  }
  const double depth = epa_depth(S.md, r.L);
  o.cached_guess = -(depth * r.L.outer_n);
  o.hint0 = r.E.hint0;
  o.hint1 = r.E.hint1;
  o.distance = fmin(0., -depth);
  epa_witness(ws, sd, r.L, depth, S.md, o.p1, o.p2, o.normal);
  recentre(S.tfa, o.distance, o.p1, o.p2, o.normal);
  unswap(S, o);
}
// EPA from GJK's final simplex `g`, up to the result record.  Returns false only when WS is a reduced-size workspace
// and the polytope outgrew it; with r.L.resumable set, (r, *ws, sd) is then the state at the top of the iteration that
// did not fit, which pair_epa_resume continues from a copy of (epa_ws_grow); otherwise the pair is run again, from the
// queued GJK state, in the full-size workspace.
template <int G, int CAPS, class WS, class Side>
HFB_HD bool pair_epa(const GjkSetup& S, const SolverP& P, GjkState& g, WS* ws, const Side& sd, EpaResume& r) {
  epa_evaluate<G, CAPS>(S.a, S.b, S.md, P.epa, g, ws, sd, r.E, r.L);
  return r.E.status != HFB_EPA_WS_OVERFLOW;
}
// the rest of a run that stopped with r.L.resumable set; `ws` and `sd` hold the grown copy of its workspace and side
template <int G, int CAPS, class WS, class Side>
HFB_HD bool pair_epa_resume(const GjkSetup& S, const SolverP& P, WS* ws, const Side& sd, EpaResume& r) {
  epa_run<G, CAPS>(S.a, S.b, S.md, P.epa, ws, sd, r.E, r.L);
  if (r.E.status == HFB_EPA_WS_OVERFLOW && r.L.resumable) return false;  // (cannot happen in the full-size workspace)
  epa_finish(P.epa, r.E, r.L);
  return r.E.status != HFB_EPA_WS_OVERFLOW;
}
// pair_epa + the result record.  Returns false (and leaves `o` unset) only when WS is a reduced-size workspace and the
// polytope outgrew it; `rs`, if given, then receives the state to resume from (see pair_epa).
template <int G, int CAPS, class WS, class Side>
HFB_HD bool pair_phase2(const PairIn& in, const SolverP& P, GjkState& g, WS* ws, const Side& sd, PairOut& o,
                        EpaResume* rs = nullptr) {
  GjkSetup S;
  make_setup<CAPS>(in, S);
  EpaResume r;
  if (!pair_epa<G, CAPS>(S, P, g, ws, sd, r)) {
    if (rs) *rs = r;
    return false;
  }
  pair_epa_result(S, g.iterations, r, ws, sd, o);
  return true;
}
// the same in a workspace that keeps the support points itself (EpaWsT)
template <int G, int CAPS, int V, int F>
HFB_HD bool pair_phase2(const PairIn& in, const SolverP& P, GjkState& g, EpaWsT<V, F>* ws, PairOut& o,
                        EpaResume* rs = nullptr) {
  return pair_phase2<G, CAPS>(in, P, g, ws, EpaSideWs<EpaWsT<V, F>>{ws}, o, rs);
}
// pair_epa_resume + the result record; `g` holds the GJK iteration count of the pair (all the record takes from it)
template <int G, int CAPS, class WS, class Side>
HFB_HD bool pair_phase2_resume(const PairIn& in, const SolverP& P, const GjkState& g, WS* ws, const Side& sd,
                               EpaResume& rs, PairOut& o) {
  GjkSetup S;
  make_setup<CAPS>(in, S);
  if (!pair_epa_resume<G, CAPS>(S, P, ws, sd, rs)) return false;
  pair_epa_result(S, g.iterations, rs, ws, sd, o);
  return true;
}
// the same in a workspace that keeps the support points itself (EpaWsT)
template <int G, int CAPS, int V, int F>
HFB_HD bool pair_phase2_resume(const PairIn& in, const SolverP& P, const GjkState& g, EpaWsT<V, F>* ws, EpaResume& rs,
                               PairOut& o) {
  return pair_phase2_resume<G, CAPS>(in, P, g, ws, EpaSideWs<EpaWsT<V, F>>{ws}, rs, o);
}

// ---- epilogues -----------------------------------------------------------------
// distance(): fresh DistanceResult + result.update (collision_data.h:1111-1124)
HFB_HD void write_distance(const PairOut& o, hfb_distance_result* r) {
  const bool unsupported = ((o.status >> 16) & 0xff) == HFB_PATH_UNSUPPORTED;
  const bool closed = ((o.status >> 16) & 0xff) == HFB_PATH_CLOSED_FORM;
  const bool take = !unsupported && (closed || DBL_MAX > o.distance);
  const v3 q = nan3();
  const v3 p1 = take ? o.p1 : q, p2 = take ? o.p2 : q, n = take ? o.normal : q;
  r->min_distance = take ? o.distance : DBL_MAX;
  r->p1[0] = p1.x; r->p1[1] = p1.y; r->p1[2] = p1.z;
  r->p2[0] = p2.x; r->p2[1] = p2.y; r->p2[2] = p2.z;
  r->normal[0] = n.x; r->normal[1] = n.y; r->normal[2] = n.z;
  r->b1 = -1;
  r->b2 = -1;
  r->status = o.status;
  r->iterations = o.iterations;
}

struct CollideP {  // CollisionRequest fields used by ShapeShapeCollider::run
  double security_margin;
  double collision_distance_threshold;
};

// collide(): ShapeShapeCollider::run (shape_shape_func.h:134-163) on a fresh CollisionResult
HFB_HD void write_contact(const PairOut& o, const CollideP& C, hfb_contact* r) {
  const bool unsupported = ((o.status >> 16) & 0xff) == HFB_PATH_UNSUPPORTED;
  const v3 q = nan3();
  v3 p1 = q, p2 = q, n = q, pos = q;
  double lb = DBL_MAX, dist = DBL_MAX;
  unsigned nc = 0;
  if (!unsupported) {
    dist = o.distance;
    const double d2c = o.distance - C.security_margin;
    if (d2c < lb) {  // updateDistanceLowerBoundFromLeaf (collision_data.h:1186-1197)
      lb = d2c;
      p1 = o.p1;
      p2 = o.p2;
      n = o.normal;
    }
    if (d2c <= C.collision_distance_threshold) {
      pos = (o.p1 + o.p2) / 2;  // Contact ctor (collision_data.h:138-148)
      nc = 1;
    }
  }
  r->distance = dist;
  r->p1[0] = p1.x; r->p1[1] = p1.y; r->p1[2] = p1.z;
  r->p2[0] = p2.x; r->p2[1] = p2.y; r->p2[2] = p2.z;
  r->normal[0] = n.x; r->normal[1] = n.y; r->normal[2] = n.z;
  r->pos[0] = pos.x; r->pos[1] = pos.y; r->pos[2] = pos.z;
  r->distance_lower_bound = lb;
  r->b1 = -1;
  r->b2 = -1;
  r->status = o.status;
  r->num_contacts = nc;
  r->iterations = o.iterations;
  r->_pad = 0;
}

}  // namespace hfb
