// OBBRSS BVH vs shape: bounding-volume tests, the per-query shape BV and the
// depth-first traversals, for one (mesh, shape) query.
//
// Replaces
//   RSS distance / rectDistance / segCoords / inVoronoi     src/BV/RSS.cpp:67-713, 995-1005
//   OBB SAT with squared lower bound                        src/BV/OBB.cpp:290-393, 475-483
//   computeBV<OBBRSS,S> = fit(getBoundVertices(S, tf))      include/hpp/fcl/shape/geometric_shapes_utility.h:73-83,
//       src/shape/geometric_shapes_utility.cpp:47-262, src/BVH/BV_fitter.cpp:49-216,
//       src/BVH/BVH_utility.cpp:183-600, include/hpp/fcl/internal/tools.h:60-203
//   distanceRecurse / collisionRecurse                      src/traversal/traversal_recurse.cpp:44-85, 153-203
//   MeshShape{Distance,Collision}TraversalNodeOBBRSS        include/hpp/fcl/internal/traversal_node_bvh_shape.h:97-194, 286-478
//
// Design: the reference recurses; here each query walks the tree with an explicit
// per-thread stack in the same order (nearer child first for distance, left child
// first for collision) so pruning, witness triangle and lower bounds come out the
// same.  Nodes are the 256-byte hfb_bvh_node records the host copies out of
// BVHModel<OBBRSS>::bvs.
#pragma once
#include "hfb_arena.cuh"
#include "hfb_pair.cuh"

namespace hfb {

struct RssD {
  m3 axes;  // columns are the axes; held as rows of the 3x3 (element (r,c))
  v3 Tr;
  double l0, l1, radius;
};
struct ObbD {
  m3 axes;
  v3 To, extent;
};

// column-major 9 doubles -> m3 rows
HFB_HD m3 load_colmajor(const double* p) {
  m3 A;
  A.r0 = mk(p[0], p[3], p[6]);
  A.r1 = mk(p[1], p[4], p[7]);
  A.r2 = mk(p[2], p[5], p[8]);
  return A;
}
HFB_HD m3 mmulm(const m3& A, const m3& B) {  // A * B, each element left to right over k
  m3 C;
  const v3 b0 = mcol(B, 0), b1 = mcol(B, 1), b2 = mcol(B, 2);
  C.r0 = mk(dot(A.r0, b0), dot(A.r0, b1), dot(A.r0, b2));
  C.r1 = mk(dot(A.r1, b0), dot(A.r1, b1), dot(A.r1, b2));
  C.r2 = mk(dot(A.r2, b0), dot(A.r2, b1), dot(A.r2, b2));
  return C;
}
HFB_HD m3 mtrans(const m3& A) {
  m3 T;
  T.r0 = mcol(A, 0);
  T.r1 = mcol(A, 1);
  T.r2 = mcol(A, 2);
  return T;
}
HFB_HD double mel(const m3& A, int r, int c) { return comp(r == 0 ? A.r0 : (r == 1 ? A.r1 : A.r2), c); }

// -------------------------------------------------------------------- RSS -------
HFB_HD void clip_range(double& val, double a, double b) {
  if (val < a) val = a;
  else if (val > b) val = b;
}
HFB_HD void seg_coords(double& t, double& u, double a, double b, double A_dot_B, double A_dot_T, double B_dot_T) {
  const double denom = 1 - A_dot_B * A_dot_B;
  if (denom == 0) t = 0;
  else {
    t = (A_dot_T - B_dot_T * A_dot_B) / denom;
    clip_range(t, 0, a);
  }
  u = t * A_dot_B - B_dot_T;
  if (u < 0) {
    u = 0;
    t = A_dot_T;
    clip_range(t, 0, a);
  } else if (u > b) {
    u = b;
    t = u * A_dot_B + A_dot_T;
    clip_range(t, 0, a);
  }
}
HFB_HD bool in_voronoi(double a, double b, double Anorm_dot_B, double Anorm_dot_T, double A_dot_B, double A_dot_T,
                       double B_dot_T) {
  if (fabs(Anorm_dot_B) < 1e-7) return false;
  double t, u, v;
  u = -Anorm_dot_T / Anorm_dot_B;
  clip_range(u, 0, b);
  t = u * A_dot_B + A_dot_T;
  clip_range(t, 0, a);
  v = t * A_dot_B - B_dot_T;
  if (Anorm_dot_B > 0) {
    if (v > (u + 1e-7)) return true;
  } else {
    if (v < (u - 1e-7)) return true;
  }
  return false;
}

// lanes that run a bounding-volume test together (a ballot of the warp-scheduled walk); 0 = alone
#if defined(__CUDA_ARCH__)
#define HFB_LANES_SYNC(m) do { if (m) __syncwarp(m); } while (0)
#define HFB_LANES_ALL(m, p) ((m) ? (__all_sync((m), (p)) != 0) : (p))
#else
#define HFB_LANES_SYNC(m) do { (void)(m); } while (0)
#define HFB_LANES_ALL(m, p) (p)
#endif

// rectDistance (RSS.cpp:121-713), closest points not requested.  The sixteen edge-pair cases
// keep the reference's expressions term for term (the association order differs between cases).
// Three pieces, so that the lanes of a group can share one rectangle pair (hfb_bvhq.cuh): the values
// every case reads (rect_prelude), the conditions of one case (rect_case: the reference returns from
// the first case whose conditions hold), and the distance of the winning case or, when no edge pair
// holds the closest points, of the face-normal separation (rect_finish).  rect_distance chains them.
struct RectPre {
  double R00, R01, R02, R10, R11, R12, R20, R21, a0, a1, b0, b1;
  double A0_dot_B0, A0_dot_B1, A1_dot_B0, A1_dot_B1, aA0_dot_B0, aA0_dot_B1, aA1_dot_B0, aA1_dot_B1, bA0_dot_B0, bA1_dot_B0, bA0_dot_B1, bA1_dot_B1;
  double Tab0, Tab1, Tab2, Tba0, Tba1, Tba2;
  double LA1_lx, LA1_ux, UA1_lx, UA1_ux, LB1_lx, LB1_ux, UB1_lx, UB1_ux;
  double LA1_ly, LA1_uy, UA1_ly, UA1_uy, LB0_lx, LB0_ux, UB0_lx, UB0_ux;
  double LA0_lx, LA0_ux, UA0_lx, UA0_ux, LB1_ly, LB1_uy, UB1_ly, UB1_uy;
  double LA0_ly, LA0_uy, UA0_ly, UA0_uy, LB0_ly, LB0_uy, UB0_ly, UB0_uy;
};
HFB_HD void rect_prelude(const m3& Rab, v3 Tab, double a0, double a1, double b0, double b1, RectPre& p) {
  const double R00 = Rab.r0.x, R01 = Rab.r0.y, R02 = Rab.r0.z;
  const double R10 = Rab.r1.x, R11 = Rab.r1.y, R12 = Rab.r1.z;
  const double R20 = Rab.r2.x, R21 = Rab.r2.y;
  const double A0_dot_B0 = R00, A0_dot_B1 = R01, A1_dot_B0 = R10, A1_dot_B1 = R11;
  const double aA0_dot_B0 = a0 * A0_dot_B0, aA0_dot_B1 = a0 * A0_dot_B1, aA1_dot_B0 = a1 * A1_dot_B0,
               aA1_dot_B1 = a1 * A1_dot_B1;
  const double bA0_dot_B0 = b0 * A0_dot_B0, bA1_dot_B0 = b0 * A1_dot_B0, bA0_dot_B1 = b1 * A0_dot_B1,
               bA1_dot_B1 = b1 * A1_dot_B1;
  const v3 Tba = mtmul(Rab, Tab);
  const double Tab0 = Tab.x, Tab1 = Tab.y, Tab2 = Tab.z, Tba0 = Tba.x, Tba1 = Tba.y, Tba2 = Tba.z;

  double LA1_lx, LA1_ux, UA1_lx, UA1_ux, LB1_lx, LB1_ux, UB1_lx, UB1_ux;
  const double ALL_x = -Tba0;
  const double ALU_x = ALL_x + aA1_dot_B0;
  const double AUL_x = ALL_x + aA0_dot_B0;
  const double AUU_x = ALU_x + aA0_dot_B0;
  if (ALL_x < ALU_x) { LA1_lx = ALL_x; LA1_ux = ALU_x; UA1_lx = AUL_x; UA1_ux = AUU_x; }
  else { LA1_lx = ALU_x; LA1_ux = ALL_x; UA1_lx = AUU_x; UA1_ux = AUL_x; }
  const double BLL_x = Tab0;
  const double BLU_x = BLL_x + bA0_dot_B1;
  const double BUL_x = BLL_x + bA0_dot_B0;
  const double BUU_x = BLU_x + bA0_dot_B0;
  if (BLL_x < BLU_x) { LB1_lx = BLL_x; LB1_ux = BLU_x; UB1_lx = BUL_x; UB1_ux = BUU_x; }
  else { LB1_lx = BLU_x; LB1_ux = BLL_x; UB1_lx = BUU_x; UB1_ux = BUL_x; }


  double LA1_ly, LA1_uy, UA1_ly, UA1_uy, LB0_lx, LB0_ux, UB0_lx, UB0_ux;
  const double ALL_y = -Tba1;
  const double ALU_y = ALL_y + aA1_dot_B1;
  const double AUL_y = ALL_y + aA0_dot_B1;
  const double AUU_y = ALU_y + aA0_dot_B1;
  if (ALL_y < ALU_y) { LA1_ly = ALL_y; LA1_uy = ALU_y; UA1_ly = AUL_y; UA1_uy = AUU_y; }
  else { LA1_ly = ALU_y; LA1_uy = ALL_y; UA1_ly = AUU_y; UA1_uy = AUL_y; }
  if (BLL_x < BUL_x) { LB0_lx = BLL_x; LB0_ux = BUL_x; UB0_lx = BLU_x; UB0_ux = BUU_x; }
  else { LB0_lx = BUL_x; LB0_ux = BLL_x; UB0_lx = BUU_x; UB0_ux = BLU_x; }


  double LA0_lx, LA0_ux, UA0_lx, UA0_ux, LB1_ly, LB1_uy, UB1_ly, UB1_uy;
  const double BLL_y = Tab1;
  const double BLU_y = BLL_y + bA1_dot_B1;
  const double BUL_y = BLL_y + bA1_dot_B0;
  const double BUU_y = BLU_y + bA1_dot_B0;
  if (ALL_x < AUL_x) { LA0_lx = ALL_x; LA0_ux = AUL_x; UA0_lx = ALU_x; UA0_ux = AUU_x; }
  else { LA0_lx = AUL_x; LA0_ux = ALL_x; UA0_lx = AUU_x; UA0_ux = ALU_x; }
  if (BLL_y < BLU_y) { LB1_ly = BLL_y; LB1_uy = BLU_y; UB1_ly = BUL_y; UB1_uy = BUU_y; }
  else { LB1_ly = BLU_y; LB1_uy = BLL_y; UB1_ly = BUU_y; UB1_uy = BUL_y; }


  double LA0_ly, LA0_uy, UA0_ly, UA0_uy, LB0_ly, LB0_uy, UB0_ly, UB0_uy;
  if (ALL_y < AUL_y) { LA0_ly = ALL_y; LA0_uy = AUL_y; UA0_ly = ALU_y; UA0_uy = AUU_y; }
  else { LA0_ly = AUL_y; LA0_uy = ALL_y; UA0_ly = AUU_y; UA0_uy = ALU_y; }
  if (BLL_y < BUL_y) { LB0_ly = BLL_y; LB0_uy = BUL_y; UB0_ly = BLU_y; UB0_uy = BUU_y; }
  else { LB0_ly = BUL_y; LB0_uy = BLL_y; UB0_ly = BUU_y; UB0_uy = BLU_y; }


  p.R00 = R00;
  p.R01 = R01;
  p.R02 = R02;
  p.R10 = R10;
  p.R11 = R11;
  p.R12 = R12;
  p.R20 = R20;
  p.R21 = R21;
  p.a0 = a0;
  p.a1 = a1;
  p.b0 = b0;
  p.b1 = b1;
  p.A0_dot_B0 = A0_dot_B0;
  p.A0_dot_B1 = A0_dot_B1;
  p.A1_dot_B0 = A1_dot_B0;
  p.A1_dot_B1 = A1_dot_B1;
  p.aA0_dot_B0 = aA0_dot_B0;
  p.aA0_dot_B1 = aA0_dot_B1;
  p.aA1_dot_B0 = aA1_dot_B0;
  p.aA1_dot_B1 = aA1_dot_B1;
  p.bA0_dot_B0 = bA0_dot_B0;
  p.bA1_dot_B0 = bA1_dot_B0;
  p.bA0_dot_B1 = bA0_dot_B1;
  p.bA1_dot_B1 = bA1_dot_B1;
  p.Tab0 = Tab0;
  p.Tab1 = Tab1;
  p.Tab2 = Tab2;
  p.Tba0 = Tba0;
  p.Tba1 = Tba1;
  p.Tba2 = Tba2;
  p.LA1_lx = LA1_lx;
  p.LA1_ux = LA1_ux;
  p.UA1_lx = UA1_lx;
  p.UA1_ux = UA1_ux;
  p.LB1_lx = LB1_lx;
  p.LB1_ux = LB1_ux;
  p.UB1_lx = UB1_lx;
  p.UB1_ux = UB1_ux;
  p.LA1_ly = LA1_ly;
  p.LA1_uy = LA1_uy;
  p.UA1_ly = UA1_ly;
  p.UA1_uy = UA1_uy;
  p.LB0_lx = LB0_lx;
  p.LB0_ux = LB0_ux;
  p.UB0_lx = UB0_lx;
  p.UB0_ux = UB0_ux;
  p.LA0_lx = LA0_lx;
  p.LA0_ux = LA0_ux;
  p.UA0_lx = UA0_lx;
  p.UA0_ux = UA0_ux;
  p.LB1_ly = LB1_ly;
  p.LB1_uy = LB1_uy;
  p.UB1_ly = UB1_ly;
  p.UB1_uy = UB1_uy;
  p.LA0_ly = LA0_ly;
  p.LA0_uy = LA0_uy;
  p.UA0_ly = UA0_ly;
  p.UA0_uy = UA0_uy;
  p.LB0_ly = LB0_ly;
  p.LB0_uy = LB0_uy;
  p.UB0_ly = UB0_ly;
  p.UB0_uy = UB0_uy;
}
// conditions of edge-pair case k (0..15, the reference's order)
HFB_HD bool rect_case(const RectPre& p, int k) {
  const double R00 = p.R00;
  const double R01 = p.R01;
  const double R02 = p.R02;
  const double R10 = p.R10;
  const double R11 = p.R11;
  const double R12 = p.R12;
  const double R20 = p.R20;
  const double R21 = p.R21;
  const double a0 = p.a0;
  const double a1 = p.a1;
  const double b0 = p.b0;
  const double b1 = p.b1;
  const double A0_dot_B0 = p.A0_dot_B0;
  const double A0_dot_B1 = p.A0_dot_B1;
  const double A1_dot_B0 = p.A1_dot_B0;
  const double A1_dot_B1 = p.A1_dot_B1;
  const double aA0_dot_B0 = p.aA0_dot_B0;
  const double aA0_dot_B1 = p.aA0_dot_B1;
  const double aA1_dot_B0 = p.aA1_dot_B0;
  const double aA1_dot_B1 = p.aA1_dot_B1;
  const double bA0_dot_B0 = p.bA0_dot_B0;
  const double bA1_dot_B0 = p.bA1_dot_B0;
  const double bA0_dot_B1 = p.bA0_dot_B1;
  const double bA1_dot_B1 = p.bA1_dot_B1;
  const double Tab0 = p.Tab0;
  const double Tab1 = p.Tab1;
  const double Tab2 = p.Tab2;
  const double Tba0 = p.Tba0;
  const double Tba1 = p.Tba1;
  const double Tba2 = p.Tba2;
  const double LA1_lx = p.LA1_lx;
  const double LA1_ux = p.LA1_ux;
  const double UA1_lx = p.UA1_lx;
  const double UA1_ux = p.UA1_ux;
  const double LB1_lx = p.LB1_lx;
  const double LB1_ux = p.LB1_ux;
  const double UB1_lx = p.UB1_lx;
  const double UB1_ux = p.UB1_ux;
  const double LA1_ly = p.LA1_ly;
  const double LA1_uy = p.LA1_uy;
  const double UA1_ly = p.UA1_ly;
  const double UA1_uy = p.UA1_uy;
  const double LB0_lx = p.LB0_lx;
  const double LB0_ux = p.LB0_ux;
  const double UB0_lx = p.UB0_lx;
  const double UB0_ux = p.UB0_ux;
  const double LA0_lx = p.LA0_lx;
  const double LA0_ux = p.LA0_ux;
  const double UA0_lx = p.UA0_lx;
  const double UA0_ux = p.UA0_ux;
  const double LB1_ly = p.LB1_ly;
  const double LB1_uy = p.LB1_uy;
  const double UB1_ly = p.UB1_ly;
  const double UB1_uy = p.UB1_uy;
  const double LA0_ly = p.LA0_ly;
  const double LA0_uy = p.LA0_uy;
  const double UA0_ly = p.UA0_ly;
  const double UA0_uy = p.UA0_uy;
  const double LB0_ly = p.LB0_ly;
  const double LB0_uy = p.LB0_uy;
  const double UB0_ly = p.UB0_ly;
  const double UB0_uy = p.UB0_uy;
  (void)R00; (void)R01; (void)R02; (void)R10; (void)R11; (void)R12; (void)R20; (void)R21; (void)Tab2; (void)Tba2;
  bool guard = false, ca = false, cb = false;
  double va0 = 0, va1 = 0, va2 = 0, va3 = 0, va4 = 0, va5 = 0, va6 = 0;
  double vb0 = 0, vb1 = 0, vb2 = 0, vb3 = 0, vb4 = 0, vb5 = 0, vb6 = 0;
  switch (k) {
  case 0:  // UA1, UB1
    guard = (UA1_ux > b0) && (UB1_ux > a0);
    ca = UA1_lx > b0;
    va0 = b1; va1 = a1; va2 = A1_dot_B0; va3 = aA0_dot_B0 - b0 - Tba0; va4 = A1_dot_B1; va5 = aA0_dot_B1 - Tba1; va6 = -Tab1 - bA1_dot_B0;
    cb = UB1_lx > a0;
    vb0 = a1; vb1 = b1; vb2 = A0_dot_B1; vb3 = Tab0 + bA0_dot_B0 - a0; vb4 = A1_dot_B1; vb5 = Tab1 + bA1_dot_B0; vb6 = Tba1 - aA0_dot_B1;
    break;
  case 1:  // UA1, LB1
    guard = (UA1_lx < 0) && (LB1_ux > a0);
    ca = UA1_ux < 0;
    va0 = b1; va1 = a1; va2 = -A1_dot_B0; va3 = Tba0 - aA0_dot_B0; va4 = A1_dot_B1; va5 = aA0_dot_B1 - Tba1; va6 = -Tab1;
    cb = LB1_lx > a0;
    vb0 = a1; vb1 = b1; vb2 = A0_dot_B1; vb3 = Tab0 - a0; vb4 = A1_dot_B1; vb5 = Tab1; vb6 = Tba1 - aA0_dot_B1;
    break;
  case 2:  // LA1, UB1
    guard = (LA1_ux > b0) && (UB1_lx < 0);
    ca = LA1_lx > b0;
    va0 = b1; va1 = a1; va2 = A1_dot_B0; va3 = -Tba0 - b0; va4 = A1_dot_B1; va5 = -Tba1; va6 = -Tab1 - bA1_dot_B0;
    cb = UB1_ux < 0;
    vb0 = a1; vb1 = b1; vb2 = -A0_dot_B1; vb3 = -Tab0 - bA0_dot_B0; vb4 = A1_dot_B1; vb5 = Tab1 + bA1_dot_B0; vb6 = Tba1;
    break;
  case 3:  // LA1, LB1
    guard = (LA1_lx < 0) && (LB1_lx < 0);
    ca = LA1_ux < 0;
    va0 = b1; va1 = a1; va2 = -A1_dot_B0; va3 = Tba0; va4 = A1_dot_B1; va5 = -Tba1; va6 = -Tab1;
    cb = LB1_ux < 0;
    vb0 = a1; vb1 = b1; vb2 = -A0_dot_B1; vb3 = -Tab0; vb4 = A1_dot_B1; vb5 = Tab1; vb6 = Tba1;
    break;
  case 4:  // UA1, UB0
    guard = (UA1_uy > b1) && (UB0_ux > a0);
    ca = UA1_ly > b1;
    va0 = b0; va1 = a1; va2 = A1_dot_B1; va3 = aA0_dot_B1 - Tba1 - b1; va4 = A1_dot_B0; va5 = aA0_dot_B0 - Tba0; va6 = -Tab1 - bA1_dot_B1;
    cb = UB0_lx > a0;
    vb0 = a1; vb1 = b0; vb2 = A0_dot_B0; vb3 = Tab0 - a0 + bA0_dot_B1; vb4 = A1_dot_B0; vb5 = Tab1 + bA1_dot_B1; vb6 = Tba0 - aA0_dot_B0;
    break;
  case 5:  // UA1, LB0
    guard = (UA1_ly < 0) && (LB0_ux > a0);
    ca = UA1_uy < 0;
    va0 = b0; va1 = a1; va2 = -A1_dot_B1; va3 = Tba1 - aA0_dot_B1; va4 = A1_dot_B0; va5 = aA0_dot_B0 - Tba0; va6 = -Tab1;
    cb = LB0_lx > a0;
    vb0 = a1; vb1 = b0; vb2 = A0_dot_B0; vb3 = Tab0 - a0; vb4 = A1_dot_B0; vb5 = Tab1; vb6 = Tba0 - aA0_dot_B0;
    break;
  case 6:  // LA1, UB0
    guard = (LA1_uy > b1) && (UB0_lx < 0);
    ca = LA1_ly > b1;
    va0 = b0; va1 = a1; va2 = A1_dot_B1; va3 = -Tba1 - b1; va4 = A1_dot_B0; va5 = -Tba0; va6 = -Tab1 - bA1_dot_B1;
    cb = UB0_ux < 0;
    vb0 = a1; vb1 = b0; vb2 = -A0_dot_B0; vb3 = -Tab0 - bA0_dot_B1; vb4 = A1_dot_B0; vb5 = Tab1 + bA1_dot_B1; vb6 = Tba0;
    break;
  case 7:  // LA1, LB0
    guard = (LA1_ly < 0) && (LB0_lx < 0);
    ca = LA1_uy < 0;
    va0 = b0; va1 = a1; va2 = -A1_dot_B1; va3 = Tba1; va4 = A1_dot_B0; va5 = -Tba0; va6 = -Tab1;
    cb = LB0_ux < 0;
    vb0 = a1; vb1 = b0; vb2 = -A0_dot_B0; vb3 = -Tab0; vb4 = A1_dot_B0; vb5 = Tab1; vb6 = Tba0;
    break;
  case 8:  // UA0, UB1
    guard = (UA0_ux > b0) && (UB1_uy > a1);
    ca = UA0_lx > b0;
    va0 = b1; va1 = a0; va2 = A0_dot_B0; va3 = aA1_dot_B0 - Tba0 - b0; va4 = A0_dot_B1; va5 = aA1_dot_B1 - Tba1; va6 = -Tab0 - bA0_dot_B0;
    cb = UB1_ly > a1;
    vb0 = a0; vb1 = b1; vb2 = A1_dot_B1; vb3 = Tab1 - a1 + bA1_dot_B0; vb4 = A0_dot_B1; vb5 = Tab0 + bA0_dot_B0; vb6 = Tba1 - aA1_dot_B1;
    break;
  case 9:  // UA0, LB1
    guard = (UA0_lx < 0) && (LB1_uy > a1);
    ca = UA0_ux < 0;
    va0 = b1; va1 = a0; va2 = -A0_dot_B0; va3 = Tba0 - aA1_dot_B0; va4 = A0_dot_B1; va5 = aA1_dot_B1 - Tba1; va6 = -Tab0;
    cb = LB1_ly > a1;
    vb0 = a0; vb1 = b1; vb2 = A1_dot_B1; vb3 = Tab1 - a1; vb4 = A0_dot_B1; vb5 = Tab0; vb6 = Tba1 - aA1_dot_B1;
    break;
  case 10:  // LA0, UB1
    guard = (LA0_ux > b0) && (UB1_ly < 0);
    ca = LA0_lx > b0;
    va0 = b1; va1 = a0; va2 = A0_dot_B0; va3 = -b0 - Tba0; va4 = A0_dot_B1; va5 = -Tba1; va6 = -bA0_dot_B0 - Tab0;
    cb = UB1_uy < 0;
    vb0 = a0; vb1 = b1; vb2 = -A1_dot_B1; vb3 = -Tab1 - bA1_dot_B0; vb4 = A0_dot_B1; vb5 = Tab0 + bA0_dot_B0; vb6 = Tba1;
    break;
  case 11:  // LA0, LB1
    guard = (LA0_lx < 0) && (LB1_ly < 0);
    ca = LA0_ux < 0;
    va0 = b1; va1 = a0; va2 = -A0_dot_B0; va3 = Tba0; va4 = A0_dot_B1; va5 = -Tba1; va6 = -Tab0;
    cb = LB1_uy < 0;
    vb0 = a0; vb1 = b1; vb2 = -A1_dot_B1; vb3 = -Tab1; vb4 = A0_dot_B1; vb5 = Tab0; vb6 = Tba1;
    break;
  case 12:  // UA0, UB0
    guard = (UA0_uy > b1) && (UB0_uy > a1);
    ca = UA0_ly > b1;
    va0 = b0; va1 = a0; va2 = A0_dot_B1; va3 = aA1_dot_B1 - Tba1 - b1; va4 = A0_dot_B0; va5 = aA1_dot_B0 - Tba0; va6 = -Tab0 - bA0_dot_B1;
    cb = UB0_ly > a1;
    vb0 = a0; vb1 = b0; vb2 = A1_dot_B0; vb3 = Tab1 - a1 + bA1_dot_B1; vb4 = A0_dot_B0; vb5 = Tab0 + bA0_dot_B1; vb6 = Tba0 - aA1_dot_B0;
    break;
  case 13:  // UA0, LB0
    guard = (UA0_ly < 0) && (LB0_uy > a1);
    ca = UA0_uy < 0;
    va0 = b0; va1 = a0; va2 = -A0_dot_B1; va3 = Tba1 - aA1_dot_B1; va4 = A0_dot_B0; va5 = aA1_dot_B0 - Tba0; va6 = -Tab0;
    cb = LB0_ly > a1;
    vb0 = a0; vb1 = b0; vb2 = A1_dot_B0; vb3 = Tab1 - a1; vb4 = A0_dot_B0; vb5 = Tab0; vb6 = Tba0 - aA1_dot_B0;
    break;
  case 14:  // LA0, UB0
    guard = (LA0_uy > b1) && (UB0_ly < 0);
    ca = LA0_ly > b1;
    va0 = b0; va1 = a0; va2 = A0_dot_B1; va3 = -Tba1 - b1; va4 = A0_dot_B0; va5 = -Tba0; va6 = -Tab0 - bA0_dot_B1;
    cb = UB0_uy < 0;
    vb0 = a0; vb1 = b0; vb2 = -A1_dot_B0; vb3 = -Tab1 - bA1_dot_B1; vb4 = A0_dot_B0; vb5 = Tab0 + bA0_dot_B1; vb6 = Tba0;
    break;
  case 15:  // LA0, LB0
    guard = (LA0_ly < 0) && (LB0_ly < 0);
    ca = LA0_uy < 0;
    va0 = b0; va1 = a0; va2 = -A0_dot_B1; va3 = Tba1; va4 = A0_dot_B0; va5 = -Tba0; va6 = -Tab0;
    cb = LB0_uy < 0;
    vb0 = a0; vb1 = b0; vb2 = -A1_dot_B0; vb3 = -Tab1; vb4 = A0_dot_B0; vb5 = Tab0; vb6 = Tba0;
    break;
  default:
    break;
}
  if (!guard) return false;
  return (ca || in_voronoi(va0, va1, va2, va3, va4, va5, va6)) && (cb || in_voronoi(vb0, vb1, vb2, vb3, vb4, vb5, vb6));
}
// kwin: the first case whose conditions hold, or -1
HFB_HD double rect_finish(const RectPre& p, int kwin) {
  const double R00 = p.R00, R01 = p.R01, R02 = p.R02, R10 = p.R10, R11 = p.R11, R12 = p.R12, R20 = p.R20, R21 = p.R21;
  const double a0 = p.a0, a1 = p.a1, b0 = p.b0, b1 = p.b1;
  const double A0_dot_B0 = p.A0_dot_B0, A0_dot_B1 = p.A0_dot_B1, A1_dot_B0 = p.A1_dot_B0, A1_dot_B1 = p.A1_dot_B1;
  const double aA0_dot_B0 = p.aA0_dot_B0, aA0_dot_B1 = p.aA0_dot_B1, aA1_dot_B0 = p.aA1_dot_B0, aA1_dot_B1 = p.aA1_dot_B1;
  const double bA0_dot_B0 = p.bA0_dot_B0, bA1_dot_B0 = p.bA1_dot_B0, bA0_dot_B1 = p.bA0_dot_B1, bA1_dot_B1 = p.bA1_dot_B1;
  const double Tab0 = p.Tab0, Tab1 = p.Tab1, Tab2 = p.Tab2, Tba0 = p.Tba0, Tba1 = p.Tba1, Tba2 = p.Tba2;
  if (kwin >= 0) {
    v3 S = mk(0, 0, 0);
    double t, u;
    double sa = 0, sb = 0, s_ab = 0, s_at = 0, s_bt = 0;
    switch (kwin) {
    case 0: sa = a1; sb = b1; s_ab = A1_dot_B1; s_at = Tab1 + bA1_dot_B0; s_bt = Tba1 - aA0_dot_B1; break;
    case 1: sa = a1; sb = b1; s_ab = A1_dot_B1; s_at = Tab1; s_bt = Tba1 - aA0_dot_B1; break;
    case 2: sa = a1; sb = b1; s_ab = A1_dot_B1; s_at = Tab1 + bA1_dot_B0; s_bt = Tba1; break;
    case 3: sa = a1; sb = b1; s_ab = A1_dot_B1; s_at = Tab1; s_bt = Tba1; break;
    case 4: sa = a1; sb = b0; s_ab = A1_dot_B0; s_at = Tab1 + bA1_dot_B1; s_bt = Tba0 - aA0_dot_B0; break;
    case 5: sa = a1; sb = b0; s_ab = A1_dot_B0; s_at = Tab1; s_bt = Tba0 - aA0_dot_B0; break;
    case 6: sa = a1; sb = b0; s_ab = A1_dot_B0; s_at = Tab1 + bA1_dot_B1; s_bt = Tba0; break;
    case 7: sa = a1; sb = b0; s_ab = A1_dot_B0; s_at = Tab1; s_bt = Tba0; break;
    case 8: sa = a0; sb = b1; s_ab = A0_dot_B1; s_at = Tab0 + bA0_dot_B0; s_bt = Tba1 - aA1_dot_B1; break;
    case 9: sa = a0; sb = b1; s_ab = A0_dot_B1; s_at = Tab0; s_bt = Tba1 - aA1_dot_B1; break;
    case 10: sa = a0; sb = b1; s_ab = A0_dot_B1; s_at = Tab0 + bA0_dot_B0; s_bt = Tba1; break;
    case 11: sa = a0; sb = b1; s_ab = A0_dot_B1; s_at = Tab0; s_bt = Tba1; break;
    case 12: sa = a0; sb = b0; s_ab = A0_dot_B0; s_at = Tab0 + bA0_dot_B1; s_bt = Tba0 - aA1_dot_B0; break;
    case 13: sa = a0; sb = b0; s_ab = A0_dot_B0; s_at = Tab0; s_bt = Tba0 - aA1_dot_B0; break;
    case 14: sa = a0; sb = b0; s_ab = A0_dot_B0; s_at = Tab0 + bA0_dot_B1; s_bt = Tba0; break;
    case 15: sa = a0; sb = b0; s_ab = A0_dot_B0; s_at = Tab0; s_bt = Tba0; break;
    default: break;
    }
    seg_coords(t, u, sa, sb, s_ab, s_at, s_bt);
    switch (kwin) {
    case 0: S.x = Tab0 + R00 * b0 + R01 * u - a0; S.y = Tab1 + R10 * b0 + R11 * u - t; S.z = Tab2 + R20 * b0 + R21 * u; break;
    case 1: S.x = Tab0 + R01 * u - a0; S.y = Tab1 + R11 * u - t; S.z = Tab2 + R21 * u; break;
    case 2: S.x = Tab0 + R00 * b0 + R01 * u; S.y = Tab1 + R10 * b0 + R11 * u - t; S.z = Tab2 + R20 * b0 + R21 * u; break;
    case 3: S.x = Tab0 + R01 * u; S.y = Tab1 + R11 * u - t; S.z = Tab2 + R21 * u; break;
    case 4: S.x = Tab0 + R01 * b1 + R00 * u - a0; S.y = Tab1 + R11 * b1 + R10 * u - t; S.z = Tab2 + R21 * b1 + R20 * u; break;
    case 5: S.x = Tab0 + R00 * u - a0; S.y = Tab1 + R10 * u - t; S.z = Tab2 + R20 * u; break;
    case 6: S.x = Tab0 + R01 * b1 + R00 * u; S.y = Tab1 + R11 * b1 + R10 * u - t; S.z = Tab2 + R21 * b1 + R20 * u; break;
    case 7: S.x = Tab0 + R00 * u; S.y = Tab1 + R10 * u - t; S.z = Tab2 + R20 * u; break;
    case 8: S.x = Tab0 + R00 * b0 + R01 * u - t; S.y = Tab1 + R10 * b0 + R11 * u - a1; S.z = Tab2 + R20 * b0 + R21 * u; break;
    case 9: S.x = Tab0 + R01 * u - t; S.y = Tab1 + R11 * u - a1; S.z = Tab2 + R21 * u; break;
    case 10: S.x = Tab0 + R00 * b0 + R01 * u - t; S.y = Tab1 + R10 * b0 + R11 * u; S.z = Tab2 + R20 * b0 + R21 * u; break;
    case 11: S.x = Tab0 + R01 * u - t; S.y = Tab1 + R11 * u; S.z = Tab2 + R21 * u; break;
    case 12: S.x = Tab0 + R01 * b1 + R00 * u - t; S.y = Tab1 + R11 * b1 + R10 * u - a1; S.z = Tab2 + R21 * b1 + R20 * u; break;
    case 13: S.x = Tab0 + R00 * u - t; S.y = Tab1 + R10 * u - a1; S.z = Tab2 + R20 * u; break;
    case 14: S.x = Tab0 + R01 * b1 + R00 * u - t; S.y = Tab1 + R11 * b1 + R10 * u; S.z = Tab2 + R21 * b1 + R20 * u; break;
    case 15: S.x = Tab0 + R00 * u - t; S.y = Tab1 + R10 * u; S.z = Tab2 + R20 * u; break;
    default: break;
    }
    return nrm(S);
  }
  // no edge pair holds the closest points: separation along the face normals
  double sep1, sep2;
  if (Tab2 > 0.0) {
    sep1 = Tab2;
    if (R20 < 0.0) sep1 += b0 * R20;
    if (R21 < 0.0) sep1 += b1 * R21;
  } else {
    sep1 = -Tab2;
    if (R20 > 0.0) sep1 -= b0 * R20;
    if (R21 > 0.0) sep1 -= b1 * R21;
  }
  if (Tba2 < 0) {
    sep2 = -Tba2;
    if (R02 < 0.0) sep2 += a0 * R02;
    if (R12 < 0.0) sep2 += a1 * R12;
  } else {
    sep2 = Tba2;
    if (R02 > 0.0) sep2 -= a0 * R02;
    if (R12 > 0.0) sep2 -= a1 * R12;
  }
  const double sep = (sep1 > sep2 ? sep1 : sep2);
  return (sep > 0 ? sep : 0);
}
HFB_HD_NOINLINE double rect_distance(const m3& Rab, v3 Tab, double a0, double a1, double b0, double b1,
                                     unsigned lanes) {
  RectPre p;
  rect_prelude(Rab, Tab, a0, a1, b0, b1, p);
  // the cases are a loop, not sixteen blocks with a return each: the lanes of `lanes` (one query each)
  // walk them side by side and the two inVoronoi tests of a case are one copy of code
  int kwin = -1;
#pragma unroll 1
  for (int k = 0; k < 16; ++k) {
    if (kwin < 0 && rect_case(p, k)) kwin = k;
    if (HFB_LANES_ALL(lanes, kwin >= 0)) break;  // every lane of the phase has its case
  }
  return rect_finish(p, kwin);
}

// distance(R0, T0, b1, b2) (RSS.cpp:995-1005)
HFB_HD double rss_distance(const m3& R0, v3 T0, const RssD& b1, const RssD& b2, unsigned lanes = 0) {
  const m3 b1t = mtrans(b1.axes);
  const m3 R = mmulm(mmulm(b1t, R0), b2.axes);
  const v3 Ttemp = mmul(R0, b2.Tr) + T0 - b1.Tr;
  const v3 T = mtmul(b1.axes, Ttemp);
  double dist = rect_distance(R, T, b1.l0, b1.l1, b2.l0, b2.l1, lanes);
  dist -= (b1.radius + b2.radius);
  return (dist < 0.0) ? 0.0 : dist;
}

// -------------------------------------------------------------------- OBB -------
// obbDisjointAndLowerBoundDistance (OBB.cpp:290-393)
HFB_HD bool obb_disjoint_lb(const m3& B, v3 T, v3 a_, v3 b_, double security_margin, double break_distance,
                            double& sq_lb) {
  const double bd2 = break_distance * break_distance;
  m3 Bf;
  Bf.r0 = mk(fabs(B.r0.x), fabs(B.r0.y), fabs(B.r0.z));
  Bf.r1 = mk(fabs(B.r1.x), fabs(B.r1.y), fabs(B.r1.z));
  Bf.r2 = mk(fabs(B.r2.x), fabs(B.r2.y), fabs(B.r2.z));
  const double hm = security_margin / 2;
  const v3 a = mk(fmax(a_.x + hm, 0.0), fmax(a_.y + hm, 0.0), fmax(a_.z + hm, 0.0));
  const v3 b = mk(fmax(b_.x + hm, 0.0), fmax(b_.y + hm, 0.0), fmax(b_.z + hm, 0.0));
  {
    v3 corner = mk(fabs(T.x) - a.x, fabs(T.y) - a.y, fabs(T.z) - a.z);
    corner = corner - mmul(Bf, b);
    const v3 c = mk(fmax(corner.x, 0.0), fmax(corner.y, 0.0), fmax(corner.z, 0.0));
    sq_lb = sqn(c);
  }
  if (sq_lb > bd2) return true;
  {
    double s, t = 0;
    s = fabs(dot(mcol(B, 0), T)) - dot(mcol(Bf, 0), a) - b.x;
    if (s > 0) t += s * s;
    s = fabs(dot(mcol(B, 1), T)) - dot(mcol(Bf, 1), a) - b.y;
    if (s > 0) t += s * s;
    s = fabs(dot(mcol(B, 2), T)) - dot(mcol(Bf, 2), a) - b.z;
    if (s > 0) t += s * s;
    sq_lb = t;
  }
  if (sq_lb > bd2) return true;
  int ja = 1, ka = 2;
  for (int ia = 0; ia < 3; ++ia) {
    for (int ib = 0; ib < 3; ++ib) {
      const int jb = (ib + 1) % 3, kb = (ib + 2) % 3;
      const double bf = mel(Bf, ia, ib);
      const double sinus2 = 1 - bf * bf;
      if (sinus2 < 1e-6) continue;
      const double s = comp(T, ka) * mel(B, ja, ib) - comp(T, ja) * mel(B, ka, ib);
      const double diff = fabs(s) - (comp(a, ja) * mel(Bf, ka, ib) + comp(a, ka) * mel(Bf, ja, ib) +
                                     comp(b, jb) * mel(Bf, ia, kb) + comp(b, kb) * mel(Bf, ia, jb));
      if (diff > 0) {
        sq_lb = diff * diff / sinus2;
        if (sq_lb > bd2) return true;
      }
    }
    ja = ka;
    ka = ia;
  }
  return false;
}
// overlap(R0, T0, b1, b2, request, sqrDistLowerBound) (OBB.cpp:475-483)
HFB_HD bool obb_overlap(const m3& R0, v3 T0, const ObbD& b1, const ObbD& b2, double security_margin,
                        double break_distance, double& sq_lb) {
  const v3 Ttemp = mtmul(R0, b2.To - T0) - b1.To;
  const v3 T = mtmul(b1.axes, Ttemp);
  const m3 R = mmulm(mmulm(mtrans(b1.axes), mtrans(R0)), b2.axes);
  return !obb_disjoint_lb(R, T, b1.extent, b2.extent, security_margin, break_distance, sq_lb);
}

// ------------------------------------------------------ shape bounding volume -----
// getBoundVertices (geometric_shapes_utility.cpp:47-262): the i-th bound vertex in the shape frame
HFB_HD int bound_vertex_count(const ShapeD& s) {
  switch (s.type) {
    case HFB_GEOM_BOX: return 8;
    case HFB_GEOM_SPHERE: return 12;
    case HFB_GEOM_ELLIPSOID: return 12;
    case HFB_GEOM_CAPSULE: return 36;
    case HFB_GEOM_CONE: return 7;
    case HFB_GEOM_CYLINDER: return 12;
    case HFB_GEOM_CONVEX: return s.nv;
    default: return 0;
  }
}
// icosahedron-like 12-point pattern used for sphere / ellipsoid / capsule caps: (0,±a,±b),(±a,±b,0),(±b,0,±a)
HFB_HD v3 ico12(int i, double ax, double ay, double az, double bx, double by, double bz) {
  switch (i) {
    case 0: return mk(0, ay, bz);
    case 1: return mk(0, -ay, bz);
    case 2: return mk(0, ay, -bz);
    case 3: return mk(0, -ay, -bz);
    case 4: return mk(ax, by, 0);
    case 5: return mk(-ax, by, 0);
    case 6: return mk(ax, -by, 0);
    case 7: return mk(-ax, -by, 0);
    case 8: return mk(bx, 0, az);
    case 9: return mk(bx, 0, -az);
    case 10: return mk(-bx, 0, az);
    default: return mk(-bx, 0, -az);
  }
}
HFB_HD v3 hexagon(int i, double r2, double c, double d, double z) {  // (r2,0),(c,d),(-c,d),(-r2,0),(-c,-d),(c,-d)
  switch (i) {
    case 0: return mk(r2, 0, z);
    case 1: return mk(c, d, z);
    case 2: return mk(-c, d, z);
    case 3: return mk(-r2, 0, z);
    case 4: return mk(-c, -d, z);
    default: return mk(c, -d, z);
  }
}
HFB_HD v3 bound_vertex_local(const ShapeD& s, int i) {
  switch (s.type) {
    case HFB_GEOM_BOX:
      return mk((i & 4) ? -s.p0 : s.p0, (i & 2) ? -s.p1 : s.p1, (i & 1) ? -s.p2 : s.p2);
    case HFB_GEOM_SPHERE: {
      const double m = (1 + sqrt(5.0)) / 2.0;
      const double e = s.p0 * 6 / (sqrt(27.0) + sqrt(15.0));
      const double a = e, b = m * e;
      return ico12(i, a, a, a, b, b, b);
    }
    case HFB_GEOM_ELLIPSOID: {
      const double phi = (1 + sqrt(5.0)) / 2.0;
      const double a = sqrt(3.0) / (phi * phi);
      const double b = phi * a;
      return ico12(i, s.p0 * a, s.p1 * a, s.p2 * a, s.p0 * b, s.p1 * b, s.p2 * b);
    }
    case HFB_GEOM_CAPSULE: {
      const double m = (1 + sqrt(5.0)) / 2.0;
      const double hl = s.p1;
      const double e = s.p0 * 6 / (sqrt(27.0) + sqrt(15.0));
      const double a = e, b = m * e;
      const double r2 = s.p0 * 2 / sqrt(3.0);
      if (i < 24) {
        const int k = i % 12;
        const bool top = i < 12;
        // z offsets: (0,±a,±b + hl) etc. -- written as in the reference: b + hl, -b + hl, a + hl, -a + hl; b - hl, ...
        switch (k) {
          case 0: return mk(0, a, top ? (b + hl) : (b - hl));
          case 1: return mk(0, -a, top ? (b + hl) : (b - hl));
          case 2: return mk(0, a, top ? (-b + hl) : (-b - hl));
          case 3: return mk(0, -a, top ? (-b + hl) : (-b - hl));
          case 4: return mk(a, b, top ? hl : -hl);
          case 5: return mk(-a, b, top ? hl : -hl);
          case 6: return mk(a, -b, top ? hl : -hl);
          case 7: return mk(-a, -b, top ? hl : -hl);
          case 8: return mk(b, 0, top ? (a + hl) : (a - hl));
          case 9: return mk(b, 0, top ? (-a + hl) : (-a - hl));
          case 10: return mk(-b, 0, top ? (a + hl) : (a - hl));
          default: return mk(-b, 0, top ? (-a + hl) : (-a - hl));
        }
      }
      const double c = 0.5 * r2, d = s.p0;
      return hexagon((i - 24) % 6, r2, c, d, (i < 30) ? hl : -hl);
    }
    case HFB_GEOM_CONE: {
      const double hl = s.p1, r2 = s.p0 * 2 / sqrt(3.0), a = 0.5 * r2, b = s.p0;
      if (i == 6) return mk(0, 0, hl);
      return hexagon(i, r2, a, b, -hl);
    }
    case HFB_GEOM_CYLINDER: {
      const double hl = s.p1, r2 = s.p0 * 2 / sqrt(3.0), a = 0.5 * r2, b = s.p0;
      return hexagon(i % 6, r2, a, b, (i < 6) ? -hl : hl);
    }
    case HFB_GEOM_CONVEX:
      return mk(s.cx[i], s.cy[i], s.cz[i]);
    default:
      return mk(0, 0, 0);
  }
}

// generateCoordinateSystem (tools.h:60-96)
HFB_HD void gen_coord_system(v3 w, v3& u, v3& v) {
  double inv_length;
  if (fabs(w.x) >= fabs(w.y)) {
    inv_length = 1.0 / sqrt(w.x * w.x + w.z * w.z);
    u = mk(-w.z * inv_length, 0, w.x * inv_length);
    v = mk(w.y * u.z, w.z * u.x - w.x * u.z, -w.y * u.x);
  } else {
    inv_length = 1.0 / sqrt(w.y * w.y + w.z * w.z);
    u = mk(0, w.z * inv_length, -w.y * inv_length);
    v = mk(w.y * u.z - w.z * u.y, -w.x * u.z, w.x * u.y);
  }
}

// Jacobi eigen-decomposition (tools.h:103-203) followed by axisFromEigen (BV_fitter.cpp:49-76)
HFB_HD_NOINLINE void fit_axes_from_covariance(const double Min[6], m3& axes) {
  // Min = {M00, M11, M22, M01, M12, M02}
  double R[3][3] = {{Min[0], Min[3], Min[5]}, {Min[3], Min[1], Min[4]}, {Min[5], Min[4], Min[2]}};
  double v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  double b[3], z[3], d[3];
  double dout[3] = {0, 0, 0};
  double vout[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  const int n = 3;
  for (int ip = 0; ip < n; ++ip) {
    b[ip] = d[ip] = R[ip][ip];
    z[ip] = 0;
  }
  bool done = false;
  for (int i = 0; i < 50 && !done; ++i) {
    double sm = 0;
    for (int ip = 0; ip < n; ++ip)
      for (int iq = ip + 1; iq < n; ++iq) sm += fabs(R[ip][iq]);
    if (sm == 0.0) {
      for (int k = 0; k < 3; ++k) {
        vout[k][0] = v[k][0];
        vout[k][1] = v[k][1];
        vout[k][2] = v[k][2];
        dout[k] = d[k];
      }
      done = true;
      break;
    }
    const double tresh = (i < 3) ? 0.2 * sm / (n * n) : 0.0;
    for (int ip = 0; ip < n; ++ip) {
      for (int iq = ip + 1; iq < n; ++iq) {
        double g = 100.0 * fabs(R[ip][iq]);
        if (i > 3 && fabs(d[ip]) + g == fabs(d[ip]) && fabs(d[iq]) + g == fabs(d[iq]))
          R[ip][iq] = 0.0;
        else if (fabs(R[ip][iq]) > tresh) {
          double h = d[iq] - d[ip];
          double t;
          if (fabs(h) + g == fabs(h))
            t = (R[ip][iq]) / h;
          else {
            const double theta = 0.5 * h / (R[ip][iq]);
            t = 1.0 / (fabs(theta) + sqrt(1.0 + theta * theta));
            if (theta < 0.0) t = -t;
          }
          const double c = 1.0 / sqrt(1 + t * t);
          const double s = t * c;
          const double tau = s / (1.0 + c);
          h = t * R[ip][iq];
          z[ip] -= h;
          z[iq] += h;
          d[ip] -= h;
          d[iq] += h;
          R[ip][iq] = 0.0;
          for (int j = 0; j < ip; ++j) {
            g = R[j][ip];
            h = R[j][iq];
            R[j][ip] = g - s * (h + g * tau);
            R[j][iq] = h + s * (g - h * tau);
          }
          for (int j = ip + 1; j < iq; ++j) {
            g = R[ip][j];
            h = R[j][iq];
            R[ip][j] = g - s * (h + g * tau);
            R[j][iq] = h + s * (g - h * tau);
          }
          for (int j = iq + 1; j < n; ++j) {
            g = R[ip][j];
            h = R[iq][j];
            R[ip][j] = g - s * (h + g * tau);
            R[iq][j] = h + s * (g - h * tau);
          }
          for (int j = 0; j < n; ++j) {
            g = v[j][ip];
            h = v[j][iq];
            v[j][ip] = g - s * (h + g * tau);
            v[j][iq] = h + s * (g - h * tau);
          }
        }
      }
    }
    for (int ip = 0; ip < n; ++ip) {
      b[ip] += z[ip];
      d[ip] = b[ip];
      z[ip] = 0.0;
    }
  }
  // axisFromEigen
  int mn, mid, mx;
  if (dout[0] > dout[1]) { mx = 0; mn = 1; } else { mn = 0; mx = 1; }
  if (dout[2] < dout[mn]) { mid = mn; mn = 2; }
  else if (dout[2] > dout[mx]) { mid = mx; mx = 2; }
  else { mid = 2; }
  const v3 c0 = mk(vout[0][mx], vout[1][mx], vout[2][mx]);
  const v3 c1 = mk(vout[0][mid], vout[1][mid], vout[2][mid]);
  const v3 c2 = mk(vout[1][mx] * vout[2][mid] - vout[1][mid] * vout[2][mx],
                   vout[0][mid] * vout[2][mx] - vout[0][mx] * vout[2][mid],
                   vout[0][mx] * vout[1][mid] - vout[0][mid] * vout[1][mx]);
  axes.r0 = mk(c0.x, c1.x, c2.x);
  axes.r1 = mk(c0.y, c1.y, c2.y);
  axes.r2 = mk(c0.z, c1.z, c2.z);
}

// world-frame bound vertex i
HFB_HD_NOINLINE v3 bound_vertex(const ShapeD& s, const xf& tf, int i) { return xform(tf, bound_vertex_local(s, i)); }

// getCovariance over the bound vertices (BVH_utility.cpp:183-259, point branch)
HFB_HD void bound_covariance(const ShapeD& s, const xf& tf, int n, double M[6]) {
  v3 S1 = mk(0, 0, 0);
  double s00 = 0, s11 = 0, s22 = 0, s01 = 0, s02 = 0, s12 = 0;
  for (int i = 0; i < n; ++i) {
    const v3 p = bound_vertex(s, tf, i);
    S1 = S1 + p;
    s00 += (p.x * p.x);
    s11 += (p.y * p.y);
    s22 += (p.z * p.z);
    s01 += (p.x * p.y);
    s02 += (p.x * p.z);
    s12 += (p.y * p.z);
  }
  const unsigned np = (unsigned)n;
  M[0] = s00 - S1.x * S1.x / np;
  M[1] = s11 - S1.y * S1.y / np;
  M[2] = s22 - S1.z * S1.z / np;
  M[3] = s01 - S1.x * S1.y / np;
  M[4] = s12 - S1.y * S1.z / np;
  M[5] = s02 - S1.x * S1.z / np;
}

// point sets the fitting routines run over: the bound vertices of a shape (computeBV), or the vertices
// of a list of mesh triangles, triangle-major (BVFitter<OBBRSS>::fit, the tree builder)
struct BoundPts {
  const ShapeD& s;
  const xf& tf;
  HFB_HD v3 at(int i) const { return bound_vertex(s, tf, i); }
};
struct TriPts {
  const double* verts;      // xyz triples
  const uint32_t* tris;     // index triples
  const uint32_t* prims;    // primitive (triangle) ids
  HFB_HD v3 at(int i) const {
    const double* p = verts + 3 * (size_t)tris[3 * (size_t)prims[i / 3] + (unsigned)(i % 3)];
    return mk(p[0], p[1], p[2]);
  }
};
// projection of point i on the three axes (P[i][k] of getRadiusAndOriginAndRectangleSize)
template <class Pts>
HFB_HD v3 pts_proj(const Pts& pts, const m3& axes, int i) {
  const v3 v = pts.at(i);
  return mk(dot(mcol(axes, 0), v), dot(mcol(axes, 1), v), dot(mcol(axes, 2), v));
}

// getRadiusAndOriginAndRectangleSize (BVH_utility.cpp:264-482) over a point set; projections
// are recomputed per pass instead of being stored (the reference heap-allocates P[size][3]).
template <class Pts>
HFB_HD_NOINLINE void fit_rss_rectangle(const Pts& pts, int n, RssD& bv) {
  const m3& axes = bv.axes;
  v3 P0 = pts_proj(pts, axes, 0);
  double minz = P0.z, maxz = P0.z;
  for (int i = 1; i < n; ++i) {
    const double zv = pts_proj(pts, axes, i).z;
    if (zv < minz) minz = zv;
    else if (zv > maxz) maxz = zv;
  }
  const double r = 0.5 * (maxz - minz);
  const double radsqr = r * r;
  const double cz = 0.5 * (maxz + minz);
  double minx, maxx, miny, maxy;
  // x
  {
    int minindex = 0, maxindex = 0;
    double mintmp = P0.x, maxtmp = P0.x;
    for (int i = 1; i < n; ++i) {
      const double xv = pts_proj(pts, axes, i).x;
      if (xv < mintmp) { minindex = i; mintmp = xv; }
      else if (xv > maxtmp) { maxindex = i; maxtmp = xv; }
    }
    v3 Pm = pts_proj(pts, axes, minindex);
    double dz = Pm.z - cz;
    minx = Pm.x + sqrt(fmax(radsqr - dz * dz, 0.0));
    Pm = pts_proj(pts, axes, maxindex);
    dz = Pm.z - cz;
    maxx = Pm.x - sqrt(fmax(radsqr - dz * dz, 0.0));
    for (int i = 0; i < n; ++i) {
      const v3 Pi = pts_proj(pts, axes, i);
      if (Pi.x < minx) {
        dz = Pi.z - cz;
        const double x = Pi.x + sqrt(fmax(radsqr - dz * dz, 0.0));
        if (x < minx) minx = x;
      } else if (Pi.x > maxx) {
        dz = Pi.z - cz;
        const double x = Pi.x - sqrt(fmax(radsqr - dz * dz, 0.0));
        if (x > maxx) maxx = x;
      }
    }
  }
  // y
  {
    int minindex = 0, maxindex = 0;
    double mintmp = P0.y, maxtmp = P0.y;
    for (int i = 1; i < n; ++i) {
      const double yv = pts_proj(pts, axes, i).y;
      if (yv < mintmp) { minindex = i; mintmp = yv; }
      else if (yv > maxtmp) { maxindex = i; maxtmp = yv; }
    }
    v3 Pm = pts_proj(pts, axes, minindex);
    double dz = Pm.z - cz;
    miny = Pm.y + sqrt(fmax(radsqr - dz * dz, 0.0));
    Pm = pts_proj(pts, axes, maxindex);
    dz = Pm.z - cz;
    maxy = Pm.y - sqrt(fmax(radsqr - dz * dz, 0.0));
    for (int i = 0; i < n; ++i) {
      const v3 Pi = pts_proj(pts, axes, i);
      if (Pi.y < miny) {
        dz = Pi.z - cz;
        const double y = Pi.y + sqrt(fmax(radsqr - dz * dz, 0.0));
        if (y < miny) miny = y;
      } else if (Pi.y > maxy) {
        dz = Pi.z - cz;
        const double y = Pi.y - sqrt(fmax(radsqr - dz * dz, 0.0));
        if (y > maxy) maxy = y;
      }
    }
  }
  // corners
  const double a = sqrt(0.5);
  for (int i = 0; i < n; ++i) {
    const v3 Pi = pts_proj(pts, axes, i);
    double dx, dy, u, t;
    if (Pi.x > maxx) {
      if (Pi.y > maxy) {
        dx = Pi.x - maxx;
        dy = Pi.y - maxy;
        u = dx * a + dy * a;
        t = (a * u - dx) * (a * u - dx) + (a * u - dy) * (a * u - dy) + (cz - Pi.z) * (cz - Pi.z);
        u = u - sqrt(fmax(radsqr - t, 0.0));
        if (u > 0) { maxx += u * a; maxy += u * a; }
      } else if (Pi.y < miny) {
        dx = Pi.x - maxx;
        dy = Pi.y - miny;
        u = dx * a - dy * a;
        t = (a * u - dx) * (a * u - dx) + (-a * u - dy) * (-a * u - dy) + (cz - Pi.z) * (cz - Pi.z);
        u = u - sqrt(fmax(radsqr - t, 0.0));
        if (u > 0) { maxx += u * a; miny -= u * a; }
      }
    } else if (Pi.x < minx) {
      if (Pi.y > maxy) {
        dx = Pi.x - minx;
        dy = Pi.y - maxy;
        u = dy * a - dx * a;
        t = (-a * u - dx) * (-a * u - dx) + (a * u - dy) * (a * u - dy) + (cz - Pi.z) * (cz - Pi.z);
        u = u - sqrt(fmax(radsqr - t, 0.0));
        if (u > 0) { minx -= u * a; maxy += u * a; }
      } else if (Pi.y < miny) {
        dx = Pi.x - minx;
        dy = Pi.y - miny;
        u = -dx * a - dy * a;
        t = (-a * u - dx) * (-a * u - dx) + (-a * u - dy) * (-a * u - dy) + (cz - Pi.z) * (cz - Pi.z);
        u = u - sqrt(fmax(radsqr - t, 0.0));
        if (u > 0) { minx -= u * a; miny -= u * a; }
      }
    }
  }
  bv.Tr = mmul(axes, mk(minx, miny, cz));
  bv.l0 = fmax(maxx - minx, 0.0);
  bv.l1 = fmax(maxy - miny, 0.0);
  bv.radius = r;
}

// getExtentAndCenter_pointcloud (BVH_utility.cpp:487-527) over the bound vertices
HFB_HD void fit_obb_extent(const ShapeD& s, const xf& tf, int n, ObbD& bv) {
  v3 mn = mk(DBL_MAX, DBL_MAX, DBL_MAX), mx = mk(-DBL_MAX, -DBL_MAX, -DBL_MAX);
  for (int i = 0; i < n; ++i) {
    const v3 proj = mtmul(bv.axes, bound_vertex(s, tf, i));
    if (proj.x > mx.x) mx.x = proj.x;
    if (proj.x < mn.x) mn.x = proj.x;
    if (proj.y > mx.y) mx.y = proj.y;
    if (proj.y < mn.y) mn.y = proj.y;
    if (proj.z > mx.z) mx.z = proj.z;
    if (proj.z < mn.z) mn.z = proj.z;
  }
  bv.To = mmul(bv.axes, mx + mn) / 2;
  bv.extent = (mx - mn) / 2;
}

// fit(ps, n, bv) (BV_fitter.cpp:455-470): n = 1, 2, 3 special cases, else covariance fit.
// Only ConvexBase with fewer than 4 vertices can take the special cases.
HFB_HD void fit_axes_small(const ShapeD& s, const xf& tf, int n, m3& axes, v3& p_first, v3& p_second, double& len12) {
  const v3 p1 = bound_vertex(s, tf, 0);
  p_first = p1;
  if (n == 1) {
    axes.r0 = mk(1, 0, 0);
    axes.r1 = mk(0, 1, 0);
    axes.r2 = mk(0, 0, 1);
    return;
  }
  const v3 p2 = bound_vertex(s, tf, 1);
  p_second = p2;
  if (n == 2) {
    v3 p1p2 = p1 - p2;
    len12 = nrm(p1p2);
    const v3 c0 = unit(p1p2);
    v3 u, v;
    gen_coord_system(c0, u, v);
    axes.r0 = mk(c0.x, u.x, v.x);
    axes.r1 = mk(c0.y, u.y, v.y);
    axes.r2 = mk(c0.z, u.z, v.z);
    return;
  }
  const v3 p3 = bound_vertex(s, tf, 2);
  const v3 e0 = p1 - p2, e1 = p2 - p3, e2 = p3 - p1;
  const double l0 = sqn(e0), l1 = sqn(e1), l2 = sqn(e2);
  int imax = 0;
  if (l1 > l0) imax = 1;
  if (l2 > (imax == 0 ? l0 : l1)) imax = 2;
  const v3 c2 = unit(cross(e0, e1));
  const v3 c0 = unit(imax == 0 ? e0 : (imax == 1 ? e1 : e2));
  const v3 c1 = cross(c2, c0);
  axes.r0 = mk(c0.x, c1.x, c2.x);
  axes.r1 = mk(c0.y, c1.y, c2.y);
  axes.r2 = mk(c0.z, c1.z, c2.z);
}

HFB_HD void compute_shape_rss(const ShapeD& s, const xf& tf, RssD& bv) {  // RSS half of computeBV<OBBRSS,S>
  const int n = bound_vertex_count(s);
  if (n <= 3) {
    v3 p1, p2;
    double len = 0;
    if (n == 2) {
      // RSS fit2 (:155-168) normalises with axes.col(0) /= len rather than normalize()
      p1 = bound_vertex(s, tf, 0);
      p2 = bound_vertex(s, tf, 1);
      v3 c0 = p1 - p2;
      len = nrm(c0);
      c0 = c0 / len;
      v3 u, v;
      gen_coord_system(c0, u, v);
      bv.axes.r0 = mk(c0.x, u.x, v.x);
      bv.axes.r1 = mk(c0.y, u.y, v.y);
      bv.axes.r2 = mk(c0.z, u.z, v.z);
      bv.l0 = len;
      bv.l1 = 0;
      bv.Tr = p2;
      bv.radius = 0;
      return;
    }
    fit_axes_small(s, tf, n, bv.axes, p1, p2, len);
    if (n == 1) {
      bv.Tr = p1;
      bv.l0 = bv.l1 = 0;
      bv.radius = 0;
      return;
    }
    fit_rss_rectangle(BoundPts{s, tf}, 3, bv);
    return;
  }
  double M[6];
  bound_covariance(s, tf, n, M);
  fit_axes_from_covariance(M, bv.axes);
  fit_rss_rectangle(BoundPts{s, tf}, n, bv);
}

HFB_HD void compute_shape_obb(const ShapeD& s, const xf& tf, ObbD& bv) {  // OBB half of computeBV<OBBRSS,S>
  const int n = bound_vertex_count(s);
  if (n <= 3) {
    v3 p1, p2;
    double len = 0;
    fit_axes_small(s, tf, n, bv.axes, p1, p2, len);
    if (n == 1) {
      bv.To = p1;
      bv.extent = mk(0, 0, 0);
      return;
    }
    if (n == 2) {
      bv.extent = mk(len * 0.5, 0, 0);
      bv.To = (p1 + p2) / 2;
      return;
    }
    fit_obb_extent(s, tf, 3, bv);
    return;
  }
  double M[6];
  bound_covariance(s, tf, n, M);
  fit_axes_from_covariance(M, bv.axes);
  fit_obb_extent(s, tf, n, bv);
}

// computeBV<OBB, S>, the specialisations a plain BVHModel<OBB> walk uses for the shape's box
// (geometric_shapes_utility.cpp:458-545): pose and half sizes for Box / Sphere / Capsule / Cone / Cylinder, the fit
// of the local vertices moved by the pose for ConvexBase; Ellipsoid has no specialisation and takes the generic fit
HFB_HD void compute_shape_obb_plain(const ShapeD& s, const xf& tf, ObbD& bv) {
  switch (s.type) {
    case HFB_GEOM_BOX:
      bv.To = tf.T;
      bv.axes = tf.R;
      bv.extent = mk(s.p0, s.p1, s.p2);
      return;
    case HFB_GEOM_SPHERE:
      bv.To = tf.T;
      bv.axes.r0 = mk(1, 0, 0);
      bv.axes.r1 = mk(0, 1, 0);
      bv.axes.r2 = mk(0, 0, 1);
      bv.extent = mk(s.p0, s.p0, s.p0);
      return;
    case HFB_GEOM_CAPSULE:
      bv.To = tf.T;
      bv.axes = tf.R;
      bv.extent = mk(s.p0, s.p0, s.p1 + s.p0);
      return;
    case HFB_GEOM_CONE:
    case HFB_GEOM_CYLINDER:
      bv.To = tf.T;
      bv.axes = tf.R;
      bv.extent = mk(s.p0, s.p0, s.p1);
      return;
    case HFB_GEOM_CONVEX: {
      xf id;
      id.R.r0 = mk(1, 0, 0);
      id.R.r1 = mk(0, 1, 0);
      id.R.r2 = mk(0, 0, 1);
      id.T = mk(0, 0, 0);
      compute_shape_obb(s, id, bv);  // fit(points, n, bv) in the shape frame
      bv.axes = mmulm(tf.R, bv.axes);
      bv.To = mmul(tf.R, bv.To) + tf.T;
      return;
    }
    default:
      compute_shape_obb(s, tf, bv);
  }
}

// ----------------------------------------------------------------- node access ----
HFB_HD RssD load_node_rss(const hfb_bvh_node& nd) {
  RssD r;
  r.axes = load_colmajor(nd.rss_axes);
  r.Tr = mk(nd.rss_Tr[0], nd.rss_Tr[1], nd.rss_Tr[2]);
  r.l0 = nd.rss_length[0];
  r.l1 = nd.rss_length[1];
  r.radius = nd.rss_radius;
  return r;
}
HFB_HD ObbD load_node_obb(const hfb_bvh_node& nd) {
  ObbD o;
  o.axes = load_colmajor(nd.obb_axes);
  o.To = mk(nd.obb_To[0], nd.obb_To[1], nd.obb_To[2]);
  o.extent = mk(nd.obb_extent[0], nd.obb_extent[1], nd.obb_extent[2]);
  return o;
}

#define HFB_BVH_STACK 128

HFB_HD bool is_bvh_type(uint32_t t) { return t == HFB_BV_OBBRSS || t == HFB_BV_OBB; }

struct BvhQuery {  // one (mesh, shape) query after the operand swap of distance()/collide()
  bool plain_obb;  // BVHModel<OBB>: collide() only (see hfb_geom_register_bvh_obb)
  const hfb_bvh_node* nodes;
  const double* verts;    // xyz triples
  const uint32_t* tris;   // index triples
  xf tf_mesh, tf_shape;
  ShapeD shape;
};

// resolves the (BVH, shape) operands of a pair; `swapped` when the caller passed (shape, BVH)
// (distance.cpp:74-89, collision.cpp:92-108).  Returns false for unsupported partners
// (mesh-mesh, triangle, plane, ...).
template <int CAPS>
HFB_HD bool bvh_make_query(const ArenaView& A, uint32_t h1, const xf& tf1, uint32_t h2, const xf& tf2, BvhQuery& q,
                           bool& swapped) {
  const hfb_shape& r1 = A.shapes[h1];
  const hfb_shape& r2 = A.shapes[h2];
  swapped = !is_bvh_type(r1.type);
  const hfb_shape& rm = swapped ? r2 : r1;
  const uint32_t hs = swapped ? h1 : h2;
  const hfb_shape& rs = swapped ? r1 : r2;
  if (!is_bvh_type(rm.type)) return false;
  q.plain_obb = rm.type == HFB_BV_OBB;
  if (!(rs.type == HFB_GEOM_BOX || rs.type == HFB_GEOM_SPHERE || rs.type == HFB_GEOM_CAPSULE ||
        rs.type == HFB_GEOM_CONE || rs.type == HFB_GEOM_CYLINDER || rs.type == HFB_GEOM_ELLIPSOID ||
        rs.type == HFB_GEOM_CONVEX))
    return false;
  // computeBV<OBBRSS, S> refuses a swept-sphere radius ("not yet supported", geometric_shapes_utility.h:73-78)
  if (rs.ssr > 0) return false;
  const BvhDesc& d = A.bvh_desc[rm.data];
  q.nodes = A.bvh_nodes + d.node_off;
  q.verts = A.bvh_verts + 3 * (size_t)d.vert_off;
  q.tris = A.bvh_tris + 3 * (size_t)d.tri_off;
  q.tf_mesh = swapped ? tf2 : tf1;
  q.tf_shape = swapped ? tf1 : tf2;
  q.shape = load_shape<CAPS>(A, hs);
  return true;
}

// leaf: TriangleP(mesh triangle) vs shape, internal::ShapeShapeDistance<TriangleP,S>
// (traversal_node_bvh_shape.h:342-364, 139-188); solver warm-start state carries from leaf to leaf.
template <int CAPS>
HFB_HD void bvh_leaf(const BvhQuery& q, int primitive_id, const SolverP& P, EpaWs* ws, PairIn& in, PairOut& o) {
  const uint32_t* t = q.tris + 3 * (size_t)primitive_id;
  const double* a = q.verts + 3 * (size_t)t[0];
  const double* b = q.verts + 3 * (size_t)t[1];
  const double* c = q.verts + 3 * (size_t)t[2];
  in.s1.type = HFB_GEOM_TRIANGLE;
  in.s1.ssr = 0;
  in.s1.p0 = in.s1.p1 = in.s1.p2 = 0;
  in.s1.nv = 0;
  in.s1.cx = in.s1.cy = in.s1.cz = nullptr;
  in.s1.center = mk(0, 0, 0);
  in.s1.ta = mk(a[0], a[1], a[2]);
  in.s1.tb = mk(b[0], b[1], b[2]);
  in.s1.tc = mk(c[0], c[1], c[2]);
  GjkState g;
  if (pair_phase1<1, CAPS, PATH_BOTH>(in, P, o, g)) pair_phase2<1, CAPS>(in, P, g, ws, o);
  // GJKSolver keeps cached_guess / support_func_cached_guess between calls (narrowphase.h:353-391, 625-626)
  in.cached_guess = o.cached_guess;
  in.hint0 = o.hint0;
  in.hint1 = o.hint1;
}

// ---- warp-scheduled walk ------------------------------------------------------------------------
// One lane walks one query's tree, depth first, in exactly the order of the reference's recursion.
// Left to itself every lane of a warp would be in a different piece of code (bounding-volume test,
// GJK on a leaf, EPA, stack handling) and queries differ tenfold in length: few lanes of a warp would be
// active per issued instruction.  So (1) a lane that finishes a query fetches the next one itself, and
// (2) the lanes vote: each is waiting to set up a query, to run a bounding-volume test or to run a
// leaf test; the warp runs the phase most lanes wait for and the others sit that round out.  The order
// of events inside a query is untouched -- a lane only ever delays its own next step.
enum { BVS_FETCH = 0, BVS_ADVANCE = 1, BVS_NEED_INIT = 2, BVS_NEED_BV = 3, BVS_NEED_LEAF = 4, BVS_EXIT = 5 };
#define HFB_BVH_INIT_QUORUM 6  // lanes waiting for a new query before the (long) set-up phase is run
struct WarpVote {
  static HFB_HD unsigned ballot(bool p) {
#if defined(__CUDA_ARCH__)
    return __ballot_sync(0xffffffffu, p);
#else
    return p ? 1u : 0u;
#endif
  }
  static HFB_HD int popc(unsigned m) {
#if defined(__CUDA_ARCH__)
    return __popc(m);
#else
    return __builtin_popcount(m);
#endif
  }
  static HFB_HD void sync() {
#if defined(__CUDA_ARCH__)
    __syncwarp();
#endif
  }
};
// 0: set-up phase, 1: bounding-volume phase, 2: leaf phase, -1: every lane has left
// `lanes`: the lanes that run the chosen phase
template <int QUORUM>
HFB_HD int bvh_vote(int state, unsigned& lanes) {
#if !defined(__CUDACC__) && defined(HFB_LANE_SIM)
  lanesim::trace_bvh_state(state);  // tests/tools/bvh_sched_model.py: per-query phase sequences for the offline model
#endif
  const unsigned mi = WarpVote::ballot(state == BVS_NEED_INIT);
  const unsigned mb = WarpVote::ballot(state == BVS_NEED_BV);
  const unsigned ml = WarpVote::ballot(state == BVS_NEED_LEAF);
  const int ni = WarpVote::popc(mi), nb = WarpVote::popc(mb), nl = WarpVote::popc(ml);
  lanes = 0;
  if (ni + nb + nl == 0) return -1;
  if (ni >= QUORUM || nb + nl == 0) {
    lanes = mi;
    return 0;
  }
  lanes = (nl >= nb) ? ml : mb;
  return (nl >= nb) ? 2 : 1;
}

// Where the contacts of a mesh pair go beyond the first (hfb_batch_collide_contacts): the reference keeps up to
// num_max_contacts of them in CollisionResult::contacts (collision_data.h:431), the batch record holds contacts[0].
// All null / zero for the plain entry points.
struct BvhContactSink {
  hfb_contact* extra;  // extra[k - 1] receives contacts[k], k >= 1
  unsigned cap;        // records available in `extra`
  uint32_t* count;     // receives CollisionResult::numContacts()
};

// one (mesh, shape) query handed to a lane by a source: the operands after the swap of
// distance()/collide(), the solver warm start and the caller's result record
struct BvhJob {
  BvhQuery q;
  bool swapped;
  v3 cached_guess;
  int hint0, hint1;
  void* rec;
};
struct BvhColJob : BvhJob {  // collide(): plus where contacts[1..] go
  BvhContactSink sink = BvhContactSink{nullptr, 0, nullptr};
};

struct BvhDistOut {
  double min_distance;
  v3 p1, p2, normal;
  int b1;
  unsigned bv_tests, leaf_tests;
};
HFB_HD void put3d(double* o, v3 v) {
  o[0] = v.x;
  o[1] = v.y;
  o[2] = v.z;
}
// distance(): the (GEOM, BVH) operand swap of distance.cpp:74-89 is undone on o1/o2, the nearest
// points and the normal -- not on b1/b2
HFB_HD void bvh_write_shape_distance(hfb_distance_result* r, bool swapped, const BvhDistOut& o) {
  r->min_distance = o.min_distance;
  put3d(r->p1, swapped ? o.p2 : o.p1);
  put3d(r->p2, swapped ? o.p1 : o.p2);
  put3d(r->normal, swapped ? -o.normal : o.normal);
  r->b1 = o.b1;
  r->b2 = -1;
  r->status = pack_status(0, 0, HFB_PATH_BVH);
  r->iterations = (o.bv_tests & 0xffffu) | ((o.leaf_tests & 0xffffu) << 16);
}

// orientedBVHShapeDistance + distance(node) + distanceRecurse (traversal_recurse.cpp:153-203), each
// query on a fresh DistanceResult.  Every lane of the warp calls this together and keeps pulling
// queries from `src` until it has none left.  A stack entry is a node still to be visited plus the
// lower bound that canStop() re-checks when the node is popped (the reference evaluates canStop for
// the second child after the first returned).
template <int CAPS, class Src, int QUORUM = HFB_BVH_INIT_QUORUM>
HFB_HD void bvh_shape_distance_stream(Src& src, const SolverP& P, double rel_err, double abs_err, EpaWs* ws,
                                      unsigned long long& bv_total, unsigned long long& leaf_total) {
  BvhJob job;
  RssD sbv;
  PairIn in;
  BvhDistOut out;
  int stk_node[HFB_BVH_STACK];
  double stk_d[HFB_BVH_STACK];
  int sp = 0;
  int state = BVS_FETCH;
  int leaf_prim = 0, first_child = 0;
  bool seed = true;
  for (;;) {
    if (state == BVS_ADVANCE) {  // pop / prune down to the next node that needs work
      state = BVS_FETCH;
      while (sp > 0) {
        --sp;
        const int b = stk_node[sp];
        const double dlow = stk_d[sp];
        if (dlow >= 0) {  // canStop(d) (:322-327)
          if ((dlow >= out.min_distance - abs_err) && (dlow * (1 + rel_err) >= out.min_distance)) continue;
        }
        const int fc = job.q.nodes[b].first_child;
        if (fc < 0) {
          leaf_prim = -(fc + 1);
          state = BVS_NEED_LEAF;
        } else if (sp + 2 > HFB_BVH_STACK) {  // cannot happen for trees of depth < 128
          sp = 0;
        } else {
          first_child = fc;
          state = BVS_NEED_BV;
        }
        break;
      }
      if (state == BVS_FETCH) {  // walk finished
        bvh_write_shape_distance(static_cast<hfb_distance_result*>(job.rec), job.swapped, out);
        bv_total += out.bv_tests;
        leaf_total += out.leaf_tests;
      }
    }
    if (state == BVS_FETCH) state = src.next(job) ? BVS_NEED_INIT : BVS_EXIT;
    unsigned lanes;
    const int phase = bvh_vote<QUORUM>(state, lanes);
    if (phase < 0) break;
    if (phase == 0) {
      if (state == BVS_NEED_INIT) {
        compute_shape_rss(job.q.shape, job.q.tf_shape, sbv);  // traversal_node_setup.h:765
        in.cached_guess = job.cached_guess;
        in.hint0 = job.hint0;
        in.hint1 = job.hint1;
        in.s2 = job.q.shape;
        in.tf1 = job.q.tf_mesh;
        in.tf2 = job.q.tf_shape;
        out.min_distance = DBL_MAX;
        out.p1 = out.p2 = out.normal = nan3();
        out.b1 = -1;
        out.bv_tests = out.leaf_tests = 0;
        sp = 1;
        stk_node[0] = 0;
        stk_d[0] = -1.0;  // root: visited unconditionally
        // preprocess(): seed with triangle 0 (traversal_node_bvh_shape.h:457-461), not a counted leaf test
        leaf_prim = 0;
        seed = true;
        state = BVS_NEED_LEAF;
      }
    } else if (phase == 2) {
      if (state == BVS_NEED_LEAF) {  // leafComputeDistance
        PairOut o;
        bvh_leaf<CAPS>(job.q, leaf_prim, P, ws, in, o);
        if (!seed) out.leaf_tests++;
        seed = false;
        if (out.min_distance > o.distance) {  // DistanceResult::update: strict '>' keeps the first minimum
          out.min_distance = o.distance;
          out.b1 = leaf_prim;
          out.p1 = o.p1;
          out.p2 = o.p2;
          out.normal = o.normal;
        }
        state = BVS_ADVANCE;
      }
    } else {
      if (state == BVS_NEED_BV) {  // BVDistanceLowerBound of both children (:465-469)
        const int a1 = first_child, c1 = first_child + 1;
        const double d1 = rss_distance(job.q.tf_mesh.R, job.q.tf_mesh.T, sbv, load_node_rss(job.q.nodes[a1]), lanes);
        const double d2 = rss_distance(job.q.tf_mesh.R, job.q.tf_mesh.T, sbv, load_node_rss(job.q.nodes[c1]), lanes);
        out.bv_tests += 2;
        // visit the nearer child first: push the farther one below it
        if (d2 < d1) {
          stk_node[sp] = a1; stk_d[sp] = d1; ++sp;
          stk_node[sp] = c1; stk_d[sp] = d2; ++sp;
        } else {
          stk_node[sp] = c1; stk_d[sp] = d2; ++sp;
          stk_node[sp] = a1; stk_d[sp] = d1; ++sp;
        }
        state = BVS_ADVANCE;
      }
    }
    WarpVote::sync();
  }
}

// GJKSolver::getGJKInitialGuess with BoundingVolumeGuess needs aabb_local of both operands
// (narrowphase.h:368-377); the TriangleP a leaf test builds never had computeLocalAABB called, so the reference
// throws std::logic_error at the first leaf that reaches GJK (sphere partners take the closed form,
// details.h:286-342).  Mirrored as an unsupported query.
HFB_HD bool bvh_leaf_guess_throws(int initial_guess, const ShapeD& partner) {
  return initial_guess == HFB_GUESS_BOUNDING_VOLUME && partner.type != HFB_GEOM_SPHERE;
}

struct BvhColOut {
  double distance_lower_bound;
  v3 lb_p1, lb_p2, lb_normal;
  bool has_contact;
  int b1;
  double distance;
  v3 p1, p2, normal;
  unsigned bv_tests, leaf_tests;
  bool threw;  // bvh_leaf_guess_throws at a leaf: the query ends as unsupported
};
// CollisionResult::clear() as a record
HFB_HD void bvh_init_contact(hfb_contact* r) {
  r->distance = DBL_MAX;
  r->distance_lower_bound = DBL_MAX;
  put3d(r->p1, nan3());
  put3d(r->p2, nan3());
  put3d(r->normal, nan3());
  put3d(r->pos, nan3());
  r->b1 = r->b2 = -1;
  r->num_contacts = 0;
  r->iterations = 0;
  r->_pad = 0;
}
// contacts[k], k >= 1, of a mesh pair as a record of its own: the Contact fields (collision_data.h:59-148), after the
// operand swap of collide() for (shape, mesh) pairs (collision.cpp:92-108)
HFB_HD void bvh_sink_contact(const BvhContactSink& s, unsigned k, bool swapped, int b1, int b2, double distance, v3 p1,
                             v3 p2, v3 normal) {
  if (!s.extra || k == 0 || k - 1 >= s.cap) return;
  hfb_contact* r = s.extra + (k - 1);
  bvh_init_contact(r);
  r->num_contacts = 1;
  r->distance = distance;
  r->b1 = swapped ? b2 : b1;
  r->b2 = swapped ? b1 : b2;
  put3d(r->pos, (p1 + p2) / 2);
  put3d(r->p1, swapped ? p2 : p1);
  put3d(r->p2, swapped ? p1 : p2);
  put3d(r->normal, swapped ? -normal : normal);
  r->status = pack_status(0, 0, HFB_PATH_BVH);
}
// collide(): swapObjects() for (GEOM, BVH) (collision.cpp:92-108) swaps contact b1/b2, nearest points
// and normals back
HFB_HD void bvh_write_shape_collide(hfb_contact* r, bool swapped, const BvhColOut& o) {
  bvh_init_contact(r);
  if (o.threw) {
    r->status = pack_status(0, 0, HFB_PATH_UNSUPPORTED);
    return;
  }
  r->distance_lower_bound = o.distance_lower_bound;
  put3d(r->p1, swapped ? o.lb_p2 : o.lb_p1);
  put3d(r->p2, swapped ? o.lb_p1 : o.lb_p2);
  put3d(r->normal, swapped ? -o.lb_normal : o.lb_normal);
  if (o.has_contact) {
    r->num_contacts = 1;
    r->distance = o.distance;
    r->b1 = swapped ? -1 : o.b1;
    r->b2 = swapped ? o.b1 : -1;
    put3d(r->pos, (o.p1 + o.p2) / 2);
    put3d(r->p1, swapped ? o.p2 : o.p1);
    put3d(r->p2, swapped ? o.p1 : o.p2);
    put3d(r->normal, swapped ? -o.normal : o.normal);
  }
  r->status = pack_status(0, 0, HFB_PATH_BVH);
  r->iterations = (o.bv_tests & 0xffffu) | ((o.leaf_tests & 0xffffu) << 16);
}

// BVHShapeCollider<OBBRSS,S>::oriented + collide(node) + collisionRecurse (traversal_recurse.cpp:44-85),
// num_max_contacts contacts (only the first is returned), each query on a fresh CollisionResult.
// Warp-scheduled like bvh_shape_distance_stream.
template <int CAPS, class Src, int QUORUM = HFB_BVH_INIT_QUORUM>
HFB_HD void bvh_shape_collide_stream(Src& src, const SolverP& P, double security_margin, double break_distance,
                                     double collision_distance_threshold, unsigned num_max_contacts, EpaWs* ws,
                                     unsigned long long& bv_total, unsigned long long& leaf_total) {
  BvhColJob job;
  ObbD sbv;
  PairIn in;
  BvhColOut out;
  unsigned ncontacts = 0;
  int stk[HFB_BVH_STACK];
  int sp = 0;
  int state = BVS_FETCH;
  int leaf_prim = 0, node = 0;
  for (;;) {
    if (state == BVS_ADVANCE) {
      state = BVS_FETCH;
      if (sp > 0) {
        node = stk[--sp];
        const int fc = job.q.nodes[node].first_child;
        if (fc < 0) {
          leaf_prim = -(fc + 1);
          state = BVS_NEED_LEAF;
        } else if (sp + 2 > HFB_BVH_STACK) {  // cannot happen for trees of depth < 128
          sp = 0;
        } else {
          state = BVS_NEED_BV;
        }
      }
      if (state == BVS_FETCH) {
        bvh_write_shape_collide(static_cast<hfb_contact*>(job.rec), job.swapped, out);
        if (job.sink.count) *job.sink.count = out.threw ? 0u : ncontacts;
        bv_total += out.bv_tests;
        leaf_total += out.leaf_tests;
      }
    }
    if (state == BVS_FETCH) state = src.next(job) ? BVS_NEED_INIT : BVS_EXIT;
    unsigned lanes;
    const int phase = bvh_vote<QUORUM>(state, lanes);
    if (phase < 0) break;
    if (phase == 0) {
      if (state == BVS_NEED_INIT) {
        if (job.q.plain_obb) compute_shape_obb_plain(job.q.shape, job.q.tf_shape, sbv);  // computeBV<OBB, S>
        else compute_shape_obb(job.q.shape, job.q.tf_shape, sbv);  // traversal_node_setup.h:655-694
        in.cached_guess = job.cached_guess;
        in.hint0 = job.hint0;
        in.hint1 = job.hint1;
        in.s2 = job.q.shape;
        in.tf1 = job.q.tf_mesh;
        in.tf2 = job.q.tf_shape;
        out.distance_lower_bound = DBL_MAX;
        out.lb_p1 = out.lb_p2 = out.lb_normal = nan3();
        out.has_contact = false;
        out.b1 = -1;
        out.distance = DBL_MAX;
        out.p1 = out.p2 = out.normal = nan3();
        out.bv_tests = out.leaf_tests = 0;
        out.threw = false;
        ncontacts = 0;
        sp = 1;
        stk[0] = 0;
        state = BVS_ADVANCE;
      }
    } else if (phase == 2) {
      if (state == BVS_NEED_LEAF && bvh_leaf_guess_throws(P.initial_guess, job.q.shape)) {
        out.threw = true;
        sp = 0;
        state = BVS_ADVANCE;
      } else if (state == BVS_NEED_LEAF) {  // leafCollides (traversal_node_bvh_shape.h:139-188)
        PairOut o;
        bvh_leaf<CAPS>(job.q, leaf_prim, P, ws, in, o);
        out.leaf_tests++;
        const double d2c = o.distance - security_margin;
        if (d2c < out.distance_lower_bound) {  // updateDistanceLowerBoundFromLeaf
          out.distance_lower_bound = d2c;
          out.lb_p1 = o.p1;
          out.lb_p2 = o.p2;
          out.lb_normal = o.normal;
        }
        if (d2c <= collision_distance_threshold) {
          if (ncontacts < num_max_contacts) {
            if (ncontacts == 0) {
              out.has_contact = true;
              out.b1 = leaf_prim;
              out.distance = o.distance;
              out.p1 = o.p1;
              out.p2 = o.p2;
              out.normal = o.normal;
            } else {
              bvh_sink_contact(job.sink, ncontacts, job.swapped, leaf_prim, -1, o.distance, o.p1, o.p2, o.normal);
            }
            ++ncontacts;
          }
        }
        state = BVS_ADVANCE;
        // canStop() (traversal_recurse.cpp:69): once the request is satisfied every frame returns
        if (ncontacts > 0 && num_max_contacts <= ncontacts) sp = 0;
      }
    } else {
      if (state == BVS_NEED_BV) {  // BVDisjoints (:120-136)
        const hfb_bvh_node& nd = job.q.nodes[node];
        double sq_lb;
        out.bv_tests++;
        const bool disjoint = !obb_overlap(job.q.tf_mesh.R, job.q.tf_mesh.T, load_node_obb(nd), sbv,
                                           security_margin, break_distance, sq_lb);
        if (disjoint) {  // updateDistanceLowerBoundFromBV (collision_data.h:1177-1184)
          if (out.distance_lower_bound > 0) {
            const double nd_lb = sqrt(sq_lb);
            if (nd_lb < out.distance_lower_bound) out.distance_lower_bound = nd_lb;
          }
        } else {
          stk[sp++] = nd.first_child + 1;  // right child visited after the left one
          stk[sp++] = nd.first_child;
        }
        state = BVS_ADVANCE;
      }
    }
    WarpVote::sync();
  }
}

// ============================ mesh-mesh: two OBBRSS trees =========================================
// MeshDistanceTraversalNodeOBBRSS / MeshCollisionTraversalNodeOBBRSS (traversal_node_bvhs.h:63-242, 386-536)
// walked with distanceRecurse / collisionRecurse (traversal_recurse.cpp:44-85, 153-203).

// TriangleDistance::segPoints (src/intersect.cpp:60-153)
HFB_HD void seg_points(v3 P, v3 A, v3 Q, v3 B, v3& VEC, v3& X, v3& Y) {
  v3 T = Q - P;
  const double A_dot_A = dot(A, A), B_dot_B = dot(B, B), A_dot_B = dot(A, B);
  const double A_dot_T = dot(A, T), B_dot_T = dot(B, T);
  const double denom = A_dot_A * B_dot_B - A_dot_B * A_dot_B;
  double t = (A_dot_T * B_dot_B - B_dot_T * A_dot_B) / denom;
  if ((t < 0) || isnan(t)) t = 0;
  else if (t > 1) t = 1;
  const double u = (t * A_dot_B - B_dot_T) / B_dot_B;
  if ((u <= 0) || isnan(u)) {
    Y = Q;
    t = A_dot_T / A_dot_A;
    if ((t <= 0) || isnan(t)) {
      X = P;
      VEC = Q - P;
    } else if (t >= 1) {
      X = P + A;
      VEC = Q - X;
    } else {
      X = P + A * t;
      VEC = cross(A, cross(T, A));
    }
  } else if (u >= 1) {
    Y = Q + B;
    t = (A_dot_B + A_dot_T) / A_dot_A;
    if ((t <= 0) || isnan(t)) {
      X = P;
      VEC = Y - P;
    } else if (t >= 1) {
      X = P + A;
      VEC = Y - X;
    } else {
      X = P + A * t;
      T = Y - P;
      VEC = cross(A, cross(T, A));
    }
  } else {
    Y = Q + B * u;
    if ((t <= 0) || isnan(t)) {
      X = P;
      VEC = cross(B, cross(T, B));
    } else if (t >= 1) {
      X = P + A;
      T = Q - X;
      VEC = cross(B, cross(T, B));
    } else {
      X = P + A * t;
      VEC = cross(A, B);
      if (dot(VEC, T) < 0) VEC = VEC * (-1.0);
    }
  }
}

struct Tri3 {
  v3 v[3];
};

// "vertex of one triangle over the face of the other" test of sqrTriDistance (:262-303 / :311-352):
// F is the face triangle with edge vectors Fv, O the other triangle.  Returns the index of the vertex
// of O whose projection falls inside F (-1: none, -2: Fn not a separating direction); `sep` reports
// that Fn separates the triangles.
HFB_HD int tri_vertex_over_face(const Tri3& F, const v3 Fv[3], const Tri3& O, v3& Fn, double& Fnl, double proj[3],
                                bool& sep) {
  sep = false;
  Fn = cross(Fv[0], Fv[1]);
  Fnl = dot(Fn, Fn);
  if (!(Fnl > 1e-15)) return -2;
  proj[0] = dot(F.v[0] - O.v[0], Fn);
  proj[1] = dot(F.v[0] - O.v[1], Fn);
  proj[2] = dot(F.v[0] - O.v[2], Fn);
  int point = -1;
  if ((proj[0] > 0) && (proj[1] > 0) && (proj[2] > 0)) {
    point = (proj[0] < proj[1]) ? 0 : 1;
    if (proj[2] < proj[point]) point = 2;
  } else if ((proj[0] < 0) && (proj[1] < 0) && (proj[2] < 0)) {
    point = (proj[0] > proj[1]) ? 0 : 1;
    if (proj[2] > proj[point]) point = 2;
  }
  if (point < 0) return -2;
  sep = true;
  if (dot(O.v[point] - F.v[0], cross(Fn, Fv[0])) > 0 && dot(O.v[point] - F.v[1], cross(Fn, Fv[1])) > 0 &&
      dot(O.v[point] - F.v[2], cross(Fn, Fv[2])) > 0)
    return point;
  return -1;
}

// TriangleDistance::sqrTriDistance (src/intersect.cpp:156-357).  P and Q are overwritten by every
// segPoints call, so the "triangles overlap" exit (return 0) leaves the last edge pair's points in them.
HFB_HD_NOINLINE double sqr_tri_distance(const Tri3& S, const Tri3& T, v3& P, v3& Q) {
  v3 Sv[3], Tv[3], VEC;
  Sv[0] = S.v[1] - S.v[0];
  Sv[1] = S.v[2] - S.v[1];
  Sv[2] = S.v[0] - S.v[2];
  Tv[0] = T.v[1] - T.v[0];
  Tv[1] = T.v[2] - T.v[1];
  Tv[2] = T.v[0] - T.v[2];
  v3 V, Z, minP = nan3(), minQ = nan3();
  bool shown_disjoint = false;
  double mindd = dot(S.v[0] - T.v[0], S.v[0] - T.v[0]) + 1;
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) {
      seg_points(S.v[i], Sv[i], T.v[j], Tv[j], VEC, P, Q);
      V = Q - P;
      const double dd = dot(V, V);
      if (dd <= mindd) {
        minP = P;
        minQ = Q;
        mindd = dd;
        Z = S.v[(i + 2) % 3] - P;
        double a = dot(Z, VEC);
        Z = T.v[(j + 2) % 3] - Q;
        double b = dot(Z, VEC);
        if ((a <= 0) && (b >= 0)) return dd;
        const double p = dot(V, VEC);
        if (a < 0) a = 0;
        if (b > 0) b = 0;
        if ((p - a + b) > 0) shown_disjoint = true;
      }
    }
  }
  v3 n;
  double nl, proj[3];
  bool sep;
  int point = tri_vertex_over_face(S, Sv, T, n, nl, proj, sep);
  if (sep) shown_disjoint = true;
  if (point >= 0) {
    P = T.v[point] + n * (proj[point] / nl);
    Q = T.v[point];
    return dot(P - Q, P - Q);
  }
  point = tri_vertex_over_face(T, Tv, S, n, nl, proj, sep);
  if (sep) shown_disjoint = true;
  if (point >= 0) {
    P = S.v[point];
    Q = S.v[point] + n * (proj[point] / nl);
    return dot(P - Q, P - Q);
  }
  if (shown_disjoint) {
    P = minP;
    Q = minQ;
    return mindd;
  }
  return 0;
}

struct BvhMeshView {
  const hfb_bvh_node* nodes;
  const double* verts;
  const uint32_t* tris;
};
struct BvhPairQuery {  // one (mesh, mesh) query
  BvhMeshView m1, m2;
  xf tf1, tf2;
  m3 R;  // RT = tf1^-1 * tf2 (internal/tools.h:91-99, traversal_node_setup.h:561-563, 688-689)
  v3 T;
};
HFB_HD BvhMeshView bvh_mesh_view(const ArenaView& A, uint32_t bvh_id) {
  const BvhDesc& d = A.bvh_desc[bvh_id];
  BvhMeshView m;
  m.nodes = A.bvh_nodes + d.node_off;
  m.verts = A.bvh_verts + 3 * (size_t)d.vert_off;
  m.tris = A.bvh_tris + 3 * (size_t)d.tri_off;
  return m;
}
HFB_HD Tri3 bvh_triangle(const BvhMeshView& m, int primitive_id) {
  const uint32_t* t = m.tris + 3 * (size_t)primitive_id;
  Tri3 r;
  for (int k = 0; k < 3; ++k) {
    const double* a = m.verts + 3 * (size_t)t[k];
    r.v[k] = mk(a[0], a[1], a[2]);
  }
  return r;
}
// firstOverSecond (traversal_node_bvhs.h:87-98, 333-344): bv.size() of an OBBRSS is the squared norm
// of the OBB extent (OBBRSS.h:114, OBB.h:110)
HFB_HD bool bvh_first_over_second(const hfb_bvh_node& n1, const hfb_bvh_node& n2) {
  const double sz1 = (n1.obb_extent[0] * n1.obb_extent[0] + n1.obb_extent[1] * n1.obb_extent[1]) +
                     n1.obb_extent[2] * n1.obb_extent[2];
  const double sz2 = (n2.obb_extent[0] * n2.obb_extent[0] + n2.obb_extent[1] * n2.obb_extent[1]) +
                     n2.obb_extent[2] * n2.obb_extent[2];
  const bool l1 = n1.first_child < 0, l2 = n2.first_child < 0;
  return l2 || (!l1 && (sz1 > sz2));
}

struct BvhPairDistOut {
  double min_distance;
  v3 p1, p2;
  int b1, b2;
  unsigned bv_tests, leaf_tests;
};

HFB_HD void bvh_tri_pair_distance(const BvhPairQuery& q, int id1, int id2, BvhPairDistOut& out) {  // :437-470
  const Tri3 S = bvh_triangle(q.m1, id1);
  Tri3 Tt = bvh_triangle(q.m2, id2);
  for (int k = 0; k < 3; ++k) Tt.v[k] = mmul(q.R, Tt.v[k]) + q.T;  // intersect.cpp:401-409
  v3 P1 = nan3(), P2 = nan3();
  const double d = sqrt(sqr_tri_distance(S, Tt, P1, P2));
  if (out.min_distance > d) {  // DistanceResult::update (collision_data.h:1126-1138)
    out.min_distance = d;
    out.b1 = id1;
    out.b2 = id2;
    out.p1 = P1;
    out.p2 = P2;
  }
}

// orientedMeshDistance + distance(node): seed with triangles (0, 0), walk the pair tree, move the
// nearest points to the world frame.  The reference never writes `normal` on this path.
HFB_HD void bvh_bvh_distance(const BvhPairQuery& q, double rel_err, double abs_err, bool enable_nearest_points,
                             BvhPairDistOut& out) {
  out.min_distance = DBL_MAX;
  out.p1 = out.p2 = nan3();
  out.b1 = out.b2 = -1;
  out.bv_tests = out.leaf_tests = 0;
  bvh_tri_pair_distance(q, 0, 0, out);  // preprocessOrientedNode (:487-510)
  int stk_a[HFB_BVH_STACK], stk_b[HFB_BVH_STACK];
  double stk_d[HFB_BVH_STACK];
  int sp = 1;
  stk_a[0] = 0;
  stk_b[0] = 0;
  stk_d[0] = -1.0;
  while (sp > 0) {
    int leaf1 = -1, leaf2 = -1;
    while (sp > 0) {  // phase A: BV pairs
      --sp;
      const int b1 = stk_a[sp], b2 = stk_b[sp];
      const double dlow = stk_d[sp];
      if (dlow >= 0) {  // canStop (:473-478)
        if ((dlow >= out.min_distance - abs_err) && (dlow * (1 + rel_err) >= out.min_distance)) continue;
      }
      const hfb_bvh_node& n1 = q.m1.nodes[b1];
      const hfb_bvh_node& n2 = q.m2.nodes[b2];
      if (n1.first_child < 0 && n2.first_child < 0) {
        leaf1 = -(n1.first_child + 1);
        leaf2 = -(n2.first_child + 1);
        break;
      }
      int a1, a2, c1, c2;
      if (bvh_first_over_second(n1, n2)) {
        a1 = n1.first_child;
        a2 = b2;
        c1 = n1.first_child + 1;
        c2 = b2;
      } else {
        a1 = b1;
        a2 = n2.first_child;
        c1 = b1;
        c2 = n2.first_child + 1;
      }
      const double d1 = rss_distance(q.R, q.T, load_node_rss(q.m1.nodes[a1]), load_node_rss(q.m2.nodes[a2]));
      const double d2 = rss_distance(q.R, q.T, load_node_rss(q.m1.nodes[c1]), load_node_rss(q.m2.nodes[c2]));
      out.bv_tests += 2;
      if (sp + 2 > HFB_BVH_STACK) {  // deeper than any tree pair the arena accepts
        sp = 0;
        break;
      }
      if (d2 < d1) {
        stk_a[sp] = a1; stk_b[sp] = a2; stk_d[sp] = d1; ++sp;
        stk_a[sp] = c1; stk_b[sp] = c2; stk_d[sp] = d2; ++sp;
      } else {
        stk_a[sp] = c1; stk_b[sp] = c2; stk_d[sp] = d2; ++sp;
        stk_a[sp] = a1; stk_b[sp] = a2; stk_d[sp] = d1; ++sp;
      }
    }
    if (leaf1 < 0) break;
    bvh_tri_pair_distance(q, leaf1, leaf2, out);  // phase B
    out.leaf_tests++;
  }
  if (enable_nearest_points) {  // postprocessOrientedNode (:527-536)
    out.p1 = xform(q.tf1, out.p1);
    out.p2 = xform(q.tf1, out.p2);
  }
}

struct BvhPairColOut {
  double distance_lower_bound;
  v3 lb_p1, lb_p2, lb_normal;
  bool has_contact;
  int b1, b2;
  double distance;
  v3 p1, p2, normal;
  unsigned bv_tests, leaf_tests;
};

// orientedMeshCollide + collide(node).  Every leaf builds its own GJKSolver from the request
// (traversal_node_bvhs.h:197), so the warm start `in0` is the same for all of them.
template <int CAPS>
HFB_HD void bvh_bvh_collide(const BvhPairQuery& q, const SolverP& P, double security_margin, double break_distance,
                            double collision_distance_threshold, unsigned num_max_contacts, EpaWs* ws,
                            const PairIn& in0, BvhPairColOut& out, const BvhContactSink& sink) {
  out.distance_lower_bound = DBL_MAX;
  out.lb_p1 = out.lb_p2 = out.lb_normal = nan3();
  out.has_contact = false;
  out.b1 = out.b2 = -1;
  out.distance = DBL_MAX;
  out.p1 = out.p2 = out.normal = nan3();
  out.bv_tests = out.leaf_tests = 0;
  unsigned ncontacts = 0;
  int stk_a[HFB_BVH_STACK], stk_b[HFB_BVH_STACK];
  int sp = 1;
  stk_a[0] = 0;
  stk_b[0] = 0;
  while (sp > 0) {
    int leaf1 = -1, leaf2 = -1;
    while (sp > 0) {  // phase A: OBB tests
      --sp;
      const int b1 = stk_a[sp], b2 = stk_b[sp];
      const hfb_bvh_node& n1 = q.m1.nodes[b1];
      const hfb_bvh_node& n2 = q.m2.nodes[b2];
      if (n1.first_child < 0 && n2.first_child < 0) {
        leaf1 = -(n1.first_child + 1);
        leaf2 = -(n2.first_child + 1);
        break;
      }
      double sq_lb;
      out.bv_tests++;
      // operand order of the reference (:147-162): (RT, bv of model 2, bv of model 1)
      const bool disjoint =
          !obb_overlap(q.R, q.T, load_node_obb(n2), load_node_obb(n1), security_margin, break_distance, sq_lb);
      if (disjoint) {  // updateDistanceLowerBoundFromBV
        if (out.distance_lower_bound > 0) {
          const double nd_lb = sqrt(sq_lb);
          if (nd_lb < out.distance_lower_bound) out.distance_lower_bound = nd_lb;
        }
        continue;
      }
      if (sp + 2 > HFB_BVH_STACK) {
        sp = 0;
        break;
      }
      if (bvh_first_over_second(n1, n2)) {
        stk_a[sp] = n1.first_child + 1; stk_b[sp] = b2; ++sp;
        stk_a[sp] = n1.first_child; stk_b[sp] = b2; ++sp;
      } else {
        stk_a[sp] = b1; stk_b[sp] = n2.first_child + 1; ++sp;
        stk_a[sp] = b1; stk_b[sp] = n2.first_child; ++sp;
      }
    }
    if (leaf1 < 0) break;
    // phase B: leafCollides (:173-232), ShapeShapeDistance<TriangleP, TriangleP> in world poses
    PairIn in = in0;
    const Tri3 t1 = bvh_triangle(q.m1, leaf1), t2 = bvh_triangle(q.m2, leaf2);
    in.s1.type = in.s2.type = HFB_GEOM_TRIANGLE;
    in.s1.ssr = in.s2.ssr = 0;
    in.s1.p0 = in.s1.p1 = in.s1.p2 = in.s2.p0 = in.s2.p1 = in.s2.p2 = 0;
    in.s1.nv = in.s2.nv = 0;
    in.s1.cx = in.s1.cy = in.s1.cz = in.s2.cx = in.s2.cy = in.s2.cz = nullptr;
    in.s1.center = in.s2.center = mk(0, 0, 0);
    in.s1.ta = t1.v[0]; in.s1.tb = t1.v[1]; in.s1.tc = t1.v[2];
    in.s2.ta = t2.v[0]; in.s2.tb = t2.v[1]; in.s2.tc = t2.v[2];
    in.tf1 = q.tf1;
    in.tf2 = q.tf2;
    PairOut o;
    GjkState g;
    if (pair_phase1<1, CAPS, PATH_BOTH>(in, P, o, g)) pair_phase2<1, CAPS>(in, P, g, ws, o);
    out.leaf_tests++;
    const double d2c = o.distance - security_margin;
    if (d2c < out.distance_lower_bound) {  // updateDistanceLowerBoundFromLeaf
      out.distance_lower_bound = d2c;
      out.lb_p1 = o.p1;
      out.lb_p2 = o.p2;
      out.lb_normal = o.normal;
    }
    if (d2c <= collision_distance_threshold) {
      if (ncontacts < num_max_contacts) {
        if (ncontacts == 0) {
          out.has_contact = true;
          out.b1 = leaf1;
          out.b2 = leaf2;
          out.distance = o.distance;
          out.p1 = o.p1;
          out.p2 = o.p2;
          out.normal = o.normal;
        } else {
          bvh_sink_contact(sink, ncontacts, false, leaf1, leaf2, o.distance, o.p1, o.p2, o.normal);
        }
        ++ncontacts;
      }
    }
    if (ncontacts > 0 && num_max_contacts <= ncontacts) break;  // canStop()
  }
  if (sink.count) *sink.count = ncontacts;
}

// ---- one pair: classification, the (mesh, mesh) walks, and a single-query source -----------------
HFB_HD void bvh_unsupported_distance(hfb_distance_result* r) {
  r->min_distance = DBL_MAX;
  put3d(r->p1, nan3());
  put3d(r->p2, nan3());
  put3d(r->normal, nan3());
  r->b1 = r->b2 = -1;
  r->status = pack_status(0, 0, HFB_PATH_UNSUPPORTED);
  r->iterations = 0;
}

struct BvhReq {  // request fields the traversals need beyond SolverP
  double rel_err, abs_err;               // DistanceRequest
  double security_margin, break_distance, collision_distance_threshold;  // CollisionRequest
  unsigned num_max_contacts;
  bool enable_nearest_points;  // DistanceRequest, mesh-mesh only
  int initial_guess;           // QueryRequest::gjk_initial_guess (see bvh_leaf_guess_throws)
};


HFB_HD BvhPairQuery bvh_make_pair_query(const ArenaView& A, uint32_t h1, const xf& tf1, uint32_t h2, const xf& tf2) {
  BvhPairQuery pq;
  pq.m1 = bvh_mesh_view(A, A.shapes[h1].data);
  pq.m2 = bvh_mesh_view(A, A.shapes[h2].data);
  pq.tf1 = tf1;
  pq.tf2 = tf2;
  pq.R = mtmulm(tf1.R, tf2.R);
  pq.T = mtmul(tf1.R, tf2.T - tf1.T);
  return pq;
}

// distance() of a (mesh, mesh) pair: BVHDistance<OBBRSS> (distance_func_matrix.cpp:259-268)
HFB_HD void bvh_mesh_pair_distance(const ArenaView& A, uint32_t h1, const xf& tf1, uint32_t h2, const xf& tf2,
                                   const BvhReq& R, hfb_distance_result* r, unsigned& bv_tests,
                                   unsigned& leaf_tests) {
  if (A.shapes[h1].type != HFB_BV_OBBRSS || A.shapes[h2].type != HFB_BV_OBBRSS) {  // plain OBB models: collide() only
    bvh_unsupported_distance(r);
    bv_tests = leaf_tests = 0;
    return;
  }
  const BvhPairQuery pq = bvh_make_pair_query(A, h1, tf1, h2, tf2);
  BvhPairDistOut o;
  bvh_bvh_distance(pq, R.rel_err, R.abs_err, R.enable_nearest_points, o);
  r->min_distance = o.min_distance;
  put3d(r->p1, o.p1);
  put3d(r->p2, o.p2);
  put3d(r->normal, nan3());
  r->b1 = o.b1;
  r->b2 = o.b2;
  r->status = pack_status(0, 0, HFB_PATH_BVH);
  r->iterations = (o.bv_tests & 0xffffu) | ((o.leaf_tests & 0xffffu) << 16);
  bv_tests = o.bv_tests;
  leaf_tests = o.leaf_tests;
}

// collide() of a (mesh, mesh) pair: BVHCollide<OBBRSS> (collision_func_matrix.cpp:248-257)
template <int CAPS>
HFB_HD void bvh_mesh_pair_collide(const ArenaView& A, uint32_t h1, const xf& tf1, uint32_t h2, const xf& tf2,
                                  const SolverP& P, const BvhReq& R, v3 cached_guess, int hint0, int hint1,
                                  EpaWs* ws, hfb_contact* r, unsigned& bv_tests, unsigned& leaf_tests,
                                  BvhContactSink sink = BvhContactSink{nullptr, 0, nullptr}) {
  if (A.shapes[h1].type != A.shapes[h2].type) {  // collision_matrix has no [BV_OBB][BV_OBBRSS] entry
    bvh_init_contact(r);
    r->status = pack_status(0, 0, HFB_PATH_UNSUPPORTED);
    if (sink.count) *sink.count = 0;
    bv_tests = leaf_tests = 0;
    return;
  }
  const BvhPairQuery pq = bvh_make_pair_query(A, h1, tf1, h2, tf2);
  PairIn in;
  in.cached_guess = cached_guess;
  in.hint0 = hint0;
  in.hint1 = hint1;
  BvhPairColOut o;
  bvh_bvh_collide<CAPS>(pq, P, R.security_margin, R.break_distance, R.collision_distance_threshold,
                        R.num_max_contacts, ws, in, o, sink);
  bvh_init_contact(r);
  r->distance_lower_bound = o.distance_lower_bound;
  put3d(r->p1, o.lb_p1);
  put3d(r->p2, o.lb_p2);
  put3d(r->normal, o.lb_normal);
  if (o.has_contact) {
    r->num_contacts = 1;
    r->distance = o.distance;
    r->b1 = o.b1;
    r->b2 = o.b2;
    put3d(r->pos, (o.p1 + o.p2) / 2);
    put3d(r->p1, o.p1);
    put3d(r->p2, o.p2);
    put3d(r->normal, o.normal);
  }
  r->status = pack_status(0, 0, HFB_PATH_BVH);
  r->iterations = (o.bv_tests & 0xffffu) | ((o.leaf_tests & 0xffffu) << 16);
  bv_tests = o.bv_tests;
  leaf_tests = o.leaf_tests;
}

// Turns pair (h1, tf1, h2, tf2) into a (mesh, shape) job.  Returns false -- with the record already
// written -- when there is nothing to walk: unsupported partner (the reference throws), or, for
// collide(), a negative security margin (collision_func_matrix.cpp:109-112).
template <int CAPS, int MODE>
HFB_HD bool bvh_make_job(const ArenaView& A, uint32_t h1, const xf& tf1, uint32_t h2, const xf& tf2, const BvhReq& R,
                         v3 cached_guess, int hint0, int hint1, void* rec, BvhJob& job) {
  bool ok = bvh_make_query<CAPS>(A, h1, tf1, h2, tf2, job.q, job.swapped);
  if (MODE == 1 && R.security_margin < 0) ok = false;
  if (MODE == 0 && ok && job.q.plain_obb) ok = false;  // no distance() on a plain OBB model
  // distance(): preprocess() always evaluates the seed triangle, so the throw is certain
  if (MODE == 0 && ok && bvh_leaf_guess_throws(R.initial_guess, job.q.shape)) ok = false;
  if (!ok) {
    if (MODE == 0) {
      bvh_unsupported_distance(static_cast<hfb_distance_result*>(rec));
    } else {
      bvh_init_contact(static_cast<hfb_contact*>(rec));
      static_cast<hfb_contact*>(rec)->status = pack_status(0, 0, HFB_PATH_UNSUPPORTED);
    }
    return false;
  }
  job.cached_guess = cached_guess;
  job.hint0 = hint0;
  job.hint1 = hint1;
  job.rec = rec;
  return true;
}

// pair kinds a k_bvh instantiation serves
enum { BVK_SHAPE = 1, BVK_MESH = 2 };

template <class Job>
struct BvhSingleSrcT {  // a source holding one job (the CPU emulation of the device code, tests)
  Job job;
  bool pending;
  HFB_HD bool next(Job& j) {
    if (!pending) return false;
    pending = false;
    j = job;
    return true;
  }
};
typedef BvhSingleSrcT<BvhJob> BvhSingleSrc;
typedef BvhSingleSrcT<BvhColJob> BvhSingleColSrc;

}  // namespace hfb
