// Forward kinematics of a robot model (hfb_robot_*, include/hppfcl_b200.h): the joint frames, the link poses, the
// linear-in-q motion samples and the sweep bounds, as HFB_HD functions that the kernel (hfb_robot.cu) and the host
// emulation (tests/emu/kin_emu.cpp) share.  Every result is built from IEEE + - * / and sqrt in a fixed order, with no
// contraction (nvcc -fmad=false, g++ -ffp-contract=off), so the device and the host give the same bits.
#pragma once
#include <string.h>

#include "hfb_math.cuh"
#include "../../include/hppfcl_b200.h"

namespace hfb {

// ---- sin and cos -------------------------------------------------------------------------------------------------
// fdlibm 5.3's __ieee754_rem_pio2 (medium arguments), __kernel_sin and __kernel_cos (Sun Microsystems, freely
// redistributable), restated: CUDA's sin and glibc's differ in the last bits, so neither can serve both sides.
// Error: below 1 ulp for |x| <= 2^20 * pi/2 (about 1.647e6 rad), the range fdlibm's three-step Cody-Waite reduction
// covers.  Beyond it, and for +-inf and NaN, both results are NaN: a joint angle there has no use, and a NaN pose is
// handled by the narrow phase's rules for non-finite input.  sin(+-0) = +-0, cos(+-0) = 1.
HFB_HD uint32_t kin_hi32(double x) {
#if defined(__CUDA_ARCH__)
  return (uint32_t)__double2hiint(x);
#else
  uint64_t u;
  memcpy(&u, &x, 8);
  return (uint32_t)(u >> 32);
#endif
}
HFB_HD double kin_from_hi32(uint32_t hi) {  // the double with high word `hi` and low word 0
#if defined(__CUDA_ARCH__)
  return __hiloint2double((int)hi, 0);
#else
  const uint64_t u = (uint64_t)hi << 32;
  double x;
  memcpy(&x, &u, 8);
  return x;
#endif
}

HFB_HD double kin_ksin(double x, double y, int iy) {  // sin(x + y), |x| <= pi/4, y the tail of the reduced argument
  const double S1 = -0x1.5555555555549p-3, S2 = 0x1.111111110f8a6p-7, S3 = -0x1.a01a019c161d5p-13,
               S4 = 0x1.71de357b1fe7dp-19, S5 = -0x1.ae5e68a2b9cebp-26, S6 = 0x1.5d93a5acfd57cp-33;
  if ((kin_hi32(x) & 0x7fffffffu) < 0x3e400000u) return x;  // |x| < 2^-27 (keeps the sign of 0)
  const double z = x * x;
  const double v = z * x;
  const double r = S2 + z * (S3 + z * (S4 + z * (S5 + z * S6)));
  if (iy == 0) return x + v * (S1 + z * r);
  return x - ((z * (0.5 * y - v * r) - y) - v * S1);
}

HFB_HD double kin_kcos(double x, double y) {  // cos(x + y), |x| <= pi/4
  const double C1 = 0x1.555555555554cp-5, C2 = -0x1.6c16c16c15177p-10, C3 = 0x1.a01a019cb1590p-16,
               C4 = -0x1.27e4f809c52adp-22, C5 = 0x1.1ee9ebdb4b1c4p-29, C6 = -0x1.8fae9be8838d4p-37;
  const uint32_t ix = kin_hi32(x) & 0x7fffffffu;
  if (ix < 0x3e400000u) return 1.0;  // |x| < 2^-27
  const double z = x * x;
  const double r = z * (C1 + z * (C2 + z * (C3 + z * (C4 + z * (C5 + z * C6)))));
  if (ix < 0x3FD33333u) return 1.0 - (0.5 * z - (z * r - x * y));  // |x| < 0.3
  const double qx = ix > 0x3fe90000u ? 0.28125 : kin_from_hi32(ix - 0x00200000u);  // x/4 truncated
  const double hz = 0.5 * z - qx;
  const double a = 1.0 - qx;
  return a - (hz - (z * r - x * y));
}

// x = n * pi/2 + (y0 + y1), |y0 + y1| <= pi/4, for pi/4 < |x| <= 2^20 * pi/2; returns n
HFB_HD int kin_rem_pio2(double x, double& y0, double& y1) {
  const double invpio2 = 0x1.45f306dc9c883p-1;
  const double pio2_1 = 0x1.921fb54400000p+0, pio2_1t = 0x1.0b4611a626331p-34;  // first 33 bits of pi/2, the rest
  const double pio2_2 = 0x1.0b4611a600000p-34, pio2_2t = 0x1.3198a2e037073p-69;  // next 33 bits, the rest
  const double pio2_3 = 0x1.3198a2e000000p-69, pio2_3t = 0x1.b839a252049c1p-104;  // next 33 bits, the rest
  const bool neg = x < 0;
  const double t = neg ? -x : x;
  const int n = (int)(t * invpio2 + 0.5);
  const double fn = (double)n;
  double r = t - fn * pio2_1;
  double w = fn * pio2_1t;  // first round: good to 85 bits
  const int j = (int)(kin_hi32(t) >> 20);
  y0 = r - w;
  if (j - (int)((kin_hi32(y0) >> 20) & 0x7ff) > 16) {  // cancellation: a second round, good to 118 bits
    double u = r;
    w = fn * pio2_2;
    r = u - w;
    w = fn * pio2_2t - ((u - r) - w);
    y0 = r - w;
    if (j - (int)((kin_hi32(y0) >> 20) & 0x7ff) > 49) {  // a third, 151 bits: covers every double in range
      u = r;
      w = fn * pio2_3;
      r = u - w;
      w = fn * pio2_3t - ((u - r) - w);
      y0 = r - w;
    }
  }
  y1 = (r - y0) - w;
  if (neg) {
    y0 = -y0;
    y1 = -y1;
    return -n;
  }
  return n;
}

HFB_HD void hfb_sincos(double x, double* s, double* c) {
  const uint32_t ix = kin_hi32(x) & 0x7fffffffu;
  if (ix <= 0x3fe921fbu) {  // |x| <= pi/4 (and NaN-free)
    *s = kin_ksin(x, 0.0, 0);
    *c = kin_kcos(x, 0.0);
    return;
  }
  if (ix > 0x413921fbu) {  // |x| > 2^20 * pi/2, +-inf, NaN
    *s = *c = NAN;
    return;
  }
  double y0, y1;
  const int n = kin_rem_pio2(x, y0, y1);
  const double ks = kin_ksin(y0, y1, 1), kc = kin_kcos(y0, y1);
  switch (n & 3) {
    case 0: *s = ks; *c = kc; break;
    case 1: *s = kc; *c = -ks; break;
    case 2: *s = -ks; *c = -kc; break;
    default: *s = -kc; *c = ks; break;
  }
}

// ---- the model on the device ----------------------------------------------------------------------------------------
struct KinJoint {
  double R[9], T[3];  // placement: the joint frame in its parent's at q = 0 (R column-major, as hfb_transform)
  double axis[3];     // unit
  double tnorm;       // |placement.T|
  int32_t parent;     // -1: the world
  uint32_t type;      // HFB_JOINT_*
};
struct KinLink {
  double R[9], T[3];  // link_placement
  double reach;       // |link_placement.T| + r, r the largest corner norm of the geometry's local box (+inf: unbounded)
  int32_t joint;      // -1: fixed to the world
  uint32_t path;      // the joints from the root down to `joint`: path_list[path .. path + depth)
  uint32_t depth;
  uint32_t handle;
};

HFB_HD double kin_norm3(const double* v) { return sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]); }

// r of a local box (mn[3], mx[3]): the largest norm of its corners, +inf when it is not finite
HFB_HD double kin_box_radius(const double* box) {
  double a[3];
  for (int k = 0; k < 3; ++k) {
    const double lo = fabs(box[k]), hi = fabs(box[3 + k]);
    if (!(lo <= DBL_MAX && hi <= DBL_MAX)) return INFINITY;
    a[k] = lo > hi ? lo : hi;
  }
  return kin_norm3(a);
}

// |link_placement.T| + r(local box): the reach of a link's points from its joint's origin
HFB_HD double kin_link_reach(const KinLink& k, const double* box) { return kin_norm3(k.T) + kin_box_radius(box); }

// Checks a robot description without allocating: the counts (1 <= J <= 64, L >= 1, L * J <= UINT32_MAX, so that
// every link's path offset i * J fits in 32 bits), the parents, the types, the axes and the link joints.  Returns a
// message for a malformed description, nullptr when it is well formed.  The pointers and the geometry handles are the
// caller's to check.
inline const char* kin_check(const hfb_robot_desc* d) {
  const uint32_t J = d->num_joints, L = d->num_links;
  if (J == 0 || J > 64) return "num_joints must be 1..64";
  if (L == 0) return "num_links must be >= 1";
  if ((uint64_t)L * J > 0xffffffffull) return "num_links * num_joints >= 2^32";
  for (uint32_t j = 0; j < J; ++j) {
    if (d->parent[j] < -1 || d->parent[j] >= (int32_t)j) return "a joint's parent is not -1 or an earlier joint";
    if (d->type[j] != HFB_JOINT_REVOLUTE && d->type[j] != HFB_JOINT_PRISMATIC) return "unknown joint type";
    const double n = kin_norm3(d->axis + 3 * j);
    if (!(n > 0 && n <= DBL_MAX)) return "a joint axis is zero or not finite";
  }
  for (uint32_t i = 0; i < L; ++i)
    if (d->link_joint[i] < -1 || d->link_joint[i] >= (int32_t)J) return "a link's joint is not -1 or a joint index";
  return nullptr;
}

// Lays a description that kin_check accepted out for the kernel: joints[J], links[L], path_list[L * J] (uint8 joint
// indices).  local_boxes: the L links' local boxes (6 doubles each, hfb_geom_commit's aabb_local), or null (reach is
// then NaN, to be set by kin_link_reach).
inline void kin_prepare(const hfb_robot_desc* d, const double* local_boxes, KinJoint* joints, KinLink* links,
                        uint8_t* path_list) {
  const uint32_t J = d->num_joints, L = d->num_links;
  for (uint32_t j = 0; j < J; ++j) {
    KinJoint& k = joints[j];
    const double* ax = d->axis + 3 * j;
    const double n = kin_norm3(ax);
    for (int c = 0; c < 3; ++c) k.axis[c] = ax[c] / n;
    memcpy(k.R, d->placement[j].R, sizeof k.R);
    memcpy(k.T, d->placement[j].T, sizeof k.T);
    k.tnorm = kin_norm3(k.T);
    k.parent = d->parent[j];
    k.type = d->type[j];
  }
  for (uint32_t i = 0; i < L; ++i) {
    KinLink& k = links[i];
    const int32_t lj = d->link_joint[i];
    memcpy(k.R, d->link_placement[i].R, sizeof k.R);
    memcpy(k.T, d->link_placement[i].T, sizeof k.T);
    k.reach = local_boxes ? kin_link_reach(k, local_boxes + 6 * (size_t)i) : NAN;
    k.joint = lj;
    k.path = i * J;
    k.handle = d->link_handles[i];
    uint32_t depth = 0;
    for (int32_t j = lj; j >= 0; j = d->parent[j]) ++depth;
    k.depth = depth;
    uint32_t p = depth;
    for (int32_t j = lj; j >= 0; j = d->parent[j]) path_list[k.path + --p] = (uint8_t)j;
  }
}

// ---- frames -------------------------------------------------------------------------------------------------------
struct KinTf {
  double R[9], T[3];
};

// A o B (R = A.R B.R, T = A.R B.T + A.T), every entry summed left to right
HFB_HD void kin_compose(const double* AR, const double* AT, const double* BR, const double* BT, KinTf& o) {
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r)
      o.R[3 * c + r] = (AR[r] * BR[3 * c] + AR[3 + r] * BR[3 * c + 1]) + AR[6 + r] * BR[3 * c + 2];
  for (int r = 0; r < 3; ++r) o.T[r] = ((AR[r] * BT[0] + AR[3 + r] * BT[1]) + AR[6 + r] * BT[2]) + AT[r];
}

// M_j = M_parent o placement_j o X_j(q); `parent` null for a joint on the world
HFB_HD void kin_joint_frame(const KinJoint& jt, const KinTf* parent, double q, KinTf& m) {
  KinTf p;
  if (parent) {
    kin_compose(parent->R, parent->T, jt.R, jt.T, p);
  } else {
    for (int k = 0; k < 9; ++k) p.R[k] = jt.R[k];
    for (int k = 0; k < 3; ++k) p.T[k] = jt.T[k];
  }
  const double* a = jt.axis;
  if (jt.type == HFB_JOINT_PRISMATIC) {
    const double v[3] = {q * a[0], q * a[1], q * a[2]};
    for (int k = 0; k < 9; ++k) m.R[k] = p.R[k];
    for (int r = 0; r < 3; ++r) m.T[r] = ((p.R[r] * v[0] + p.R[3 + r] * v[1]) + p.R[6 + r] * v[2]) + p.T[r];
    return;
  }
  // Rodrigues: X = c I + s [a]x + (1 - c) a a^T
  double s, c;
  hfb_sincos(q, &s, &c);
  const double t = 1.0 - c;
  double X[9];
  X[0] = t * a[0] * a[0] + c;
  X[4] = t * a[1] * a[1] + c;
  X[8] = t * a[2] * a[2] + c;
  X[1] = t * a[0] * a[1] + s * a[2];  // (1, 0)
  X[3] = t * a[0] * a[1] - s * a[2];  // (0, 1)
  X[2] = t * a[0] * a[2] - s * a[1];  // (2, 0)
  X[6] = t * a[0] * a[2] + s * a[1];  // (0, 2)
  X[5] = t * a[1] * a[2] + s * a[0];  // (2, 1)
  X[7] = t * a[1] * a[2] - s * a[0];  // (1, 2)
  for (int cc = 0; cc < 3; ++cc)
    for (int r = 0; r < 3; ++r)
      m.R[3 * cc + r] = (p.R[r] * X[3 * cc] + p.R[3 + r] * X[3 * cc + 1]) + p.R[6 + r] * X[3 * cc + 2];
  for (int r = 0; r < 3; ++r) m.T[r] = p.T[r];
}

// sample k of an n-sample motion from q_from to q_to: q_from at k = 0, q_to at k = n - 1, and
// q_from + (k / (n - 1)) * (q_to - q_from) in between (OMPL's RealVectorStateSpace::interpolate)
HFB_HD double kin_sample(double from, double to, uint32_t k, uint32_t n) {
  if (k == 0) return from;
  if (k + 1 == n) return to;
  const double t = (double)k / (double)(n - 1);
  return from + t * (to - from);
}

// The pose of link `link` at the joint values q(j) (j < J): the frames of its path, root first.
template <class Q>
HFB_HD void kin_link_pose(const KinJoint* joints, const KinLink& link, const uint8_t* path_list, const Q& q,
                          hfb_transform& out) {
  if (link.joint < 0) {
    for (int k = 0; k < 9; ++k) out.R[k] = link.R[k];
    for (int k = 0; k < 3; ++k) out.T[k] = link.T[k];
    return;
  }
  KinTf m;
  for (uint32_t p = 0; p < link.depth; ++p) {
    const uint32_t j = path_list[link.path + p];
    if (p == 0) {
      kin_joint_frame(joints[j], nullptr, q(j), m);
    } else {
      const KinTf parent = m;
      kin_joint_frame(joints[j], &parent, q(j), m);
    }
  }
  KinTf o;
  kin_compose(m.R, m.T, link.R, link.T, o);
  for (int k = 0; k < 9; ++k) out.R[k] = o.R[k];
  for (int k = 0; k < 3; ++k) out.T[k] = o.T[k];
}

// The sweep bound of link `link` over a segment from joint values q0(j) to q1(j), linear in q:
//   s = sum over the joints k of its path of |dq_k| * rho_k, walked from the link up to the root, where rho_k = 1 for a
//   prismatic k, and for a revolute k the bound on a link point's distance to k's origin: acc, which starts at
//   link.reach and grows past each joint j by |placement_j.T| and, for a prismatic j, by max(|q0_j|, |q1_j|).
// A joint that does not move adds nothing (also when rho is +inf).  The sum is rounded up by a relative margin of
// 2^-46 * J, far above its rounding error (at most about (2 J + 8) * 2^-53 relative: every term is >= 0), then to the
// next double.  0 when nothing moves; NaN when a q is NaN.
template <class Q0, class Q1>
HFB_HD double kin_link_sweep(const KinJoint* joints, const KinLink& link, const uint8_t* path_list, uint32_t J,
                             const Q0& q0, const Q1& q1) {
  double s = 0.0, acc = link.reach;
  for (uint32_t p = link.depth; p-- > 0;) {
    const uint32_t j = path_list[link.path + p];
    const KinJoint& jt = joints[j];
    const double a = q0(j), b = q1(j);
    const double d = fabs(b - a);
    const bool prism = jt.type == HFB_JOINT_PRISMATIC;
    if (!(d == 0)) s = s + (prism ? d : d * acc);
    acc = acc + jt.tnorm;
    if (prism) {
      const double fa = fabs(a), fb = fabs(b);
      acc = acc + (fa > fb ? fa : fb);
    }
  }
  if (s == 0) return 0.0;
  s = s * (1.0 + (double)J * 0x1p-46);
  return nextafter(s, (double)INFINITY);
}

}  // namespace hfb
