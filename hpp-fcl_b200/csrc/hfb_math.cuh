// FP64 3-vector arithmetic for the narrow-phase kernels.
//
// Parity contract (DESIGN.md "floating point"): every reduction is evaluated
// left to right, (x*x + y*y) + z*z, with no FMA contraction (nvcc -fmad=false)
// and IEEE div/sqrt -- the operation order Eigen >= 3.3 emits on x86-64 for the
// reference's fixed 3-vectors (Vec3f/Matrix3f of include/hpp/fcl/data_types.h).
#pragma once
#include <float.h>
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define HFB_HD __host__ __device__ __forceinline__
#define HFB_D __device__ __forceinline__
// out-of-line on the device: multi-call-site helpers that run once per pair; inlining
// them multiplies the kernel's code size (instruction-cache misses then dominate k_pairs)
#define HFB_HD_NOINLINE __host__ __device__ __noinline__ inline
#else
#define HFB_HD inline
#define HFB_D inline
#define HFB_HD_NOINLINE inline
#endif

namespace hfb {

struct v3 {
  double x, y, z;
};

HFB_HD v3 mk(double x, double y, double z) {
  v3 r;
  r.x = x;
  r.y = y;
  r.z = z;
  return r;
}
HFB_HD v3 operator+(v3 a, v3 b) { return mk(a.x + b.x, a.y + b.y, a.z + b.z); }
HFB_HD v3 operator-(v3 a, v3 b) { return mk(a.x - b.x, a.y - b.y, a.z - b.z); }
HFB_HD v3 operator-(v3 a) { return mk(-a.x, -a.y, -a.z); }
HFB_HD v3 operator*(double s, v3 a) { return mk(s * a.x, s * a.y, s * a.z); }
HFB_HD v3 operator*(v3 a, double s) { return mk(a.x * s, a.y * s, a.z * s); }
HFB_HD v3 operator/(v3 a, double s) { return mk(a.x / s, a.y / s, a.z / s); }
HFB_HD double dot(v3 a, v3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
HFB_HD double sqn(v3 a) { return dot(a, a); }
HFB_HD double nrm(v3 a) { return sqrt(sqn(a)); }
HFB_HD v3 cross(v3 a, v3 b) {
  return mk(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
// Eigen normalized(): divide by sqrt(squaredNorm) iff squaredNorm > 0
HFB_HD v3 unit(v3 a) {
  double z = sqn(a);
  if (z > 0) return a / sqrt(z);
  return a;
}
HFB_HD double triple(v3 a, v3 b, v3 c) { return dot(a, cross(b, c)); }
HFB_HD bool is_zero(v3 a, double prec) {
  return fabs(a.x) <= prec && fabs(a.y) <= prec && fabs(a.z) <= prec;
}
HFB_HD v3 nan3() {
#if defined(__CUDA_ARCH__)
  double q = __longlong_as_double(0x7ff8000000000000LL);
#else
  double q = NAN;
#endif
  return mk(q, q, q);
}
HFB_HD double comp(v3 a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }
HFB_HD v3 sel(bool c, v3 a, v3 b) { return c ? a : b; }

// 3x3 matrix held as rows r0,r1,r2 (element (i,j) = row i, component j)
struct m3 {
  v3 r0, r1, r2;
};
HFB_HD v3 mcol(const m3& A, int c) { return mk(comp(A.r0, c), comp(A.r1, c), comp(A.r2, c)); }
HFB_HD v3 mmul(const m3& A, v3 v) { return mk(dot(A.r0, v), dot(A.r1, v), dot(A.r2, v)); }
// A^T * v : component j = (A00*v0 + A10*v1) + A20*v2 for column j
HFB_HD v3 mtmul(const m3& A, v3 v) {
  return mk((A.r0.x * v.x + A.r1.x * v.y) + A.r2.x * v.z, (A.r0.y * v.x + A.r1.y * v.y) + A.r2.y * v.z,
            (A.r0.z * v.x + A.r1.z * v.y) + A.r2.z * v.z);
}
// A^T * B
HFB_HD m3 mtmulm(const m3& A, const m3& B) {
  m3 C;
  // row i of C = sum_k A[k][i] * B[k][:]
  C.r0 = mk((A.r0.x * B.r0.x + A.r1.x * B.r1.x) + A.r2.x * B.r2.x,
            (A.r0.x * B.r0.y + A.r1.x * B.r1.y) + A.r2.x * B.r2.y,
            (A.r0.x * B.r0.z + A.r1.x * B.r1.z) + A.r2.x * B.r2.z);
  C.r1 = mk((A.r0.y * B.r0.x + A.r1.y * B.r1.x) + A.r2.y * B.r2.x,
            (A.r0.y * B.r0.y + A.r1.y * B.r1.y) + A.r2.y * B.r2.y,
            (A.r0.y * B.r0.z + A.r1.y * B.r1.z) + A.r2.y * B.r2.z);
  C.r2 = mk((A.r0.z * B.r0.x + A.r1.z * B.r1.x) + A.r2.z * B.r2.x,
            (A.r0.z * B.r0.y + A.r1.z * B.r1.y) + A.r2.z * B.r2.y,
            (A.r0.z * B.r0.z + A.r1.z * B.r1.z) + A.r2.z * B.r2.z);
  return C;
}
// Eigen isIdentity(prec): diagonal isApprox 1, off-diagonal isMuchSmallerThan 1
HFB_HD bool is_identity(const m3& A, double prec) {
  bool ok = true;
  ok = ok && (fabs(A.r0.x - 1.0) <= fmin(fabs(A.r0.x), 1.0) * prec);
  ok = ok && (fabs(A.r1.y - 1.0) <= fmin(fabs(A.r1.y), 1.0) * prec);
  ok = ok && (fabs(A.r2.z - 1.0) <= fmin(fabs(A.r2.z), 1.0) * prec);
  ok = ok && (fabs(A.r0.y) <= prec) && (fabs(A.r0.z) <= prec);
  ok = ok && (fabs(A.r1.x) <= prec) && (fabs(A.r1.z) <= prec);
  ok = ok && (fabs(A.r2.x) <= prec) && (fabs(A.r2.y) <= prec);
  return ok;
}

// Transform3f (math/transform.h:56-216): R (held as rows) and T
struct xf {
  m3 R;
  v3 T;
};
HFB_HD v3 xform(const xf& t, v3 v) { return mmul(t.R, v) + t.T; }  // R*v + T
// load from the column-major POD (hfb_transform)
HFB_HD xf load_xf(const double* p) {
  xf t;
  t.R.r0 = mk(p[0], p[3], p[6]);
  t.R.r1 = mk(p[1], p[4], p[7]);
  t.R.r2 = mk(p[2], p[5], p[8]);
  t.T = mk(p[9], p[10], p[11]);
  return t;
}

}  // namespace hfb
