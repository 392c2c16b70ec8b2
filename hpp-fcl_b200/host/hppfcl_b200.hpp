// C++ host-side mirror of the hpp-fcl query interface for the accelerated hot
// path, above the C-ABI of include/hppfcl_b200.h.  Header-only, C++17, no Eigen.
//
// Same names, argument meaning and error behaviour as the reference:
//   collide(o1, tf1, o2, tf2, CollisionRequest, CollisionResult&)   include/hpp/fcl/collision.h:65-70
//   distance(o1, tf1, o2, tf2, DistanceRequest, DistanceResult&)    include/hpp/fcl/distance.h:60-65
//   ComputeCollision / ComputeDistance functors                     collision.h:79-117, distance.h:74-112
//   CollisionRequest/Result, DistanceRequest/Result, Contact        include/hpp/fcl/collision_data.h
//   shapes (Box, Sphere, Capsule, Cone, Cylinder, Ellipsoid,
//           ConvexBase, TriangleP)                                  include/hpp/fcl/shape/geometric_shapes.h
// plus the batched form (`BatchNarrowPhase`) a broadphase pair collector
// (CollisionCallBackCollect, broadphase/default_broadphase_callbacks.h:224-252)
// feeds.  Every query runs on the GPU; unsupported pairs and invalid requests
// throw std::invalid_argument like HPP_FCL_THROW_PRETTY does (fwd.hh:63-72).
#pragma once
#include <array>
#include <algorithm>
#include <cmath>
#include <limits>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/hppfcl_b200.h"

namespace hppfcl_b200 {

typedef double FCL_REAL;

struct Vec3f {
  FCL_REAL v[3];
  Vec3f() : v{0, 0, 0} {}
  Vec3f(FCL_REAL x, FCL_REAL y, FCL_REAL z) : v{x, y, z} {}
  FCL_REAL& operator[](int i) { return v[i]; }
  FCL_REAL operator[](int i) const { return v[i]; }
  static Vec3f Constant(FCL_REAL c) { return Vec3f(c, c, c); }
  FCL_REAL norm() const { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }
};
inline Vec3f operator+(const Vec3f& a, const Vec3f& b) { return Vec3f(a[0] + b[0], a[1] + b[1], a[2] + b[2]); }
inline Vec3f operator-(const Vec3f& a, const Vec3f& b) { return Vec3f(a[0] - b[0], a[1] - b[1], a[2] - b[2]); }
inline Vec3f operator*(FCL_REAL s, const Vec3f& a) { return Vec3f(s * a[0], s * a[1], s * a[2]); }

// column-major 3x3 like Eigen::Matrix3d
struct Matrix3f {
  FCL_REAL m[9];
  Matrix3f() : m{1, 0, 0, 0, 1, 0, 0, 0, 1} {}
  FCL_REAL& operator()(int r, int c) { return m[c * 3 + r]; }
  FCL_REAL operator()(int r, int c) const { return m[c * 3 + r]; }
  static Matrix3f Identity() { return Matrix3f(); }
};
inline Vec3f operator*(const Matrix3f& R, const Vec3f& x) {
  return Vec3f(R(0, 0) * x[0] + R(0, 1) * x[1] + R(0, 2) * x[2], R(1, 0) * x[0] + R(1, 1) * x[1] + R(1, 2) * x[2],
               R(2, 0) * x[0] + R(2, 1) * x[1] + R(2, 2) * x[2]);
}
inline Matrix3f operator*(const Matrix3f& A, const Matrix3f& B) {
  Matrix3f C;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C(i, j) = A(i, 0) * B(0, j) + A(i, 1) * B(1, j) + A(i, 2) * B(2, j);
  return C;
}

struct Quatf {
  FCL_REAL w, x, y, z;
  Quatf(FCL_REAL w_, FCL_REAL x_, FCL_REAL y_, FCL_REAL z_) : w(w_), x(x_), y(y_), z(z_) {}
  Matrix3f toRotationMatrix() const {
    Matrix3f R;
    R(0, 0) = 1 - 2 * (y * y + z * z); R(0, 1) = 2 * (x * y - z * w); R(0, 2) = 2 * (x * z + y * w);
    R(1, 0) = 2 * (x * y + z * w); R(1, 1) = 1 - 2 * (x * x + z * z); R(1, 2) = 2 * (y * z - x * w);
    R(2, 0) = 2 * (x * z - y * w); R(2, 1) = 2 * (y * z + x * w); R(2, 2) = 1 - 2 * (x * x + y * y);
    return R;
  }
};
inline Quatf makeQuat(FCL_REAL w, FCL_REAL x, FCL_REAL y, FCL_REAL z) { return Quatf(w, x, y, z); }

// math/transform.h:56-216
class Transform3f {
  Matrix3f R;
  Vec3f T;

 public:
  Transform3f() {}
  Transform3f(const Matrix3f& R_, const Vec3f& T_) : R(R_), T(T_) {}
  Transform3f(const Quatf& q, const Vec3f& T_) : R(q.toRotationMatrix()), T(T_) {}
  explicit Transform3f(const Vec3f& T_) : T(T_) {}
  const Vec3f& getTranslation() const { return T; }
  const Matrix3f& getRotation() const { return R; }
  void setTranslation(const Vec3f& t) { T = t; }
  void setRotation(const Matrix3f& r) { R = r; }
  void setQuatRotation(const Quatf& q) { R = q.toRotationMatrix(); }
  Vec3f transform(const Vec3f& v) const { return R * v + T; }
  Transform3f operator*(const Transform3f& o) const { return Transform3f(R * o.R, R * o.T + T); }
  hfb_transform pod() const {
    hfb_transform t;
    for (int i = 0; i < 9; ++i) t.R[i] = R.m[i];
    for (int i = 0; i < 3; ++i) t.T[i] = T[i];
    return t;
  }
};

// ------------------------------------------------------------------ geometry --
enum NODE_TYPE {  // collision_object.h:65-89 (subset)
  GEOM_BOX = HFB_GEOM_BOX, GEOM_SPHERE = HFB_GEOM_SPHERE, GEOM_CAPSULE = HFB_GEOM_CAPSULE,
  GEOM_CONE = HFB_GEOM_CONE, GEOM_CYLINDER = HFB_GEOM_CYLINDER, GEOM_CONVEX = HFB_GEOM_CONVEX,
  GEOM_PLANE = HFB_GEOM_PLANE, GEOM_HALFSPACE = HFB_GEOM_HALFSPACE, GEOM_TRIANGLE = HFB_GEOM_TRIANGLE,
  GEOM_ELLIPSOID = HFB_GEOM_ELLIPSOID, BV_OBB = HFB_BV_OBB, BV_OBBRSS = HFB_BV_OBBRSS
};

class CollisionGeometry {
 public:
  virtual ~CollisionGeometry() {}
  virtual NODE_TYPE getNodeType() const = 0;
  // flattening hooks used by the arena
  virtual void params(double p[3]) const { p[0] = p[1] = p[2] = 0; }
  virtual const std::vector<Vec3f>* vertices() const { return nullptr; }
  // triangle meshes: flattened tree + geometry (null for shapes)
  struct MeshData {
    const std::vector<hfb_bvh_node>* nodes;
    const std::vector<double>* verts;
    const std::vector<uint32_t>* tris;
  };
  virtual bool mesh(MeshData&) const { return false; }
  // Plane / Halfspace: unit normal and offset (the 40-byte record has no room for them)
  virtual bool plane(double /*n_d*/[4]) const { return false; }
};

class ShapeBase : public CollisionGeometry {  // geometric_shapes.h:59-102
 public:
  void setSweptSphereRadius(FCL_REAL radius) {
    if (radius < 0) throw std::invalid_argument("Swept-sphere radius must be positive.");
    m_swept_sphere_radius = radius;
  }
  FCL_REAL getSweptSphereRadius() const { return m_swept_sphere_radius; }

 protected:
  FCL_REAL m_swept_sphere_radius{0};
};

class Box : public ShapeBase {  // :164-236
 public:
  Box(FCL_REAL x, FCL_REAL y, FCL_REAL z) : halfSide(x / 2, y / 2, z / 2) {}
  Vec3f halfSide;
  NODE_TYPE getNodeType() const override { return GEOM_BOX; }
  void params(double p[3]) const override { p[0] = halfSide[0]; p[1] = halfSide[1]; p[2] = halfSide[2]; }
};
class Sphere : public ShapeBase {  // :238-301
 public:
  explicit Sphere(FCL_REAL r) : radius(r) {}
  FCL_REAL radius;
  NODE_TYPE getNodeType() const override { return GEOM_SPHERE; }
  void params(double p[3]) const override { p[0] = radius; p[1] = p[2] = 0; }
};
class Ellipsoid : public ShapeBase {  // :303-379
 public:
  Ellipsoid(FCL_REAL rx, FCL_REAL ry, FCL_REAL rz) : radii(rx, ry, rz) {}
  Vec3f radii;
  NODE_TYPE getNodeType() const override { return GEOM_ELLIPSOID; }
  void params(double p[3]) const override { p[0] = radii[0]; p[1] = radii[1]; p[2] = radii[2]; }
};
#define HFB_RADIUS_LENGTH_SHAPE(Name, Type)                                         \
  class Name : public ShapeBase {                                                   \
   public:                                                                          \
    Name(FCL_REAL radius_, FCL_REAL lz_) : radius(radius_), halfLength(lz_ / 2) {}  \
    FCL_REAL radius, halfLength;                                                    \
    NODE_TYPE getNodeType() const override { return Type; }                         \
    void params(double p[3]) const override { p[0] = radius; p[1] = halfLength; p[2] = 0; } \
  };
HFB_RADIUS_LENGTH_SHAPE(Capsule, GEOM_CAPSULE)    // :381-463
HFB_RADIUS_LENGTH_SHAPE(Cone, GEOM_CONE)          // :465-553
HFB_RADIUS_LENGTH_SHAPE(Cylinder, GEOM_CYLINDER)  // :555-634
#undef HFB_RADIUS_LENGTH_SHAPE

// Halfspace n . x <= d (:885-961) and Plane n . x = d (:977-1050); the constructors normalise (n, d) like the
// reference's unitNormalTest (src/shape/geometric_shapes.cpp:121-143)
#define HFB_PLANE_SHAPE(Name, Type)                                                        \
  class Name : public ShapeBase {                                                          \
   public:                                                                                 \
    Name(const Vec3f& n_, FCL_REAL d_) : n(n_), d(d_) { unitNormalTest(); }                \
    Name(FCL_REAL a, FCL_REAL b, FCL_REAL c, FCL_REAL d_) : n(a, b, c), d(d_) { unitNormalTest(); } \
    Name() : n(1, 0, 0), d(0) {}                                                           \
    Vec3f n;                                                                               \
    FCL_REAL d;                                                                            \
    NODE_TYPE getNodeType() const override { return Type; }                                \
    void params(double p[3]) const override { p[0] = n[0]; p[1] = n[1]; p[2] = n[2]; }     \
    bool plane(double nd[4]) const override {                                              \
      nd[0] = n[0]; nd[1] = n[1]; nd[2] = n[2]; nd[3] = d;                                 \
      return true;                                                                         \
    }                                                                                      \
                                                                                           \
   protected:                                                                              \
    void unitNormalTest() {                                                                \
      const FCL_REAL l = std::sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]);             \
      if (l > 0) {                                                                         \
        const FCL_REAL inv_l = 1.0 / l;                                                    \
        n = Vec3f(n[0] * inv_l, n[1] * inv_l, n[2] * inv_l);                               \
        d *= inv_l;                                                                        \
      } else {                                                                             \
        n = Vec3f(1, 0, 0);                                                                \
        d = 0;                                                                             \
      }                                                                                    \
    }                                                                                      \
  };
HFB_PLANE_SHAPE(Halfspace, GEOM_HALFSPACE)
HFB_PLANE_SHAPE(Plane, GEOM_PLANE)
#undef HFB_PLANE_SHAPE

class ConvexBase : public ShapeBase {  // :638-872 (vertex set; faces/neighbours are not needed on the device)
 public:
  explicit ConvexBase(std::vector<Vec3f> pts) : points(std::make_shared<std::vector<Vec3f>>(std::move(pts))) {
    num_points = (unsigned)points->size();
  }
  std::shared_ptr<std::vector<Vec3f>> points;
  unsigned num_points;
  NODE_TYPE getNodeType() const override { return GEOM_CONVEX; }
  const std::vector<Vec3f>* vertices() const override { return points.get(); }
};
class TriangleP : public ShapeBase {  // :109-162
 public:
  TriangleP(const Vec3f& a_, const Vec3f& b_, const Vec3f& c_) : a(a_), b(b_), c(c_), abc{a_, b_, c_} {}
  Vec3f a, b, c;
  NODE_TYPE getNodeType() const override { return GEOM_TRIANGLE; }
  const std::vector<Vec3f>* vertices() const override { return &abc; }

 private:
  std::vector<Vec3f> abc;
};
// BVHModel<OBBRSS> (include/hpp/fcl/BVH/BVH_model.h): the build protocol of the reference
// (beginModel / addVertex / addTriangle / addSubModel / endModel), triangles only, SPLIT_METHOD_MEAN.
// endModel() builds the tree on the host (hfb_bvh_build_obbrss: bit-identical to the reference's
// BVHModel::bvs); queries walk it on the GPU.  BVHModel<OBB> (collide() only, as in the library) shares the builder:
// the plain OBB tree of a mesh is the OBB half of its OBBRSS tree (oracle/ref_driver.cpp: ref_bvh_obb_is_obbrss_half).
// Other BV types are not provided.
struct OBBRSS {};
struct OBB {};
struct Triangle {  // data_types.h
  size_t vids[3];
  Triangle() : vids{0, 0, 0} {}
  Triangle(size_t a, size_t b, size_t c) : vids{a, b, c} {}
  size_t operator[](int i) const { return vids[i]; }
};
enum BVHBuildState { BVH_BUILD_STATE_EMPTY, BVH_BUILD_STATE_BEGUN, BVH_BUILD_STATE_PROCESSED };
enum BVHReturnCode { BVH_OK = 0, BVH_ERR_BUILD_OUT_OF_SEQUENCE = -2, BVH_ERR_BUILD_EMPTY_MODEL = -3 };
class BVHModelTriangles : public CollisionGeometry {  // what the two models share (BVHModelBase + the tree)
 public:
  unsigned num_tris = 0, num_vertices = 0;
  BVHBuildState build_state = BVH_BUILD_STATE_EMPTY;
  int beginModel(unsigned num_tris_ = 0, unsigned num_vertices_ = 0) {  // BVH_model.cpp:226-263
    if (build_state != BVH_BUILD_STATE_EMPTY) {
      verts_.clear();
      tris_.clear();
      nodes_.clear();
      num_tris = num_vertices = 0;
    }
    tris_.reserve(3 * (size_t)num_tris_);
    verts_.reserve(3 * (size_t)num_vertices_);
    build_state = BVH_BUILD_STATE_BEGUN;
    return BVH_OK;
  }
  int addVertex(const Vec3f& p) {
    if (build_state != BVH_BUILD_STATE_BEGUN) return BVH_ERR_BUILD_OUT_OF_SEQUENCE;
    for (int k = 0; k < 3; ++k) verts_.push_back(p[k]);
    ++num_vertices;
    return BVH_OK;
  }
  int addTriangle(const Vec3f& p1, const Vec3f& p2, const Vec3f& p3) {  // :359-414: three new vertices
    if (build_state != BVH_BUILD_STATE_BEGUN) return BVH_ERR_BUILD_OUT_OF_SEQUENCE;
    const uint32_t offset = num_vertices;
    addVertex(p1);
    addVertex(p2);
    addVertex(p3);
    tris_.push_back(offset);
    tris_.push_back(offset + 1);
    tris_.push_back(offset + 2);
    ++num_tris;
    return BVH_OK;
  }
  int addSubModel(const std::vector<Vec3f>& ps, const std::vector<Triangle>& ts) {  // :470-538
    if (build_state != BVH_BUILD_STATE_BEGUN) return BVH_ERR_BUILD_OUT_OF_SEQUENCE;
    const uint32_t offset = num_vertices;
    for (const Vec3f& p : ps) addVertex(p);
    for (const Triangle& t : ts) {
      for (int k = 0; k < 3; ++k) tris_.push_back((uint32_t)t[k] + offset);
      ++num_tris;
    }
    return BVH_OK;
  }
  int endModel() {  // :540-586 + buildTree
    if (build_state != BVH_BUILD_STATE_BEGUN) return BVH_ERR_BUILD_OUT_OF_SEQUENCE;
    if (num_tris == 0) return BVH_ERR_BUILD_EMPTY_MODEL;
    nodes_.resize(2 * (size_t)num_tris - 1);
    if (hfb_bvh_build_obbrss(verts_.data(), num_vertices, tris_.data(), num_tris, nodes_.data(),
                             (uint32_t)nodes_.size()) != HFB_OK)
      throw std::invalid_argument("BVHModel: invalid triangle indices");
    build_state = BVH_BUILD_STATE_PROCESSED;
    return BVH_OK;
  }
  unsigned getNumBVs() const { return (unsigned)nodes_.size(); }
  const hfb_bvh_node& getBV(unsigned i) const { return nodes_[i]; }
  bool mesh(MeshData& m) const override {
    if (build_state != BVH_BUILD_STATE_PROCESSED) throw std::invalid_argument("BVHModel: endModel() was not called");
    m.nodes = &nodes_;
    m.verts = &verts_;
    m.tris = &tris_;
    return true;
  }

 private:
  std::vector<double> verts_;
  std::vector<uint32_t> tris_;
  std::vector<hfb_bvh_node> nodes_;
};
template <typename BV>
class BVHModel;
template <>
class BVHModel<OBBRSS> : public BVHModelTriangles {
 public:
  NODE_TYPE getNodeType() const override { return BV_OBBRSS; }
};
template <>
class BVHModel<OBB> : public BVHModelTriangles {
 public:
  NODE_TYPE getNodeType() const override { return BV_OBB; }
};
inline bool isMeshType(NODE_TYPE t) { return t == BV_OBBRSS || t == BV_OBB; }
typedef std::shared_ptr<CollisionGeometry> CollisionGeometryPtr_t;

struct AABB {  // BV/AABB.h
  Vec3f min_, max_;
  bool overlap(const AABB& o) const {  // :111-118, closed intervals
    for (int k = 0; k < 3; ++k)
      if (min_[k] > o.max_[k] || max_[k] < o.min_[k]) return false;
    return true;
  }
};

class CollisionObject {  // collision_object.h
 public:
  CollisionObject(const CollisionGeometryPtr_t& g, const Transform3f& tf) : geom(g), t(tf) {}
  const CollisionGeometry* collisionGeometryPtr() const { return geom.get(); }
  const CollisionGeometryPtr_t& collisionGeometry() const { return geom; }
  const Transform3f& getTransform() const { return t; }
  void setTransform(const Transform3f& tf) { t = tf; }
  /// world-space box (:258-278); filled by the broadphase manager's setup() / update() for all its objects at once
  const AABB& getAABB() const { return aabb; }
  AABB& getAABB() { return aabb; }

 private:
  CollisionGeometryPtr_t geom;
  Transform3f t;
  AABB aabb;
};

// -------------------------------------------------------------- requests ------
enum GJKInitialGuess { DefaultGuess, CachedGuess, BoundingVolumeGuess };
enum GJKVariant { DefaultGJK, PolyakAcceleration, NesterovAcceleration };
enum GJKConvergenceCriterion { Default, DualityGap, Hybrid };
enum GJKConvergenceCriterionType { Relative, Absolute };

struct QueryResult;
struct QueryRequest {  // collision_data.h:171-274
  GJKInitialGuess gjk_initial_guess = DefaultGuess;
  GJKVariant gjk_variant = DefaultGJK;
  GJKConvergenceCriterion gjk_convergence_criterion = Default;
  GJKConvergenceCriterionType gjk_convergence_criterion_type = Relative;
  FCL_REAL gjk_tolerance = 1e-6;
  size_t gjk_max_iterations = 128;
  mutable Vec3f cached_gjk_guess = Vec3f(1, 0, 0);
  mutable std::array<int, 2> cached_support_func_guess{{0, 0}};
  size_t epa_max_iterations = 64;
  FCL_REAL epa_tolerance = 1e-6;
  bool enable_timings = false;
  FCL_REAL collision_distance_threshold = 1e-12;
  inline void updateGuess(const QueryResult& result) const;  // :291-300
  void fill(hfb_query_request& q) const {
    q.gjk_initial_guess = gjk_initial_guess;
    q.gjk_variant = gjk_variant;
    q.gjk_convergence_criterion = gjk_convergence_criterion;
    q.gjk_convergence_criterion_type = gjk_convergence_criterion_type;
    q.gjk_max_iterations = (uint32_t)gjk_max_iterations;
    q.epa_max_iterations = (uint32_t)epa_max_iterations;
    q.gjk_tolerance = gjk_tolerance;
    q.epa_tolerance = epa_tolerance;
    q.collision_distance_threshold = collision_distance_threshold;
    q.cached_gjk_guess = nullptr;
    q.cached_support_func_guess = nullptr;
  }
};
struct QueryResult {
  Vec3f cached_gjk_guess = Vec3f(1, 0, 0);
  std::array<int, 2> cached_support_func_guess{{0, 0}};
};
inline void QueryRequest::updateGuess(const QueryResult& result) const {
  if (gjk_initial_guess == CachedGuess) {
    cached_gjk_guess = result.cached_gjk_guess;
    cached_support_func_guess = result.cached_support_func_guess;
  }
}

struct Contact {  // collision_data.h:59-166
  const CollisionGeometry* o1 = nullptr;
  const CollisionGeometry* o2 = nullptr;
  int b1 = -1, b2 = -1;
  Vec3f normal;
  std::array<Vec3f, 2> nearest_points;
  Vec3f pos;
  FCL_REAL penetration_depth = (std::numeric_limits<FCL_REAL>::max)();
  static const int NONE = -1;
};

struct CollisionResult;
struct CollisionRequest : QueryRequest {  // :312-383
  size_t num_max_contacts = 1;
  bool enable_contact = true;
  FCL_REAL security_margin = 0;
  FCL_REAL break_distance = 1e-3;
  FCL_REAL distance_upper_bound = (std::numeric_limits<FCL_REAL>::max)();
  inline bool isSatisfied(const CollisionResult& result) const;
};
struct CollisionResult : QueryResult {  // :391-509
  std::vector<Contact> contacts;
  FCL_REAL distance_lower_bound = (std::numeric_limits<FCL_REAL>::max)();
  Vec3f normal = Vec3f::Constant(std::numeric_limits<FCL_REAL>::quiet_NaN());
  std::array<Vec3f, 2> nearest_points{{normal, normal}};
  bool isCollision() const { return contacts.size() > 0; }
  size_t numContacts() const { return contacts.size(); }
  const Contact& getContact(size_t i) const {
    if (contacts.size() == 0) throw std::invalid_argument("The number of contacts is zero. No Contact can be returned.");
    return i < contacts.size() ? contacts[i] : contacts.back();
  }
  void addContact(const Contact& c) { contacts.push_back(c); }
  void clear() { *this = CollisionResult(); }
};
inline bool CollisionRequest::isSatisfied(const CollisionResult& r) const {  // collision_data.cpp:44-46
  return r.isCollision() && (num_max_contacts <= r.numContacts());
}

struct DistanceResult;
struct DistanceRequest : QueryRequest {  // :987-1050
  bool enable_nearest_points = true;
  bool enable_signed_distance = true;
  FCL_REAL rel_err = 0, abs_err = 0;
  DistanceRequest(bool enable_nearest_points_ = true, bool enable_signed_distance_ = true, FCL_REAL rel_err_ = 0,
                  FCL_REAL abs_err_ = 0)
      : enable_nearest_points(enable_nearest_points_), enable_signed_distance(enable_signed_distance_),
        rel_err(rel_err_), abs_err(abs_err_) {}
  inline bool isSatisfied(const DistanceResult& result) const;
};
struct DistanceResult : QueryResult {  // :1053-1174
  FCL_REAL min_distance = (std::numeric_limits<FCL_REAL>::max)();
  Vec3f normal = Vec3f::Constant(std::numeric_limits<FCL_REAL>::quiet_NaN());
  std::array<Vec3f, 2> nearest_points{{normal, normal}};
  const CollisionGeometry* o1 = nullptr;
  const CollisionGeometry* o2 = nullptr;
  int b1 = -1, b2 = -1;
  static const int NONE = -1;
  void clear() { *this = DistanceResult(); }
};
inline bool DistanceRequest::isSatisfied(const DistanceResult& r) const { return r.min_distance <= 0; }

// ------------------------------------------------------------- device arena ----
// One context per device; geometry handle cache keyed by object address (the
// caller keeps ownership, like the reference; re-registration on parameter change
// is the caller's job via Context::invalidate).
class Context {
 public:
  static Context& instance(int device = 0) {
    static std::mutex mu;
    static std::unordered_map<int, std::unique_ptr<Context>> all;
    std::lock_guard<std::mutex> lk(mu);
    auto& c = all[device];
    if (!c) c.reset(new Context(device));
    return *c;
  }
  ~Context() { hfb_ctx_destroy(ctx); }
  hfb_ctx* raw() { return ctx; }
  uint32_t handle(const CollisionGeometry* g) {
    CollisionGeometry::MeshData md;
    if (g->mesh(md)) return mesh_handle(g, md);
    double nd[4];
    if (g->plane(nd)) return plane_handle(g, nd);
    hfb_shape rec;
    rec.type = (uint32_t)g->getNodeType();
    rec.data = 0;
    g->params(rec.p);
    const ShapeBase* sb = dynamic_cast<const ShapeBase*>(g);
    rec.ssr = sb ? sb->getSweptSphereRadius() : 0.0;
    const std::vector<Vec3f>* verts = g->vertices();
    // the cache is keyed by address, so an entry is only valid while the flattened record still
    // matches (a freed geometry's address can be reused by a different shape)
    auto it = handles.find(g);
    if (it != handles.end()) {
      const Entry& e = it->second;
      bool same = e.rec.type == rec.type && e.rec.p[0] == rec.p[0] && e.rec.p[1] == rec.p[1] &&
                  e.rec.p[2] == rec.p[2] && e.rec.ssr == rec.ssr && e.nverts == (verts ? verts->size() : 0);
      if (same && verts)
        for (size_t i = 0; i < verts->size() && same; ++i)
          for (int k = 0; k < 3; ++k) same = same && e.verts[3 * i + k] == (*verts)[i][k];
      if (same) return e.handle;
      // changed in place: the handle stays when the arena can absorb the change (same node type, same number of
      // vertices) -- record and vertex set are updated; otherwise it is retired and a new one registered
      if (e.rec.type == rec.type && e.nverts == (verts ? verts->size() : 0)) {
        Entry& m = it->second;
        rec.data = m.rec.data;
        if (verts) {
          for (size_t i = 0; i < verts->size(); ++i)
            for (int k = 0; k < 3; ++k) m.verts[3 * i + k] = (*verts)[i][k];
          check(hfb_geom_update_convex(ctx, rec.data, m.verts.data(), (uint32_t)verts->size()));
        }
        check(hfb_geom_update_shapes(ctx, &m.handle, &rec, 1));
        m.rec = rec;
        dirty = true;
        return m.handle;
      }
      check(hfb_geom_release_shapes(ctx, &e.handle, 1));
      handles.erase(it);
    }
    Entry ent;
    if (const std::vector<Vec3f>* v = verts) {
      std::vector<double>& flat = ent.verts;
      flat.resize(3 * v->size());
      for (size_t i = 0; i < v->size(); ++i)
        for (int k = 0; k < 3; ++k) flat[3 * i + k] = (*v)[i][k];
      check(hfb_geom_register_convex(ctx, flat.data(), (uint32_t)v->size(), &rec.data));
      ent.nverts = v->size();
    }
    uint32_t h;
    check(hfb_geom_register_shapes(ctx, &rec, 1, &h));
    ent.rec = rec;
    ent.handle = h;
    handles[g] = ent;
    dirty = true;
    return h;
  }
  // Plane / Halfspace: (n, d) live outside the record, so one changed in place is registered anew
  uint32_t plane_handle(const CollisionGeometry* g, const double nd[4]) {
    const uint32_t type = (uint32_t)g->getNodeType();
    const double ssr = static_cast<const ShapeBase*>(g)->getSweptSphereRadius();
    auto it = handles.find(g);
    if (it != handles.end()) {
      const Entry& e = it->second;
      if (e.rec.type == type && e.rec.ssr == ssr && e.verts.size() == 4 && e.verts[0] == nd[0] && e.verts[1] == nd[1] &&
          e.verts[2] == nd[2] && e.verts[3] == nd[3])
        return e.handle;
      check(hfb_geom_release_shapes(ctx, &e.handle, 1));
      handles.erase(it);
    }
    Entry ent;
    ent.rec = hfb_shape{};
    ent.rec.type = type;
    ent.rec.ssr = ssr;
    ent.verts.assign(nd, nd + 4);
    uint32_t h;
    check(hfb_geom_register_halfspaces(ctx, type, nd, &ssr, 1, &h));
    ent.handle = h;
    handles[g] = ent;
    dirty = true;
    return h;
  }
  uint32_t mesh_handle(const CollisionGeometry* g, const CollisionGeometry::MeshData& md) {
    auto it = handles.find(g);
    if (it != handles.end()) {
      const Entry& e = it->second;
      if (e.rec.type == (uint32_t)g->getNodeType() && e.verts == *md.verts && e.tris == *md.tris) return e.handle;
      check(hfb_geom_release_shapes(ctx, &e.handle, 1));  // a rebuilt model: the old handle is retired
      handles.erase(it);
    }
    Entry ent;
    ent.rec = hfb_shape{};
    ent.rec.type = (uint32_t)g->getNodeType();
    check((ent.rec.type == HFB_BV_OBB ? hfb_geom_register_bvh_obb : hfb_geom_register_bvh_obbrss)(
        ctx, md.nodes->data(), (uint32_t)md.nodes->size(), md.verts->data(), (uint32_t)(md.verts->size() / 3), md.tris->data(),
        (uint32_t)(md.tris->size() / 3), &ent.rec.data));
    uint32_t h;
    check(hfb_geom_register_shapes(ctx, &ent.rec, 1, &h));
    ent.handle = h;
    ent.verts = *md.verts;
    ent.tris = *md.tris;
    handles[g] = ent;
    dirty = true;
    return h;
  }
  void invalidate(const CollisionGeometry* g) { handles.erase(g); }
  void commit() {
    if (dirty) check(hfb_geom_commit(ctx));
    dirty = false;
  }
  void check(int rc) {
    if (rc == HFB_OK) return;
    const std::string msg = hfb_last_error(ctx);
    if (rc == HFB_ERR_INVALID_ARGUMENT || rc == HFB_ERR_UNSUPPORTED_PAIR) throw std::invalid_argument(msg);
    throw std::runtime_error(msg);
  }

 private:
  explicit Context(int device) {
    const int rc = hfb_ctx_create(device, &ctx);
    if (rc != HFB_OK) throw std::runtime_error("hppfcl_b200: no usable CUDA device (there is no CPU fallback)");
  }
  struct Entry {
    hfb_shape rec{};
    uint32_t handle = 0;
    size_t nverts = 0;
    std::vector<double> verts;
    std::vector<uint32_t> tris;
  };
  hfb_ctx* ctx = nullptr;
  std::unordered_map<const CollisionGeometry*, Entry> handles;
  bool dirty = false;
};

namespace detail {
inline Vec3f v3(const double* p) { return Vec3f(p[0], p[1], p[2]); }
inline void fill(const CollisionRequest& r, hfb_collision_request& q) {
  r.fill(q.q);
  q.num_max_contacts = (uint32_t)r.num_max_contacts;
  q.enable_contact = r.enable_contact;
  q.security_margin = r.security_margin;
  q.break_distance = r.break_distance;
  q.distance_upper_bound = r.distance_upper_bound;
}
inline void fill(const DistanceRequest& r, hfb_distance_request& q) {
  r.fill(q.q);
  q.enable_signed_distance = r.enable_signed_distance;
  q.enable_nearest_points = r.enable_nearest_points;
  q.rel_err = r.rel_err;
  q.abs_err = r.abs_err;
}
inline void unsupported(const char* what, const CollisionGeometry* o1, const CollisionGeometry* o2) {
  throw std::invalid_argument(std::string(what) + " function between node type " +
                              std::to_string((int)o1->getNodeType()) + " and node type " +
                              std::to_string((int)o2->getNodeType()) + " is not yet supported.");
}
}  // namespace detail

// ------------------------------------------------------------------ batched ----
struct BatchNarrowPhase {
  explicit BatchNarrowPhase(int device = 0) : C(Context::instance(device)) {}
  void add(const CollisionGeometry* o1, const Transform3f& tf1, const CollisionGeometry* o2, const Transform3f& tf2) {
    h1.push_back(C.handle(o1));
    h2.push_back(C.handle(o2));
    t1.push_back(tf1.pod());
    t2.push_back(tf2.pod());
  }
  size_t size() const { return h1.size(); }
  void clear() { h1.clear(); h2.clear(); t1.clear(); t2.clear(); }
  std::vector<hfb_contact> collide(const CollisionRequest& request) {
    if (request.num_max_contacts == 0 && request.security_margin != -std::numeric_limits<FCL_REAL>::infinity())
      throw std::invalid_argument("Invalid number of max contacts (current value is 0).");
    hfb_collision_request q;
    detail::fill(request, q);
    C.commit();
    std::vector<hfb_contact> out(h1.size());
    C.check(hfb_batch_collide(C.raw(), h1.size(), h1.data(), t1.data(), h2.data(), t2.data(), &q, out.data(), nullptr));
    return out;
  }
  std::vector<hfb_distance_result> distance(const DistanceRequest& request) {
    hfb_distance_request q;
    detail::fill(request, q);
    C.commit();
    std::vector<hfb_distance_result> out(h1.size());
    C.check(hfb_batch_distance(C.raw(), h1.size(), h1.data(), t1.data(), h2.data(), t2.data(), &q, out.data(), nullptr));
    return out;
  }
  Context& C;
  std::vector<uint32_t> h1, h2;
  std::vector<hfb_transform> t1, t2;
};

// ------------------------------------------------------------ broadphase feed ----
// The seam BASELINE config 5 goes through: a broadphase manager hands candidate pairs to a callback
// (broadphase/broadphase_callbacks.h:54-75); the collecting callback (default_broadphase_callbacks.h:224-252,
// src/broadphase/default_broadphase_callbacks.cpp:43-60... CollisionCallBackCollect) keeps them, and the batch then
// goes to the narrow phase in ONE call (hfb_batch_collide_objects) instead of one collide() per callback.
struct CollisionCallBackBase {
  virtual void init() {}
  virtual bool collide(CollisionObject* o1, CollisionObject* o2) = 0;  // true: stop the broadphase
  virtual bool operator()(CollisionObject* o1, CollisionObject* o2) { return collide(o1, o2); }
  virtual ~CollisionCallBackBase() {}
};
struct CollisionCallBackCollect : CollisionCallBackBase {
  typedef std::pair<CollisionObject*, CollisionObject*> CollisionPair;
  explicit CollisionCallBackCollect(size_t max_size_) : max_size(max_size_) { collision_pairs.resize(max_size); }
  bool collide(CollisionObject* o1, CollisionObject* o2) override {
    collision_pairs.push_back(std::make_pair(o1, o2));
    return false;
  }
  size_t numCollisionPairs() const { return collision_pairs.size(); }
  const std::vector<CollisionPair>& getCollisionPairs() const { return collision_pairs; }
  void init() override { collision_pairs.clear(); }
  bool exist(const CollisionPair& pair) const {
    return std::find(collision_pairs.begin(), collision_pairs.end(), pair) != collision_pairs.end();
  }
  bool exist(CollisionObject* o1, CollisionObject* o2) const { return exist(std::make_pair(o1, o2)); }

 protected:
  std::vector<CollisionPair> collision_pairs;
  size_t max_size;
};

// The manager: BroadPhaseCollisionManager's interface (broadphase/broadphase_collision_manager.h:56-134) for the
// self-collision query of config 5.  setup() / update() compute every object's box (CollisionObject::computeAABB)
// and collide(callback) reports every pair of objects with overlapping boxes exactly once -- the set the reference's
// DynamicAABBTreeCollisionManager reports (broadphase_dynamic_AABB_tree.cpp:336-407,716-721); the order is each
// manager's own.  No tree is kept: a uniform grid is rebuilt per query (hfb_broadphase.cuh), so update() costs a
// re-computation of the boxes and nothing else.
class DynamicAABBTreeCollisionManager {
 public:
  explicit DynamicAABBTreeCollisionManager(int device = 0) : C(Context::instance(device)) {}
  void registerObjects(const std::vector<CollisionObject*>& other_objs) {
    objs.insert(objs.end(), other_objs.begin(), other_objs.end());
    stale = true;
  }
  void registerObject(CollisionObject* obj) {
    objs.push_back(obj);
    stale = true;
  }
  void unregisterObject(CollisionObject* obj) {
    objs.erase(std::remove(objs.begin(), objs.end(), obj), objs.end());
    stale = true;
  }
  void clear() {
    objs.clear();
    stale = true;
  }
  size_t size() const { return objs.size(); }
  bool empty() const { return objs.empty(); }
  void getObjects(std::vector<CollisionObject*>& out) const { out = objs; }
  void setup() { refresh(); }
  void update() { refresh(); }
  /// the box of one object / of some objects from their current poses (broadphase_collision_manager.h:76-79)
  void update(CollisionObject* updated_obj) { update(std::vector<CollisionObject*>(1, updated_obj)); }
  void update(const std::vector<CollisionObject*>& updated_objs) {
    if (stale) return refresh();
    std::vector<size_t> idx;
    std::vector<uint32_t> h;
    std::vector<hfb_transform> t;
    for (CollisionObject* o : updated_objs) {
      const size_t i = std::find(objs.begin(), objs.end(), o) - objs.begin();
      if (i == objs.size()) continue;  // not one of this manager's objects
      tfs[i] = o->getTransform().pod();
      idx.push_back(i);
      h.push_back(hs[i]);
      t.push_back(tfs[i]);
    }
    std::vector<double> bb(6 * idx.size());
    C.check(hfb_scene_aabbs(C.raw(), idx.size(), h.data(), t.data(), bb.data()));
    for (size_t k = 0; k < idx.size(); ++k) {
      std::copy(bb.begin() + 6 * k, bb.begin() + 6 * k + 6, boxes.begin() + 6 * idx[k]);
      AABB& b = objs[idx[k]]->getAABB();
      b.min_ = Vec3f(bb[6 * k], bb[6 * k + 1], bb[6 * k + 2]);
      b.max_ = Vec3f(bb[6 * k + 3], bb[6 * k + 4], bb[6 * k + 5]);
    }
  }
  /// self collision: callback(o1, o2) for every pair with overlapping boxes until it returns true
  void collide(CollisionCallBackBase* callback) {
    callback->init();
    if (stale) refresh();
    std::vector<uint32_t> first, second;
    pairs(first, second);
    for (size_t k = 0; k < first.size(); ++k)
      if ((*callback)(objs[first[k]], objs[second[k]])) return;
  }
  /// the candidate pairs as object indices (what collide(callback) iterates over)
  void pairs(std::vector<uint32_t>& first, std::vector<uint32_t>& second) {
    if (stale) refresh();
    size_t cap = std::max<size_t>(16 * objs.size(), 1024), cnt = 0;
    for (;;) {
      first.resize(cap);
      second.resize(cap);
      C.check(hfb_broadphase_pairs(objs.size(), boxes.data(), first.data(), second.data(), cap, &cnt));
      if (cnt <= cap) break;
      cap = cnt;
    }
    first.resize(cnt);
    second.resize(cnt);
  }
  /// every object of this manager against every object of `other`: callback(o1 from this manager, o2 from other)
  /// for every pair with overlapping boxes until it returns true (broadphase_collision_manager.h:110-118);
  /// collide(this, callback) is the self form
  void collide(DynamicAABBTreeCollisionManager* other, CollisionCallBackBase* callback) {
    if (other == this) return collide(callback);
    callback->init();
    std::vector<uint32_t> first, second;
    pairs(*other, first, second);
    for (size_t k = 0; k < first.size(); ++k)
      if ((*callback)(objs[first[k]], other->objs[second[k]])) return;
  }
  /// one object against every object of this manager: callback(the manager's object, obj), the order of
  /// DynamicAABBTreeCollisionManager::collide(obj, callback) (broadphase_dynamic_AABB_tree.cpp:361-390; the naive
  /// manager passes (obj, object) instead).  obj's box is computed here, as setup() computes the manager's.
  void collide(CollisionObject* obj, CollisionCallBackBase* callback) {
    callback->init();
    if (stale) refresh();
    const uint32_t h = C.handle(obj->collisionGeometryPtr());
    C.commit();
    const hfb_transform t = obj->getTransform().pod();
    double bb[6];
    C.check(hfb_scene_aabbs(C.raw(), 1, &h, &t, bb));
    obj->getAABB().min_ = Vec3f(bb[0], bb[1], bb[2]);
    obj->getAABB().max_ = Vec3f(bb[3], bb[4], bb[5]);
    std::vector<uint32_t> first, second;
    cross_pairs(bb, 1, first, second);
    for (size_t k = 0; k < first.size(); ++k)
      if ((*callback)(objs[first[k]], obj)) return;
  }
  /// the cross candidates as object indices: first in this manager, second in `other`; pairs(*this, ...) is the self
  /// form (first < second), as collide(this, callback) is
  void pairs(DynamicAABBTreeCollisionManager& other, std::vector<uint32_t>& first, std::vector<uint32_t>& second) {
    if (&other == this) return pairs(first, second);
    if (stale) refresh();
    if (other.stale) other.refresh();
    cross_pairs(other.boxes.data(), other.objs.size(), first, second);
  }
  /// the object table of the scene in the form hfb_batch_*_objects takes
  const std::vector<uint32_t>& handles() const { return hs; }
  const std::vector<hfb_transform>& transforms() const { return tfs; }
  Context& context() { return C; }

 private:
  friend class ResidentEnvironment;
  friend class RobotModel;
  void cross_pairs(const double* boxes_b, size_t n_b, std::vector<uint32_t>& first, std::vector<uint32_t>& second) {
    size_t cap = std::max<size_t>(16 * (objs.size() + n_b), 1024), cnt = 0;
    for (;;) {
      first.resize(cap);
      second.resize(cap);
      C.check(hfb_broadphase_cross_pairs(objs.size(), boxes.data(), n_b, boxes_b, first.data(), second.data(), cap, &cnt));
      if (cnt <= cap) break;
      cap = cnt;
    }
    first.resize(cnt);
    second.resize(cnt);
  }
  void refresh() {
    hs.resize(objs.size());
    tfs.resize(objs.size());
    for (size_t i = 0; i < objs.size(); ++i) {
      hs[i] = C.handle(objs[i]->collisionGeometryPtr());
      tfs[i] = objs[i]->getTransform().pod();
    }
    C.commit();
    boxes.resize(6 * objs.size());
    C.check(hfb_scene_aabbs(C.raw(), objs.size(), hs.data(), tfs.data(), boxes.data()));
    for (size_t i = 0; i < objs.size(); ++i) {
      AABB& b = objs[i]->getAABB();
      b.min_ = Vec3f(boxes[6 * i], boxes[6 * i + 1], boxes[6 * i + 2]);
      b.max_ = Vec3f(boxes[6 * i + 3], boxes[6 * i + 4], boxes[6 * i + 5]);
    }
    stale = false;
  }
  Context& C;
  std::vector<CollisionObject*> objs;
  std::vector<uint32_t> hs;
  std::vector<hfb_transform> tfs;
  std::vector<double> boxes;
  bool stale = true;
};

/// Link poses of configurations from a RobotModel, in the form ResidentEnvironment's configuration and motion calls
/// take a robot manager: object g * L + i is link i of configuration g (its table: handles(), transforms()).  It holds
/// no CollisionObject, so the manager's object calls are not offered on it.  q(): the configurations' joint values
/// (n_configs x nq); sweep(): the bounds certify_motions takes (sample_motions with sweep = true, else empty);
/// offsets(): the motion offsets of sample_motions (empty for poses).
class RobotSamples : public DynamicAABBTreeCollisionManager {
 public:
  explicit RobotSamples(int device = 0) : DynamicAABBTreeCollisionManager(device) {}
  size_t size() const { return handles().size(); }
  const std::vector<double>& q() const { return q_; }
  const std::vector<double>& sweep() const { return sweep_; }
  const std::vector<uint32_t>& offsets() const { return offsets_; }
  template <class... A> void registerObject(A&&...) = delete;
  template <class... A> void registerObjects(A&&...) = delete;
  template <class... A> void unregisterObject(A&&...) = delete;
  template <class... A> void clear(A&&...) = delete;
  template <class... A> void setup(A&&...) = delete;
  template <class... A> void update(A&&...) = delete;
  template <class... A> void collide(A&&...) = delete;
  template <class... A> void pairs(A&&...) = delete;
  template <class... A> void getObjects(A&&...) = delete;

 private:
  friend class RobotModel;
  std::vector<double> q_, sweep_;
  std::vector<uint32_t> offsets_;
};

/// A kinematic tree of 1-DoF joints with a geometry per link, kept on the device (hfb_robot): Pinocchio's
/// forwardKinematics + updateGeometryPlacements, batched.  Joint: parent (-1 or an earlier joint), type
/// (HFB_JOINT_REVOLUTE / HFB_JOINT_PRISMATIC), axis, placement (the joint frame in its parent's at q = 0); Link: joint
/// (-1 for fixed to the world), placement, geometry.  nq = the number of joints.  include/hppfcl_b200.h states the
/// semantics and the sweep bounds.  A malformed model, q of the wrong size or malformed offsets throw
/// std::invalid_argument.  Owns the hfb_robot.
class RobotModel {
 public:
  struct Joint {
    int32_t parent;
    uint32_t type;
    Vec3f axis;
    Transform3f placement;
  };
  struct Link {
    int32_t joint;
    Transform3f placement;
    CollisionGeometryPtr_t geometry;
  };
  RobotModel(const std::vector<Joint>& joints, const std::vector<Link>& links, int device = 0)
      : device(device), C(Context::instance(device)) {
    if (joints.size() > 64 || links.size() > 0xffffffffull) throw std::invalid_argument("robot model: too many joints or links");
    std::vector<int32_t> parent, link_joint;
    std::vector<uint32_t> type, handles;
    std::vector<double> axis;
    std::vector<hfb_transform> placement, link_placement;
    for (const Joint& j : joints) {
      parent.push_back(j.parent);
      type.push_back(j.type);
      for (int k = 0; k < 3; ++k) axis.push_back(j.axis[k]);
      placement.push_back(j.placement.pod());
    }
    for (const Link& l : links) {
      link_joint.push_back(l.joint);
      link_placement.push_back(l.placement.pod());
      geoms.push_back(l.geometry);
      handles.push_back(C.handle(l.geometry.get()));
    }
    C.commit();
    hfb_robot_desc d{(uint32_t)joints.size(), parent.data(), type.data(),       axis.data(),  placement.data(),
                     (uint32_t)links.size(),  link_joint.data(), link_placement.data(), handles.data()};
    C.check(hfb_robot_create(C.raw(), &d, &robot));
    nq_ = joints.size();
    L = links.size();
  }
  ~RobotModel() {
    if (robot) hfb_robot_destroy(C.raw(), robot);
  }
  RobotModel(const RobotModel&) = delete;
  RobotModel& operator=(const RobotModel&) = delete;
  size_t nq() const { return nq_; }
  size_t num_links() const { return L; }

  /// q: n_configs x nq joint values -> the links' poses of every configuration (hfb_robot_poses)
  RobotSamples poses(const std::vector<double>& q) {
    if (q.size() % nq_) throw std::invalid_argument("q: nq values per configuration");
    const size_t n = q.size() / nq_;
    sync();
    RobotSamples s(device);
    s.hs.resize(n * L);
    s.tfs.resize(n * L);
    C.check(hfb_robot_poses(C.raw(), robot, n, q.data(), s.tfs.data(), s.hs.data()));
    s.stale = false;
    s.q_ = q;
    return s;
  }

  /// motion m from q_from[m] to q_to[m] (n_motions x nq each), offsets[m+1] - offsets[m] samples linear in q, end points
  /// included -> the samples' poses, their q and (sweep = true) the sweep bounds (hfb_robot_sample_motions)
  RobotSamples sample_motions(const std::vector<double>& q_from, const std::vector<double>& q_to,
                              const std::vector<uint32_t>& offsets, bool sweep = true) {
    if (offsets.empty() || offsets[0] != 0) throw std::invalid_argument("motion offsets must start at 0");
    for (size_t m = 0; m + 1 < offsets.size(); ++m) {
      if (offsets[m + 1] < offsets[m]) throw std::invalid_argument("motion offsets decrease");
      if (offsets[m + 1] - offsets[m] > 0x7fffffffu) throw std::invalid_argument("a motion has more than INT32_MAX samples");
    }
    const size_t n_motions = offsets.size() - 1, n = offsets.back();
    if (q_from.size() != n_motions * nq_ || q_to.size() != n_motions * nq_)
      throw std::invalid_argument("q_from, q_to: nq values per motion");
    sync();
    RobotSamples s(device);
    s.hs.resize(n * L);
    s.tfs.resize(n * L);
    s.q_.resize(n * nq_);
    if (sweep) s.sweep_.resize(n * L);
    hfb_robot_samples_out o{s.tfs.data(), s.hs.data(), s.q_.data(), sweep ? s.sweep_.data() : nullptr};
    C.check(hfb_robot_sample_motions(C.raw(), robot, n_motions, q_from.data(), q_to.data(), offsets.data(), &o));
    s.stale = false;
    s.offsets_ = offsets;
    return s;
  }

 private:
  // the links' geometry changed in place since: its records updated and committed, as a manager's setup() does
  void sync() {
    for (const CollisionGeometryPtr_t& g : geoms) C.handle(g.get());
    C.commit();
  }
  friend class ResidentEnvironment;
  int device;
  Context& C;
  std::vector<CollisionGeometryPtr_t> geoms;
  hfb_robot* robot = nullptr;
  size_t nq_ = 0, L = 0;
};

/// What ResidentEnvironment::validate_motions returns: per motion status (0 valid, 1 collides, 2 unresolved, -1 outside
/// the range), t_valid (the certified prefix is [0, t_valid]), t_collide (the earliest colliding sample found, -1 for
/// none) and the witness there (kind, first, second: link indices, or an environment index for kind 0; contacts); the
/// counts summed over the rounds.
struct MotionValidation {
  std::vector<int8_t> status;
  std::vector<double> t_valid, t_collide;
  std::vector<int8_t> kind;
  std::vector<uint32_t> first, second;
  std::vector<hfb_contact> contacts;
  uint32_t n_rounds = 0;
  uint64_t n_samples = 0, n_env_candidates = 0, n_self_candidates = 0, n_unsupported = 0;
};

/// config 5 in one call: the manager's candidate pairs through the batched narrow phase.  Returns, per candidate
/// pair, the record hfb_batch_collide writes (first / second: object indices in registration order).
inline std::vector<hfb_contact> collide(DynamicAABBTreeCollisionManager& manager, const CollisionRequest& request,
                                        std::vector<uint32_t>& first, std::vector<uint32_t>& second) {
  if (request.num_max_contacts == 0 && request.security_margin != -std::numeric_limits<FCL_REAL>::infinity())
    throw std::invalid_argument("Invalid number of max contacts (current value is 0).");
  manager.pairs(first, second);
  hfb_collision_request q;
  detail::fill(request, q);
  hfb_object_pairs sc;
  sc.n_objects = manager.handles().size();
  sc.object_handles = manager.handles().data();
  sc.object_tfs = manager.transforms().data();
  sc.n_pairs = first.size();
  sc.first = first.data();
  sc.second = second.data();
  std::vector<hfb_contact> out(first.size());
  manager.context().check(hfb_batch_collide_objects(manager.context().raw(), &sc, &q, out.data(), nullptr, nullptr));
  return out;
}

/// the cross form in one call: the candidates of manager x other (first: index in `manager`, second: index in `other`)
/// through the batched narrow phase over the object table [manager; other], o1 from `manager`.  Returns, per
/// candidate pair, the record hfb_batch_collide writes.  collide(m, m, ...) is the self form collide(m, ...).
inline std::vector<hfb_contact> collide(DynamicAABBTreeCollisionManager& manager, DynamicAABBTreeCollisionManager& other,
                                        const CollisionRequest& request, std::vector<uint32_t>& first,
                                        std::vector<uint32_t>& second) {
  if (&other == &manager) return collide(manager, request, first, second);
  if (request.num_max_contacts == 0 && request.security_margin != -std::numeric_limits<FCL_REAL>::infinity())
    throw std::invalid_argument("Invalid number of max contacts (current value is 0).");
  manager.pairs(other, first, second);
  hfb_collision_request q;
  detail::fill(request, q);
  std::vector<uint32_t> hs(manager.handles());
  hs.insert(hs.end(), other.handles().begin(), other.handles().end());
  std::vector<hfb_transform> tfs(manager.transforms());
  tfs.insert(tfs.end(), other.transforms().begin(), other.transforms().end());
  std::vector<uint32_t> table_second(second);
  for (uint32_t& s : table_second) s += (uint32_t)manager.handles().size();
  hfb_object_pairs sc;
  sc.n_objects = hs.size();
  sc.object_handles = hs.data();
  sc.object_tfs = tfs.data();
  sc.n_pairs = first.size();
  sc.first = first.data();
  sc.second = table_second.data();
  std::vector<hfb_contact> out(first.size());
  manager.context().check(hfb_batch_collide_objects(manager.context().raw(), &sc, &q, out.data(), nullptr, nullptr));
  return out;
}

/// A manager's objects kept on the device as set B of the two-set collide (hfb_env): the table, the boxes as of
/// construction / update(objs) and the grid over them stay there between queries, as the reference's tree does between
/// setup() and update().  collide(), collide_flags(), distance() and clearance() upload only the robot manager's poses.
/// Owns the hfb_env.
class ResidentEnvironment {
 public:
  explicit ResidentEnvironment(DynamicAABBTreeCollisionManager& manager) : C(manager.C) {
    if (manager.stale) manager.refresh();
    for (size_t i = 0; i < manager.objs.size(); ++i) index[manager.objs[i]] = (uint32_t)i;
    C.check(hfb_env_create(C.raw(), manager.hs.size(), manager.hs.data(), manager.tfs.data(), &env));
  }
  ~ResidentEnvironment() { hfb_env_destroy(C.raw(), env); }
  ResidentEnvironment(const ResidentEnvironment&) = delete;
  ResidentEnvironment& operator=(const ResidentEnvironment&) = delete;
  /// the current poses of these environment objects pushed to the device (their boxes and the grid are redone)
  void update(const std::vector<CollisionObject*>& objs) {
    std::vector<uint32_t> idx;
    std::vector<hfb_transform> t;
    for (CollisionObject* o : objs) {
      auto it = index.find(o);
      if (it == index.end()) throw std::invalid_argument("not an object of this environment");
      idx.push_back(it->second);
      t.push_back(o->getTransform().pod());
    }
    C.check(hfb_env_update(C.raw(), env, idx.size(), idx.data(), t.data()));
  }
  /// the colliding pairs (first: index in the robot manager, second: index in the environment) and their records
  std::vector<hfb_contact> collide(DynamicAABBTreeCollisionManager& robot, const CollisionRequest& request,
                                   std::vector<uint32_t>& first, std::vector<uint32_t>& second) {
    hfb_collision_request q;
    prepare(robot, request, q);
    uint32_t hits = 0, cand = 0;
    std::vector<hfb_contact> rec;
    for (size_t cap = std::max<size_t>(4 * robot.hs.size(), 1024);;) {
      first.resize(cap);
      second.resize(cap);
      rec.resize(cap);
      hfb_env_out out{first.data(), second.data(), rec.data(), (uint32_t)cap, &hits, &cand, nullptr};
      C.check(hfb_env_collide(C.raw(), env, robot.hs.size(), robot.hs.data(), robot.tfs.data(), 0, robot.hs.size(), &q, &out));
      if (hits <= cap) break;
      cap = hits;
    }
    first.resize(hits);
    second.resize(hits);
    rec.resize(hits);
    return rec;
  }
  /// one byte per robot object: 1 iff it collides with the environment (no pair records come back)
  std::vector<uint8_t> collide_flags(DynamicAABBTreeCollisionManager& robot, const CollisionRequest& request) {
    hfb_collision_request q;
    prepare(robot, request, q);
    std::vector<uint8_t> flags(robot.hs.size());
    hfb_env_out out{nullptr, nullptr, nullptr, 0, nullptr, nullptr, flags.data()};
    C.check(hfb_env_collide(C.raw(), env, robot.hs.size(), robot.hs.data(), robot.tfs.data(), 0, robot.hs.size(), &q, &out));
    return flags;
  }
  /// colliding pairs of one kind: object indices and the records
  struct Pairs {
    std::vector<uint32_t> first, second;
    std::vector<hfb_contact> contacts;
  };
  /// A planner's validity check: the robot manager holds configurations of links_per_config objects each,
  /// configuration-major (object g * L + i is link i of configuration g); self_pairs is the template of link pairs
  /// (i, j) each configuration checks against itself (an SRDF's enabled pairs).  Returns one byte per configuration,
  /// 1 iff it collides with the environment or with itself; env_pairs gets the colliding (robot index, environment
  /// index) pairs, self_pairs_out the colliding (robot index, robot index) pairs.  A malformed template throws
  /// std::invalid_argument.
  std::vector<uint8_t> collide_configurations(DynamicAABBTreeCollisionManager& robot, size_t links_per_config,
                                              const std::vector<std::pair<uint32_t, uint32_t>>& self_pairs,
                                              const CollisionRequest& request, Pairs& env_pairs, Pairs& self_pairs_out) {
    hfb_collision_request q;
    prepare(robot, request, q);
    std::vector<uint8_t> verdicts(links_per_config ? robot.hs.size() / links_per_config : 0);
    uint32_t hits[2] = {0, 0}, cand[2] = {0, 0};
    Pairs* kinds[2] = {&env_pairs, &self_pairs_out};
    for (size_t cap[2] = {std::max<size_t>(4 * robot.hs.size(), 1024), std::max<size_t>(4 * robot.hs.size(), 1024)};;) {
      hfb_scene_contacts o[2];
      for (int k = 0; k < 2; ++k) {
        kinds[k]->first.resize(cap[k]);
        kinds[k]->second.resize(cap[k]);
        kinds[k]->contacts.resize(cap[k]);
        o[k] = {kinds[k]->first.data(), kinds[k]->second.data(), kinds[k]->contacts.data(), (uint32_t)cap[k], &hits[k], &cand[k]};
      }
      hfb_configs_out out{verdicts.data(), o[0], o[1]};
      check_configs(robot, links_per_config, self_pairs, q, out);
      if (hits[0] <= cap[0] && hits[1] <= cap[1]) break;
      cap[0] = std::max<size_t>(cap[0], hits[0]);
      cap[1] = std::max<size_t>(cap[1], hits[1]);
    }
    for (int k = 0; k < 2; ++k) {
      kinds[k]->first.resize(hits[k]);
      kinds[k]->second.resize(hits[k]);
      kinds[k]->contacts.resize(hits[k]);
    }
    return verdicts;
  }
  /// one byte per configuration: 1 iff it collides with the environment or with itself (no pair records come back)
  std::vector<uint8_t> configuration_flags(DynamicAABBTreeCollisionManager& robot, size_t links_per_config,
                                           const std::vector<std::pair<uint32_t, uint32_t>>& self_pairs,
                                           const CollisionRequest& request) {
    hfb_collision_request q;
    prepare(robot, request, q);
    std::vector<uint8_t> verdicts(links_per_config ? robot.hs.size() / links_per_config : 0);
    hfb_configs_out out{verdicts.data(), {nullptr, nullptr, nullptr, 0, nullptr, nullptr},
                        {nullptr, nullptr, nullptr, 0, nullptr, nullptr}};
    check_configs(robot, links_per_config, self_pairs, q, out);
    return verdicts;
  }
  /// each robot object's nearest environment object: nearest[i] (index in the environment, -1 when no pair is
  /// eligible), min_distance[i] (DBL_MAX when none) and the distance record.  distance() runs with a fresh
  /// DistanceResult on each pair; the eligible pairs are those at min_distance <= max_distance and not unsupported; the
  /// smallest distance wins, the lowest environment index on ties (hfb_env_distance).  A max_distance that is NaN or
  /// negative throws std::invalid_argument.
  std::vector<hfb_distance_result> distance(DynamicAABBTreeCollisionManager& robot, const DistanceRequest& request,
                                            std::vector<int32_t>& nearest, std::vector<FCL_REAL>& min_distance,
                                            FCL_REAL max_distance = std::numeric_limits<FCL_REAL>::infinity()) {
    std::vector<hfb_distance_result> rec(robot_size(robot, max_distance));
    nearest.resize(rec.size());
    min_distance.resize(rec.size());
    query_distance(robot, request, max_distance, {nearest.data(), min_distance.data(), rec.data(), nullptr, nullptr});
    return rec;
  }
  /// the distances alone: each robot object's distance to its nearest environment object (no records come back)
  std::vector<FCL_REAL> clearance(DynamicAABBTreeCollisionManager& robot,
                                  FCL_REAL max_distance = std::numeric_limits<FCL_REAL>::infinity(),
                                  const DistanceRequest& request = DistanceRequest()) {
    std::vector<FCL_REAL> d(robot_size(robot, max_distance));
    query_distance(robot, request, max_distance, {nullptr, d.data(), nullptr, nullptr, nullptr});
    return d;
  }
  /// A planner's clearance: per configuration (robot manager laid out as in collide_configurations) its nearest pair
  /// over the environment pairs and the template's self pairs.  kind[g]: 0 environment, 1 self, -1 none eligible;
  /// first[g]: index in the robot manager; second[g]: index in the environment (kind 0) or in the robot manager (kind
  /// 1), UINT32_MAX when none; min_distance[g]: DBL_MAX when none; returns the records.  The eligible pairs and the
  /// argmin are those of distance(); on a tie an environment pair beats a self pair, and earlier links and template
  /// entries beat later ones (hfb_env_distance_configs).  A max_distance that is NaN or negative, or a malformed
  /// template, throws std::invalid_argument.
  std::vector<hfb_distance_result> distance_configurations(
      DynamicAABBTreeCollisionManager& robot, size_t links_per_config,
      const std::vector<std::pair<uint32_t, uint32_t>>& self_pairs, const DistanceRequest& request,
      std::vector<int8_t>& kind, std::vector<uint32_t>& first, std::vector<uint32_t>& second,
      std::vector<FCL_REAL>& min_distance, FCL_REAL max_distance = std::numeric_limits<FCL_REAL>::infinity()) {
    const size_t n = robot_size(robot, max_distance), n_configs = links_per_config ? n / links_per_config : 0;
    std::vector<hfb_distance_result> rec(n_configs);
    kind.resize(n_configs);
    first.resize(n_configs);
    second.resize(n_configs);
    min_distance.resize(n_configs);
    distance_configs(robot, links_per_config, self_pairs, request, max_distance,
                     {kind.data(), first.data(), second.data(), min_distance.data(), rec.data(), nullptr, nullptr, nullptr});
    return rec;
  }
  /// the distances alone: each configuration's clearance (no records come back)
  std::vector<FCL_REAL> configuration_clearance(DynamicAABBTreeCollisionManager& robot, size_t links_per_config,
                                                const std::vector<std::pair<uint32_t, uint32_t>>& self_pairs,
                                                FCL_REAL max_distance = std::numeric_limits<FCL_REAL>::infinity(),
                                                const DistanceRequest& request = DistanceRequest()) {
    const size_t n = robot_size(robot, max_distance);
    std::vector<FCL_REAL> d(links_per_config ? n / links_per_config : 0);
    distance_configs(robot, links_per_config, self_pairs, request, max_distance,
                     {nullptr, nullptr, nullptr, d.data(), nullptr, nullptr, nullptr, nullptr});
    return d;
  }
  /// A planner's motion validation: the robot manager holds configurations laid out as in collide_configurations, the
  /// samples of each motion one after another in walking order; motion m is configurations [offsets[m], offsets[m+1]).
  /// Per motion: first_invalid[m], the first sample that collides with the environment or with itself (-1 when none
  /// does); kind[m]: 0 environment pair, 1 self pair, -1 none; first[m]: index in the robot manager; second[m]: index
  /// in the environment (kind 0) or in the robot manager (kind 1), UINT32_MAX when none; returns the pairs' contact
  /// records.  The pair is the first colliding one of that sample: environment pairs by link, then by environment
  /// index, then self pairs in template order (hfb_env_collide_motions).  Malformed offsets (not starting at 0,
  /// decreasing, not ending at the number of configurations) or a malformed template throw std::invalid_argument.
  std::vector<hfb_contact> collide_motions(DynamicAABBTreeCollisionManager& robot, size_t links_per_config,
                                           const std::vector<std::pair<uint32_t, uint32_t>>& self_pairs,
                                           const std::vector<uint32_t>& offsets, const CollisionRequest& request,
                                           std::vector<int32_t>& first_invalid, std::vector<int8_t>& kind,
                                           std::vector<uint32_t>& first, std::vector<uint32_t>& second) {
    if (offsets.empty()) throw std::invalid_argument("motion offsets: n_motions + 1 values, at least one");
    const size_t n = offsets.size() - 1;
    std::vector<hfb_contact> rec(n);
    first_invalid.resize(n);
    kind.resize(n);
    first.resize(n);
    second.resize(n);
    check_motions(robot, links_per_config, self_pairs, offsets, request,
                  {first_invalid.data(), kind.data(), first.data(), second.data(), rec.data(), nullptr, nullptr, nullptr,
                   nullptr});
    return rec;
  }
  /// the first colliding samples alone (no pair records come back)
  std::vector<int32_t> first_invalid_samples(DynamicAABBTreeCollisionManager& robot, size_t links_per_config,
                                             const std::vector<std::pair<uint32_t, uint32_t>>& self_pairs,
                                             const std::vector<uint32_t>& offsets,
                                             const CollisionRequest& request = CollisionRequest()) {
    if (offsets.empty()) throw std::invalid_argument("motion offsets: n_motions + 1 values, at least one");
    std::vector<int32_t> first_invalid(offsets.size() - 1);
    check_motions(robot, links_per_config, self_pairs, offsets, request,
                  {first_invalid.data(), nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr});
    return first_invalid;
  }

  /// A planner's continuous motion validation: the motions of collide_motions, and sweep (one bound per robot object):
  /// sweep[g * links_per_config + i] bounds the path length of every point of link i from configuration g to g + 1
  /// (hpp-core's maximal velocity times the step; not finite and >= 0: the segment is not certified).  Per motion:
  /// first_invalid[m], what collide_motions gives; first_uncertified[m], the first segment not certified free (-1 when
  /// all are); returns per configuration 1 when the segment to the next sample of its motion is certified free
  /// (hfb_env_certify_motions states the rule and its guarantee).  A sweep whose size is not the robot's, malformed
  /// offsets or a malformed template throw std::invalid_argument.
  std::vector<uint8_t> certify_motions(DynamicAABBTreeCollisionManager& robot, size_t links_per_config,
                                       const std::vector<std::pair<uint32_t, uint32_t>>& self_pairs,
                                       const std::vector<uint32_t>& offsets, const std::vector<double>& sweep,
                                       const CollisionRequest& request, std::vector<int32_t>& first_invalid,
                                       std::vector<int32_t>& first_uncertified) {
    if (offsets.empty()) throw std::invalid_argument("motion offsets: n_motions + 1 values, at least one");
    if (sweep.size() != robot.hs.size()) throw std::invalid_argument("sweep: one bound per object of the robot manager");
    const size_t n = offsets.size() - 1;
    first_invalid.resize(n);
    first_uncertified.resize(n);
    std::vector<uint8_t> certified(links_per_config ? robot.hs.size() / links_per_config : 0);
    hfb_collision_request q;
    prepare(robot, request, q);
    std::vector<uint32_t> tpl;
    for (const auto& p : self_pairs) {
      tpl.push_back(p.first);
      tpl.push_back(p.second);
    }
    // empty vectors may hand out null data(), which the C ABI would take for outputs not asked for (or a missing
    // sweep); one slot stands in (nothing is read from or written to it)
    int32_t none = -1;
    double no_sweep = 0;
    hfb_certify_out o{first_invalid.data(), first_uncertified.data(), certified.data(), nullptr, nullptr, nullptr,
                      nullptr};
    if (n == 0) o.first_invalid = &none;
    C.check(hfb_env_certify_motions(C.raw(), env, robot.hs.size(), robot.hs.data(), robot.tfs.data(),
                                    sweep.empty() ? &no_sweep : sweep.data(), links_per_config, self_pairs.size(),
                                    tpl.data(), n, offsets.data(), 0, n, &q, &o));
    return certified;
  }

  /// A planner's progressive motion validation: motion m runs from q_from[m] to q_to[m] (n_motions x nq each) of the
  /// robot model, linear in q.  Each motion is cut into 2^initial_depth segments, certified as certify_motions
  /// certifies them, and the uncertified segments are split again, down to 2^-max_depth of the motion, with at most
  /// max_samples samples per round (hfb_env_validate_motions states the rounds and their guarantee).  Only motions
  /// [first_motion, first_motion + num_motions) are validated (num_motions = SIZE_MAX: the rest).  q of the wrong size,
  /// depths outside 0 <= initial_depth <= max_depth <= 30, max_samples < 2, a range past the end or a malformed
  /// template throw std::invalid_argument.
  MotionValidation validate_motions(RobotModel& robot, const std::vector<double>& q_from, const std::vector<double>& q_to,
                                    const std::vector<std::pair<uint32_t, uint32_t>>& self_pairs, uint32_t initial_depth,
                                    uint32_t max_depth, uint64_t max_samples,
                                    const CollisionRequest& request = CollisionRequest(), size_t first_motion = 0,
                                    size_t num_motions = SIZE_MAX) {
    if (request.num_max_contacts == 0 && request.security_margin != -std::numeric_limits<FCL_REAL>::infinity())
      throw std::invalid_argument("Invalid number of max contacts (current value is 0).");
    if (initial_depth > max_depth || max_depth > 30 || max_samples < 2)
      throw std::invalid_argument("need 0 <= initial_depth <= max_depth <= 30 and max_samples >= 2");
    if (q_from.size() % robot.nq_ || q_to.size() != q_from.size())
      throw std::invalid_argument("q_from, q_to: nq values per motion, as many motions in each");
    const size_t n = q_from.size() / robot.nq_;
    if (num_motions == SIZE_MAX) num_motions = first_motion <= n ? n - first_motion : 0;
    if (first_motion > n || num_motions > n - first_motion) throw std::invalid_argument("motion range past the end");
    hfb_collision_request q;
    detail::fill(request, q);
    std::vector<uint32_t> tpl;
    for (const auto& p : self_pairs) {
      tpl.push_back(p.first);
      tpl.push_back(p.second);
    }
    robot.sync();
    MotionValidation v;
    v.status.resize(n);
    v.t_valid.resize(n);
    v.t_collide.resize(n);
    v.kind.resize(n);
    v.first.resize(n);
    v.second.resize(n);
    v.contacts.resize(n);
    // no motions: the vectors may hand out null data(), which the C ABI refuses for the required outputs; one slot
    // each stands in (nothing is written to it)
    int8_t s0 = -1;
    double tv0 = 0, tc0 = -1;
    hfb_validate_out o{n ? v.status.data() : &s0, n ? v.t_valid.data() : &tv0, n ? v.t_collide.data() : &tc0,
                       v.kind.data(), v.first.data(), v.second.data(), v.contacts.data(), &v.n_rounds, &v.n_samples,
                       &v.n_env_candidates, &v.n_self_candidates, &v.n_unsupported};
    const hfb_validate_params p{initial_depth, max_depth, max_samples};
    C.check(hfb_env_validate_motions(C.raw(), env, robot.robot, n, q_from.data(), q_to.data(), self_pairs.size(),
                                     tpl.data(), first_motion, num_motions, &q, &p, &o));
    return v;
  }

 private:
  void check_motions(DynamicAABBTreeCollisionManager& robot, size_t links_per_config,
                     const std::vector<std::pair<uint32_t, uint32_t>>& self_pairs, const std::vector<uint32_t>& offsets,
                     const CollisionRequest& request, const hfb_motions_out& out) {
    hfb_collision_request q;
    prepare(robot, request, q);
    std::vector<uint32_t> tpl;
    for (const auto& p : self_pairs) {
      tpl.push_back(p.first);
      tpl.push_back(p.second);
    }
    const size_t n = offsets.size() - 1;
    // no motions: the callers' vectors are empty and may hand out null data(), which the C ABI would take for
    // outputs not asked for; one slot stands in (nothing is written to it)
    int32_t none = -1;
    hfb_motions_out o = out;
    if (n == 0) o.first_invalid = &none;
    C.check(hfb_env_collide_motions(C.raw(), env, robot.hs.size(), robot.hs.data(), robot.tfs.data(), links_per_config,
                                    self_pairs.size(), tpl.data(), n, offsets.data(), 0, n, &q, &o));
  }
  void distance_configs(DynamicAABBTreeCollisionManager& robot, size_t links_per_config,
                        const std::vector<std::pair<uint32_t, uint32_t>>& self_pairs, const DistanceRequest& request,
                        FCL_REAL max_distance, const hfb_configs_distance_out& out) {
    hfb_distance_request q;
    detail::fill(request, q);
    std::vector<uint32_t> tpl;
    for (const auto& p : self_pairs) {
      tpl.push_back(p.first);
      tpl.push_back(p.second);
    }
    const size_t n_configs = links_per_config ? robot.hs.size() / links_per_config : 0;
    C.check(hfb_env_distance_configs(C.raw(), env, robot.hs.size(), robot.hs.data(), robot.tfs.data(), links_per_config,
                                     self_pairs.size(), tpl.data(), 0, n_configs, &q, max_distance, &out));
  }
  size_t robot_size(DynamicAABBTreeCollisionManager& robot, FCL_REAL max_distance) {
    if (!(max_distance >= 0)) throw std::invalid_argument("max_distance must be >= 0 or inf");
    if (robot.stale) robot.refresh();
    return robot.hs.size();
  }
  void query_distance(DynamicAABBTreeCollisionManager& robot, const DistanceRequest& request, FCL_REAL max_distance,
                      const hfb_env_distance_out& out) {
    hfb_distance_request q;
    detail::fill(request, q);
    C.check(hfb_env_distance(C.raw(), env, robot.hs.size(), robot.hs.data(), robot.tfs.data(), 0, robot.hs.size(), &q,
                             max_distance, &out));
  }
  void check_configs(DynamicAABBTreeCollisionManager& robot, size_t links_per_config,
                     const std::vector<std::pair<uint32_t, uint32_t>>& self_pairs, const hfb_collision_request& q,
                     const hfb_configs_out& out) {
    std::vector<uint32_t> tpl;
    for (const auto& p : self_pairs) {
      tpl.push_back(p.first);
      tpl.push_back(p.second);
    }
    const size_t n_configs = links_per_config ? robot.hs.size() / links_per_config : 0;
    C.check(hfb_env_collide_configs(C.raw(), env, robot.hs.size(), robot.hs.data(), robot.tfs.data(), links_per_config,
                                    self_pairs.size(), tpl.data(), 0, n_configs, &q, &out));
  }
  void prepare(DynamicAABBTreeCollisionManager& robot, const CollisionRequest& request, hfb_collision_request& q) {
    if (request.num_max_contacts == 0 && request.security_margin != -std::numeric_limits<FCL_REAL>::infinity())
      throw std::invalid_argument("Invalid number of max contacts (current value is 0).");
    if (robot.stale) robot.refresh();
    detail::fill(request, q);
  }
  Context& C;
  hfb_env* env = nullptr;
  std::unordered_map<const CollisionObject*, uint32_t> index;
};

// ---------------------------------------------------------------- free functions
// collide(): src/collision.cpp:69-130 (results accumulate; callers clear()).
inline std::size_t collide(const CollisionGeometry* o1, const Transform3f& tf1, const CollisionGeometry* o2,
                           const Transform3f& tf2, const CollisionRequest& request, CollisionResult& result) {
  if (request.security_margin == -std::numeric_limits<FCL_REAL>::infinity()) {
    result.clear();
    return false;
  }
  if (request.num_max_contacts == 0) throw std::invalid_argument("Invalid number of max contacts (current value is 0).");
  if (request.isSatisfied(result)) return result.numContacts();  // shape_shape_func.h:139
  Context& C = Context::instance();
  const uint32_t h1 = C.handle(o1), h2 = C.handle(o2);
  C.commit();
  hfb_collision_request q;
  detail::fill(request, q);
  double gin[3] = {request.cached_gjk_guess[0], request.cached_gjk_guess[1], request.cached_gjk_guess[2]};
  int32_t hin[2] = {request.cached_support_func_guess[0], request.cached_support_func_guess[1]};
  q.q.cached_gjk_guess = gin;
  q.q.cached_support_func_guess = hin;
  double gout[3];
  int32_t hout[2];
  hfb_guess_out go{gout, hout};
  hfb_contact rec;
  const hfb_transform t1 = tf1.pod(), t2 = tf2.pod();
  // a mesh pair can have more than one contact (CollisionResult::contacts): fetch them all when asked to
  std::vector<hfb_contact> more;
  uint32_t count = 0;
  const bool mesh = isMeshType(o1->getNodeType()) || isMeshType(o2->getNodeType());
  if (mesh && request.num_max_contacts > 1) {
    more.resize(request.num_max_contacts - 1);
    C.check(hfb_batch_collide_contacts(C.raw(), 1, &h1, &t1, &h2, &t2, &q, &rec, (uint32_t)more.size(), more.data(),
                                       &count, &go));
    more.resize(count > 1 ? count - 1 : 0);
  } else {
    C.check(hfb_batch_collide(C.raw(), 1, &h1, &t1, &h2, &t2, &q, &rec, &go));
  }
  if (HFB_STATUS_PATH(rec.status) == HFB_PATH_UNSUPPORTED) detail::unsupported("Collision", o1, o2);
  if (rec.distance_lower_bound < result.distance_lower_bound) {  // collision_data.h:1186-1197
    result.distance_lower_bound = rec.distance_lower_bound;
    result.nearest_points = {{detail::v3(rec.p1), detail::v3(rec.p2)}};
    result.normal = detail::v3(rec.normal);
  }
  std::size_t res = 0;
  if (rec.num_contacts && result.numContacts() < request.num_max_contacts) {
    Contact c;
    c.o1 = o1;
    c.o2 = o2;
    c.b1 = rec.b1;
    c.b2 = rec.b2;
    c.normal = detail::v3(rec.normal);
    c.nearest_points = {{detail::v3(rec.p1), detail::v3(rec.p2)}};
    c.pos = detail::v3(rec.pos);
    c.penetration_depth = rec.distance;
    result.addContact(c);
    for (const hfb_contact& x : more) {
      if (!(result.numContacts() < request.num_max_contacts)) break;
      Contact d;
      d.o1 = o1;
      d.o2 = o2;
      d.b1 = x.b1;
      d.b2 = x.b2;
      d.normal = detail::v3(x.normal);
      d.nearest_points = {{detail::v3(x.p1), detail::v3(x.p2)}};
      d.pos = detail::v3(x.pos);
      d.penetration_depth = x.distance;
      result.addContact(d);
    }
    res = result.numContacts();
  }
  result.cached_gjk_guess = detail::v3(gout);  // collision.cpp:125-127
  result.cached_support_func_guess = {{hout[0], hout[1]}};
  request.updateGuess(result);
  return res;
}
inline std::size_t collide(const CollisionObject* o1, const CollisionObject* o2, const CollisionRequest& request,
                           CollisionResult& result) {
  return collide(o1->collisionGeometryPtr(), o1->getTransform(), o2->collisionGeometryPtr(), o2->getTransform(),
                 request, result);
}

// distance(): src/distance.cpp:60-109
inline FCL_REAL distance(const CollisionGeometry* o1, const Transform3f& tf1, const CollisionGeometry* o2,
                         const Transform3f& tf2, const DistanceRequest& request, DistanceResult& result) {
  if (request.isSatisfied(result)) return result.min_distance;  // shape_shape_func.h:57
  Context& C = Context::instance();
  const uint32_t h1 = C.handle(o1), h2 = C.handle(o2);
  C.commit();
  hfb_distance_request q;
  detail::fill(request, q);
  double gin[3] = {request.cached_gjk_guess[0], request.cached_gjk_guess[1], request.cached_gjk_guess[2]};
  int32_t hin[2] = {request.cached_support_func_guess[0], request.cached_support_func_guess[1]};
  q.q.cached_gjk_guess = gin;
  q.q.cached_support_func_guess = hin;
  double gout[3];
  int32_t hout[2];
  hfb_guess_out go{gout, hout};
  hfb_distance_result rec;
  const hfb_transform t1 = tf1.pod(), t2 = tf2.pod();
  C.check(hfb_batch_distance(C.raw(), 1, &h1, &t1, &h2, &t2, &q, &rec, &go));
  if (HFB_STATUS_PATH(rec.status) == HFB_PATH_UNSUPPORTED) detail::unsupported("Distance", o1, o2);
  const bool closed = HFB_STATUS_PATH(rec.status) == HFB_PATH_CLOSED_FORM;
  if (closed || result.min_distance > rec.min_distance) {  // DistanceResult::update, collision_data.h:1111-1124
    result.min_distance = rec.min_distance;
    result.o1 = o1;
    result.o2 = o2;
    result.b1 = rec.b1;
    result.b2 = rec.b2;
    result.nearest_points = {{detail::v3(rec.p1), detail::v3(rec.p2)}};
    result.normal = detail::v3(rec.normal);
  }
  result.cached_gjk_guess = detail::v3(gout);
  result.cached_support_func_guess = {{hout[0], hout[1]}};
  request.updateGuess(result);
  return rec.min_distance;
}
inline FCL_REAL distance(const CollisionObject* o1, const CollisionObject* o2, const DistanceRequest& request,
                         DistanceResult& result) {
  return distance(o1->collisionGeometryPtr(), o1->getTransform(), o2->collisionGeometryPtr(), o2->getTransform(),
                  request, result);
}

// functors (collision.h:79-117, distance.h:74-112): geometry handles are resolved once
class ComputeCollision {
 public:
  ComputeCollision(const CollisionGeometry* o1_, const CollisionGeometry* o2_) : o1(o1_), o2(o2_) {
    Context::instance().handle(o1);
    Context::instance().handle(o2);
  }
  std::size_t operator()(const Transform3f& tf1, const Transform3f& tf2, const CollisionRequest& request,
                         CollisionResult& result) const {
    return collide(o1, tf1, o2, tf2, request, result);
  }

 private:
  const CollisionGeometry* o1;
  const CollisionGeometry* o2;
};
class ComputeDistance {
 public:
  ComputeDistance(const CollisionGeometry* o1_, const CollisionGeometry* o2_) : o1(o1_), o2(o2_) {
    Context::instance().handle(o1);
    Context::instance().handle(o2);
  }
  FCL_REAL operator()(const Transform3f& tf1, const Transform3f& tf2, const DistanceRequest& request,
                      DistanceResult& result) const {
    return distance(o1, tf1, o2, tf2, request, result);
  }

 private:
  const CollisionGeometry* o1;
  const CollisionGeometry* o2;
};

}  // namespace hppfcl_b200
