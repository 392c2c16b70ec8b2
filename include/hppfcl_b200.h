/*
 * hppfcl_b200.h -- C-ABI of the batched narrow-phase engine (CUDA, NVIDIA H100).
 *
 * This is the drop-in boundary for the hot path of hpp-fcl
 * (collide()/distance() -> ShapeShapeDistance -> GJKSolver::shapeDistance ->
 * GJK::evaluate / EPA::evaluate, plus OBBRSS BVH traversal).  The reference has
 * no FFI of its own; its de-facto operator interface is the function-pointer
 * matrix and the two free functions:
 *
 *   CollisionFunc   include/hpp/fcl/collision_func_matrix.h:61-67
 *   DistanceFunc    include/hpp/fcl/distance_func_matrix.h:59-65
 *   collide(o1,tf1,o2,tf2,CollisionRequest,CollisionResult&)  include/hpp/fcl/collision.h:65-70
 *   distance(o1,tf1,o2,tf2,DistanceRequest,DistanceResult&)   include/hpp/fcl/distance.h:60-65
 *
 * Every entry point below is the batched form of one of those calls: plain
 * pointers and sizes, no C++ / torch types, int error codes (0 = ok), no
 * exceptions across the boundary.  Geometry (the reference's caller-owned
 * `const CollisionGeometry*`) is registered once into a device-resident arena
 * and referred to by a 32-bit handle; per pair the caller passes two handles
 * and two Transform3f-compatible poses.
 *
 * All floating point is IEEE binary64 (FCL_REAL = double,
 * include/hpp/fcl/data_types.h:66-71).
 */
#ifndef HPPFCL_B200_H
#define HPPFCL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- node types: numeric values mirror hpp::fcl::NODE_TYPE
 *      (include/hpp/fcl/collision_object.h:65-89) ------------------------- */
enum {
  HFB_BV_OBB = 2,    /* BVHModel<OBB>: collide() only, see hfb_geom_register_bvh_obb */
  HFB_BV_OBBRSS = 5,
  HFB_GEOM_BOX = 9,
  HFB_GEOM_SPHERE = 10,
  HFB_GEOM_CAPSULE = 11,
  HFB_GEOM_CONE = 12,
  HFB_GEOM_CYLINDER = 13,
  HFB_GEOM_CONVEX = 14,
  HFB_GEOM_PLANE = 15,     /* registered with hfb_geom_register_halfspaces */
  HFB_GEOM_HALFSPACE = 16, /* registered with hfb_geom_register_halfspaces */
  HFB_GEOM_TRIANGLE = 17,
  HFB_GEOM_ELLIPSOID = 19
};

/* ---- enums of include/hpp/fcl/data_types.h:85-98 ----------------------- */
enum { HFB_GUESS_DEFAULT = 0, HFB_GUESS_CACHED = 1, HFB_GUESS_BOUNDING_VOLUME = 2 };
enum { HFB_GJK_DEFAULT = 0, HFB_GJK_POLYAK = 1, HFB_GJK_NESTEROV = 2 };
enum { HFB_CRIT_DEFAULT = 0, HFB_CRIT_DUALITY_GAP = 1, HFB_CRIT_HYBRID = 2 };
enum { HFB_CRIT_RELATIVE = 0, HFB_CRIT_ABSOLUTE = 1 };

/* ---- GJK::Status (include/hpp/fcl/narrowphase/gjk.h:95-102) ------------ */
enum {
  HFB_GJK_DID_NOT_RUN = 0,
  HFB_GJK_FAILED = 1,
  HFB_GJK_NO_COLLISION_EARLY_STOPPED = 2,
  HFB_GJK_NO_COLLISION = 3,
  HFB_GJK_COLLISION_WITH_PENETRATION = 4,
  HFB_GJK_COLLISION = 5
};
/* ---- EPA::Status (gjk.h:330-341), stored as (value & 0xff) ------------- */
enum {
  HFB_EPA_DID_NOT_RUN = 0xff, /* -1 */
  HFB_EPA_FAILED = 0,
  HFB_EPA_VALID = 1,
  HFB_EPA_ACCURACY_REACHED = 3,
  HFB_EPA_DEGENERATED = 2,
  HFB_EPA_NON_CONVEX = 4,
  HFB_EPA_INVALID_HULL = 6,
  HFB_EPA_OUT_OF_FACES = 8,
  HFB_EPA_OUT_OF_VERTICES = 10,
  HFB_EPA_FALLBACK = 12
};

/* status word layout of hfb_distance_result.status / hfb_contact.status */
#define HFB_STATUS_GJK(s) ((s) & 0xffu)
#define HFB_STATUS_EPA(s) (((s) >> 8) & 0xffu)
#define HFB_STATUS_PATH(s) (((s) >> 16) & 0xffu)
enum { HFB_PATH_GJK = 0, HFB_PATH_CLOSED_FORM = 1, HFB_PATH_BVH = 2, HFB_PATH_UNSUPPORTED = 0xee };
/* HFB_PATH_UNSUPPORTED marks a record of a pair on which the reference throws: the record is the cleared
 * result (DistanceResult::clear / CollisionResult::clear) and a binding re-raises.  Cases: a type pair outside
 * the function matrices covered here (collision.cpp:110-117); collide() of a mesh with a negative security
 * margin (collision_func_matrix.cpp:109-112); a mesh-shape query whose shape has a swept-sphere radius
 * (geometric_shapes_utility.h:73-78); BoundingVolumeGuess on a mesh-shape query that evaluates a GJK leaf --
 * every distance(), a collide() whose walk reaches a leaf; sphere partners excepted (narrowphase.h:368-377). */

/* error codes */
enum {
  HFB_OK = 0,
  HFB_ERR_INVALID_ARGUMENT = 1, /* std::invalid_argument in the reference */
  HFB_ERR_NO_DEVICE = 2,        /* no CUDA device / extension unusable   */
  HFB_ERR_CUDA = 3,
  HFB_ERR_UNSUPPORTED_PAIR = 4, /* collision.cpp:110-117 "not yet supported" */
  HFB_ERR_OUT_OF_MEMORY = 5
};

/* ---- Transform3f (include/hpp/fcl/math/transform.h:56-216): R then T.
 *      R is COLUMN-major, exactly Eigen's Matrix3d storage, so a binding can
 *      memcpy tf.getRotation().data() and tf.getTranslation().data(). 96 B. */
typedef struct hfb_transform {
  double R[9];
  double T[3];
} hfb_transform;

/* ---- one shape record (40 B), the flattened ShapeBase subclass
 *      (include/hpp/fcl/shape/geometric_shapes.h:164-634):
 *        BOX        p = halfSide
 *        SPHERE     p[0] = radius
 *        CAPSULE    p[0] = radius, p[1] = halfLength
 *        CONE       p[0] = radius, p[1] = halfLength
 *        CYLINDER   p[0] = radius, p[1] = halfLength
 *        ELLIPSOID  p = radii
 *        CONVEX     data = convex id (see hfb_geom_register_convex)
 *        TRIANGLE   data = convex id of a 3-point vertex set (a,b,c)
 *      ssr = ShapeBase::getSweptSphereRadius()                             */
typedef struct hfb_shape {
  uint32_t type;
  uint32_t data;
  double p[3];
  double ssr;
} hfb_shape;

/* ---- QueryRequest (include/hpp/fcl/collision_data.h:171-274) ----------- */
typedef struct hfb_query_request {
  int32_t gjk_initial_guess;              /* HFB_GUESS_*            default DEFAULT */
  int32_t gjk_variant;                    /* HFB_GJK_*              default DEFAULT */
  int32_t gjk_convergence_criterion;      /* HFB_CRIT_*             default DEFAULT */
  int32_t gjk_convergence_criterion_type; /* HFB_CRIT_RELATIVE/ABS  default RELATIVE */
  uint32_t gjk_max_iterations;            /* 128 */
  uint32_t epa_max_iterations;            /* 64; more is refused with HFB_ERR_INVALID_ARGUMENT: the EPA polytope lives
                                           * in shared memory, sized for the reference's default of 64 iterations
                                           * (68 vertices, 132 faces) */
  double gjk_tolerance;                   /* 1e-6 */
  double epa_tolerance;                   /* 1e-6 */
  double collision_distance_threshold;    /* 1e-12 (Eigen dummy_precision) */
  /* optional per-pair warm start (QueryRequest::cached_gjk_guess /
   * cached_support_func_guess, collision_data.h:180-184); NULL => (1,0,0),(0,0).
   * Host pointers for the host entry points, device pointers for *_device. */
  const double* cached_gjk_guess;           /* n x 3 */
  const int32_t* cached_support_func_guess; /* n x 2 */
} hfb_query_request;

/* ---- DistanceRequest (collision_data.h:987-1050) ----------------------- */
typedef struct hfb_distance_request {
  hfb_query_request q;
  int32_t enable_signed_distance; /* default 1 */
  int32_t enable_nearest_points;  /* default 1; read by the mesh-mesh walk only: when 0 the nearest
                                     points stay in the first mesh's frame (traversal_node_bvhs.h:527-536) */
  /* carried for layout parity with DistanceRequest; like in the reference they do not influence any
   * OBBRSS walk: the mesh-shape traversal node zeroes its copies in its constructor
   * (internal/traversal_node_bvh_shape.h:294-295), the mesh-mesh node takes them from its own default
   * request before the caller's is stored (internal/traversal_node_bvhs.h:409-410) */
  double rel_err;
  double abs_err;
} hfb_distance_request;

/* ---- CollisionRequest (collision_data.h:312-383) ----------------------- */
typedef struct hfb_collision_request {
  hfb_query_request q;
  uint32_t num_max_contacts; /* default 1 (the batch path returns <= 1 per pair) */
  int32_t enable_contact;    /* default 1 */
  double security_margin;    /* default 0 */
  double break_distance;     /* default 1e-3 */
  double distance_upper_bound; /* default +DBL_MAX */
} hfb_collision_request;

/* ---- DistanceResult (collision_data.h:1053-1096) as a flat 96 B record:
 *      min_distance, nearest_points[2], normal, b1, b2 (+ status, iterations,
 *      and the warm-start outputs QueryResult::cached_* when requested).   */
typedef struct hfb_distance_result {
  double min_distance;
  double p1[3];
  double p2[3];
  double normal[3];
  int32_t b1, b2;      /* -1 (NONE) for primitives, triangle id for meshes */
  uint32_t status;     /* HFB_STATUS_* */
  uint32_t iterations; /* gjk | epa << 16 */
} hfb_distance_result;

/* ---- one collide() outcome: CollisionResult with <= 1 Contact
 *      (collision_data.h:59-166, 391-509).  distance = signed distance
 *      (= Contact::penetration_depth), distance_lower_bound as the reference
 *      sets it in updateDistanceLowerBoundFromLeaf (:1186-1197). 136 B.    */
typedef struct hfb_contact {
  double distance;
  double p1[3];
  double p2[3];
  double normal[3];
  double pos[3];
  double distance_lower_bound;
  int32_t b1, b2;
  uint32_t status;
  uint32_t num_contacts; /* 0 or 1: the collide() return value */
  uint32_t iterations;
  uint32_t _pad;
} hfb_contact;

/* optional warm-start outputs (QueryResult::cached_gjk_guess,
 * cached_support_func_guess; collision.cpp:125-127) */
typedef struct hfb_guess_out {
  double* cached_gjk_guess;           /* n x 3 or NULL */
  int32_t* cached_support_func_guess; /* n x 2 or NULL */
} hfb_guess_out;

typedef struct hfb_ctx hfb_ctx;

/* ---- lifetime ---------------------------------------------------------- */
/* Creates a context bound to CUDA device `device`. Fails with
 * HFB_ERR_NO_DEVICE when there is no usable GPU: there is no CPU fallback.
 * Threading: a context is thread-compatible, not thread-safe -- one thread at a time per context,
 * any number of contexts (one per GPU, or several per GPU) in a process.  The reference's collide() /
 * distance() are re-entrant because every call builds its solver on the stack; here the per-call
 * state (streams, scratch buffers, the EPA queue) lives in the context.  The host entry points block
 * until the results are in the caller's buffers; the *_device entry points enqueue on the caller's
 * stream and return, the results are ready when that stream reaches the point of the call.
 * Streams: the *_device calls of one context share its scratch, so they run one at a time on the device -- a
 * call enqueued on a different stream than the context's previous *_device call first waits (on the device,
 * cudaStreamWaitEvent) for that call; use one context per stream for concurrent batches.  Device handles are
 * trusted up to the arena size: a handle >= hfb_geom_num_shapes() is answered with HFB_PATH_UNSUPPORTED in the
 * pair's record, never dereferenced. */
int hfb_ctx_create(int device, hfb_ctx** out);
void hfb_ctx_destroy(hfb_ctx* ctx);
const char* hfb_last_error(const hfb_ctx* ctx);
/* library self-description; callable without a GPU */
const char* hfb_version(void);
void hfb_default_distance_request(hfb_distance_request* r);
void hfb_default_collision_request(hfb_collision_request* r);

/* ---- geometry arena (replaces caller-owned `const CollisionGeometry*`) -- */
/* Registers `n` primitive shape records; handles_out[i] is the handle of
 * shapes[i]. CONVEX/TRIANGLE records must carry a convex id from
 * hfb_geom_register_convex. */
int hfb_geom_register_shapes(hfb_ctx* ctx, const hfb_shape* shapes, size_t n,
                             uint32_t* handles_out);
/* Registers `count` Halfspace (type = HFB_GEOM_HALFSPACE: the points with n.x <= d) or Plane
 * (HFB_GEOM_PLANE: n.x = d) geometries (geometric_shapes.h:885-1031).  n_d = count x 4 doubles
 * (n.x, n.y, n.z, d), normalised here as the reference's constructors do (unitNormalTest,
 * geometric_shapes.cpp:121-143); ssr = count swept-sphere radii or NULL.  handles_out[i] is the handle
 * of record i.  Such a geometry is closed-form against every primitive, ConvexBase, TriangleP and
 * another plane or halfspace, in either operand order (details::halfspaceDistance / planeDistance /
 * halfspaceHalfspaceDistance / halfspacePlaneDistance / planePlaneDistance, src/narrowphase/details.h:
 * 343-693, through the ShapeShapeDistance specialisations of src/distance/<shape>_halfspace.cpp and
 * <shape>_plane.cpp); against a BVH model the pair comes back as HFB_PATH_UNSUPPORTED.  Box partners: the
 * reference's box support has a process-wide `inflate` static fixed by the first direction ever asked for
 * (support_functions.cpp:146); this library computes with 1 + 1e-10, its value whenever that first
 * direction had a zero component (a floor).  hfb_geom_register_shapes refuses these two types (a 40-byte
 * record has no room for n and d). */
int hfb_geom_register_halfspaces(hfb_ctx* ctx, uint32_t type, const double* n_d, const double* ssr,
                                 size_t count, uint32_t* handles_out);
/* Registers the vertex set of a ConvexBase (geometric_shapes.h:638-872):
 * `points` = num_points x 3 doubles. Returns the convex id in *convex_id. */
int hfb_geom_register_convex(hfb_ctx* ctx, const double* points,
                             uint32_t num_points, uint32_t* convex_id);
/* `count` vertex sets of `num_points` vertices each, back to back in `points`; their ids are
 * first_id, first_id + 1, ... (one call instead of `count`). */
int hfb_geom_register_convex_batch(hfb_ctx* ctx, const double* points, uint32_t num_points,
                                   uint32_t count, uint32_t* first_id);
/* Registers a BVHModel<OBBRSS> (include/hpp/fcl/BVH/BVH_model.h:315-496,
 * BV/BV_node.h:52-148, BV/OBBRSS.h) built on the host: `nodes` = num_nodes
 * records of hfb_bvh_node, vertices num_vertices x 3, triangles num_tris x 3. */
typedef struct hfb_bvh_node {
  int32_t first_child;      /* <0: leaf, primitive id = -(first_child+1) */
  uint32_t first_primitive;
  uint32_t num_primitives;
  uint32_t _pad;
  double obb_axes[9];   /* OBB::axes, column-major */
  double obb_To[3];     /* OBB::To     */
  double obb_extent[3]; /* OBB::extent */
  double rss_axes[9];   /* RSS::axes, column-major */
  double rss_Tr[3];     /* RSS::Tr     */
  double rss_length[2]; /* RSS::length */
  double rss_radius;    /* RSS::radius */
} hfb_bvh_node;
/* Returns the BVH id in *bvh_id; a shape record {type = HFB_BV_OBBRSS, data = bvh id}
 * registered with hfb_geom_register_shapes gives the handle used in batches.  Supported
 * partners: the primitive shapes and ConvexBase (mesh-shape distance and collide, either
 * operand order: BVHShapeCollider / BVHShapeDistancer<OBBRSS, S>, collision_func_matrix.cpp:
 * 97-186, distance_func_matrix.cpp:77-127) and another BVHModel<OBBRSS> (mesh-mesh:
 * BVHCollide<OBBRSS> collision_func_matrix.cpp:248-257, BVHDistance<OBBRSS>
 * distance_func_matrix.cpp:259-268; both contact primitive ids b1, b2 are returned, the
 * normal of a mesh-mesh distance is NaN as the reference never writes it). */
/* Host-side tree builder, no context or GPU involved: BVHModel<OBBRSS>::endModel() for a triangle
 * model with the default SPLIT_METHOD_MEAN (src/BVH/BVH_model.cpp:860-960, BV_fitter.cpp:501-531,
 * BV_splitter.cpp:80-118,242-278).  Writes 2 * num_triangles - 1 nodes, bit-identical to the
 * reference's BVHModel::bvs for the same vertices/triangles; pass them to
 * hfb_geom_register_bvh_obbrss.  A caller that already holds a reference BVHModel passes its bvs
 * instead and never calls this. */
int hfb_bvh_build_obbrss(const double* vertices, uint32_t num_vertices, const uint32_t* triangles,
                         uint32_t num_triangles, hfb_bvh_node* nodes_out, uint32_t nodes_capacity);
int hfb_geom_register_bvh_obbrss(hfb_ctx* ctx, const hfb_bvh_node* nodes,
                                 uint32_t num_nodes, const double* vertices,
                                 uint32_t num_vertices, const uint32_t* triangles,
                                 uint32_t num_triangles, uint32_t* bvh_id);
/* A plain BVHModel<OBB> (collision_func_matrix.cpp:488-501, 652: BVHShapeCollider<OBB, S>, BVHCollide<OBB>): the same
 * node records with the RSS half ignored -- BVFitter<OBB>::fit and the mean splitter over OBB::axes.col(0)
 * (BV_fitter.cpp:480-499, BV_splitter.cpp:44-46,163-170) produce exactly the OBB half of the OBBRSS tree of the same
 * mesh, so hfb_bvh_build_obbrss serves both.  A shape record {type = HFB_BV_OBB, data = bvh id} gives the handle.
 * collide(): mesh-shape and mesh-mesh (both operands plain OBB models), the OBB tests and the leaf tests of the
 * OBBRSS walks.  distance() on a BVHModel<OBB> is NOT offered (HFB_PATH_UNSUPPORTED): the reference has no OBB
 * distance (OBB::distance prints "OBB distance not implemented" and returns 0, BV/OBB.cpp), so its generic walk
 * visits every triangle of a tree it first REBUILDS from the transformed vertices on every call
 * (traversal_node_setup.h:709-723) -- not a path to accelerate; use the OBBRSS model for distances. */
int hfb_geom_register_bvh_obb(hfb_ctx* ctx, const hfb_bvh_node* nodes, uint32_t num_nodes, const double* vertices,
                              uint32_t num_vertices, const uint32_t* triangles, uint32_t num_triangles,
                              uint32_t* bvh_id);
/* Uploads everything registered so far to the device. Must be called before
 * the first query and after any further registration. */
int hfb_geom_commit(hfb_ctx* ctx);
/* Device pointers of the committed arena (for NCCL broadcast by the host
 * layer): shape table, point pool, convex descriptors. */
int hfb_geom_device_arena(hfb_ctx* ctx, void** base, size_t* bytes);
size_t hfb_geom_num_shapes(const hfb_ctx* ctx);
/* Empties the arena: every shape handle, convex id and BVH id issued so far becomes invalid.  The
 * reference has no counterpart (geometry is caller-owned and passed by pointer on every call); this
 * is how a long-running caller of the batch ABI drops geometry it no longer queries. */
int hfb_geom_clear(hfb_ctx* ctx);
/* In-place changes of registered geometry (the reference's callers mutate the CollisionGeometry they own:
 * Box::halfSide, Sphere::radius, ConvexBase::points, setSweptSphereRadius ... and pass it again).  Handles
 * and ids stay valid; hfb_geom_commit must follow before the next query.
 *   update_shapes:  the records of `handles[i]` are replaced by `shapes[i]` (validated like a registration);
 *   update_convex:  vertex set `convex_id` replaced by `points` (same number of points);
 *   release_shapes: the handles are retired -- a pair that still names one comes back with
 *                   HFB_PATH_UNSUPPORTED; the storage of hulls and meshes is reclaimed by hfb_geom_clear. */
int hfb_geom_update_shapes(hfb_ctx* ctx, const uint32_t* handles, const hfb_shape* shapes, size_t n);
int hfb_geom_update_convex(hfb_ctx* ctx, uint32_t convex_id, const double* points, uint32_t num_points);
int hfb_geom_release_shapes(hfb_ctx* ctx, const uint32_t* handles, size_t n);

/* ---- batched distance(): n independent (o1,tf1,o2,tf2) queries --------- */
/* HOST buffers in/out; blocking.  Mirrors distance() of src/distance.cpp:60-109
 * applied to each pair with a fresh DistanceResult.  Pinned host buffers make the
 * copies asynchronous.  A batch is pipelined: uploads, kernels and downloads of its
 * chunks overlap (large plain calls: the whole batch on the device, EPA once for all
 * chunks; calls with warm-start or all-contacts outputs and the compact modes: every
 * chunk run to the end on one of four streams).  Handles are validated on the host
 * while the GPU already works: a bad one fails the call (the results are then
 * undefined), never the device. */
int hfb_batch_distance(hfb_ctx* ctx, size_t n, const uint32_t* h1,
                       const hfb_transform* tf1, const uint32_t* h2,
                       const hfb_transform* tf2, const hfb_distance_request* req,
                       hfb_distance_result* out, const hfb_guess_out* guess_out);
/* DEVICE buffers in/out; asynchronous on `cuda_stream` (a cudaStream_t). */
int hfb_batch_distance_device(hfb_ctx* ctx, size_t n, const uint32_t* d_h1,
                              const hfb_transform* d_tf1, const uint32_t* d_h2,
                              const hfb_transform* d_tf2,
                              const hfb_distance_request* req,
                              hfb_distance_result* d_out,
                              const hfb_guess_out* d_guess_out, void* cuda_stream);

/* collide() keeping every contact of a mesh pair (CollisionResult::contacts, up to request.num_max_contacts;
 * collision_data.h:431).  `out` is what hfb_batch_collide returns (contacts[0], the lower bound, the status);
 * counts[i] = numContacts() of pair i (0 or 1 for a shape pair); contacts[k], 1 <= k < min(counts[i], max_extra + 1),
 * are extra[i * max_extra + k - 1]: b1, b2, normal, p1, p2, pos and distance (= Contact::penetration_depth) set,
 * num_contacts = 1.  Contacts beyond max_extra + 1 are counted, not stored.  HOST buffers; blocking. */
int hfb_batch_collide_contacts(hfb_ctx* ctx, size_t n, const uint32_t* h1, const hfb_transform* tf1,
                               const uint32_t* h2, const hfb_transform* tf2,
                               const hfb_collision_request* req, hfb_contact* out, uint32_t max_extra,
                               hfb_contact* extra, uint32_t* counts, const hfb_guess_out* guess_out);
/* ---- batched collide(): mirrors collide() of src/collision.cpp:69-130 --- */
int hfb_batch_collide(hfb_ctx* ctx, size_t n, const uint32_t* h1,
                      const hfb_transform* tf1, const uint32_t* h2,
                      const hfb_transform* tf2, const hfb_collision_request* req,
                      hfb_contact* out, const hfb_guess_out* guess_out);
int hfb_batch_collide_device(hfb_ctx* ctx, size_t n, const uint32_t* d_h1,
                             const hfb_transform* d_tf1, const uint32_t* d_h2,
                             const hfb_transform* d_tf2,
                             const hfb_collision_request* req, hfb_contact* d_out,
                             const hfb_guess_out* d_guess_out, void* cuda_stream);

/* ---- broadphase feed: scene boxes and the overlapping pairs (BASELINE config 5) -------------------------
 * hfb_scene_aabbs: CollisionObject::computeAABB (include/hpp/fcl/collision_object.h:258-278) of n objects over
 * the aabb_local of their geometry (computeLocalAABB: src/shape/geometric_shapes.cpp:145-260, BVH_model.cpp);
 * aabbs: 6 doubles per object (min xyz, max xyz).
 * hfb_broadphase_pairs: every pair i < j whose boxes overlap (AABB::overlap, closed intervals: BV/AABB.h:111-118)
 * -- the set of pairs BroadPhaseCollisionManager::collide(callback) hands to its callback
 * (src/broadphase/broadphase_dynamic_AABB_tree.cpp:336-407,716-721), in no particular order; all of them are
 * counted in *n_pairs, at most `capacity` stored.  The pair list is what hfb_batch_*_objects takes.
 * The first two are HOST functions (no GPU work; hfb_broadphase_pairs needs no context at all); the _device forms
 * take and leave everything on the device, asynchronous on `cuda_stream` (the count is a device word). */
int hfb_scene_aabbs(hfb_ctx* ctx, size_t n_objects, const uint32_t* handles, const hfb_transform* tfs, double* aabbs);
int hfb_broadphase_pairs(size_t n_objects, const double* aabbs, uint32_t* first, uint32_t* second, size_t capacity,
                         size_t* n_pairs);
int hfb_scene_aabbs_device(hfb_ctx* ctx, size_t n_objects, const uint32_t* d_handles, const hfb_transform* d_tfs,
                           double* d_aabbs, void* cuda_stream);
/* [first_object, first_object + num_first_objects): the pairs (i, j), i < j, whose SMALLER index i lies in this
 * range (pass 0 and n_objects for all of them) -- the way a scene is cut over several GPUs: every rank holds all the
 * boxes and reports the pairs of its own range of objects. */
int hfb_broadphase_pairs_device(hfb_ctx* ctx, size_t n_objects, const double* d_aabbs, size_t first_object,
                                size_t num_first_objects, uint32_t* d_first, uint32_t* d_second, size_t capacity,
                                uint32_t* d_n_pairs, void* cuda_stream);

/* Broadphase and narrow phase of a scene in ONE call: the batched form of BroadPhaseCollisionManager::collide(callback)
 * with the default collision callback (broadphase/default_broadphase_callbacks.h:69-130 -- collide() of every candidate
 * pair, contacts collected).  HOST buffers; blocking.  Between the upload of the poses and the download of the
 * colliding pairs everything happens on the device: boxes, grid + sweep, collide() of the candidates (as
 * hfb_batch_collide_objects), compaction.  The colliding pairs (object indices, first < second) and their records
 * come back in no particular order, at most `capacity` of them; *n_candidates = pairs with overlapping boxes,
 * *n_colliding = pairs with a contact.  [first_object, first_object + num_first_objects) as in
 * hfb_broadphase_pairs_device: the candidates whose smaller index lies there (one GPU's share of the scene). */
typedef struct hfb_scene_contacts {
  uint32_t* first;
  uint32_t* second;
  hfb_contact* contacts;
  uint32_t capacity;
  uint32_t* n_colliding;
  uint32_t* n_candidates;
} hfb_scene_contacts;
int hfb_scene_collide(hfb_ctx* ctx, size_t n_objects, const uint32_t* object_handles, const hfb_transform* object_tfs,
                      size_t first_object, size_t num_first_objects, const hfb_collision_request* req,
                      const hfb_scene_contacts* out);

/* ---- object-table batches: the batched form of the CollisionObject overloads --------------------------
 * collide(const CollisionObject* o1, const CollisionObject* o2, ...) / distance(...) (include/hpp/fcl/collision.h:
 * 58-61, distance.h:53-56) take their geometry and pose from the objects.  A scene here is a table of objects
 * (geometry handle + pose, the two things a CollisionObject holds: collision_object.h:214-330) and a list of
 * pairs of table indices -- what a broadphase manager's collide()/distance() callback receives
 * (broadphase/default_broadphase_callbacks.h:224-252).  The host sends 100 B per object and 8 B per pair instead
 * of 200 B per pair; the pairs are expanded on the device.  Results are those of hfb_batch_distance /
 * hfb_batch_collide on the expanded rows, bit for bit.  An object index >= n_objects is an invalid argument. */
typedef struct hfb_object_pairs {
  size_t n_objects;
  const uint32_t* object_handles;   /* n_objects shape handles */
  const hfb_transform* object_tfs;  /* n_objects poses */
  size_t n_pairs;
  const uint32_t* first;   /* n_pairs indices into the object table: o1 of pair k */
  const uint32_t* second;  /*                                         o2 of pair k */
} hfb_object_pairs;
/* HOST buffers; blocking.  `out` (full 96-byte records) and `min_distance_out` (DistanceResult::min_distance only,
 * 8 bytes per pair back over PCIe) may each be null, not both. */
int hfb_batch_distance_objects(hfb_ctx* ctx, const hfb_object_pairs* scene, const hfb_distance_request* req,
                               hfb_distance_result* out, double* min_distance_out, const hfb_guess_out* guess_out);
/* compact collide() results: bit k of flags[k / 32] = CollisionResult::isCollision() of pair k; the records of the
 * colliding pairs (as hfb_batch_collide writes them) are appended to `contacts`, their pair indices to `pair_ids`,
 * in no particular order, at most `capacity` of them; *n_colliding counts all of them. */
typedef struct hfb_compact_contacts {
  uint32_t* flags;       /* (n_pairs + 31) / 32 words */
  uint32_t* n_colliding;
  uint32_t* pair_ids;    /* capacity */
  hfb_contact* contacts; /* capacity */
  uint32_t capacity;
} hfb_compact_contacts;
/* `out` (full records) and `compact` may each be null, not both. */
int hfb_batch_collide_objects(hfb_ctx* ctx, const hfb_object_pairs* scene, const hfb_collision_request* req,
                              hfb_contact* out, const hfb_compact_contacts* compact, const hfb_guess_out* guess_out);
/* every pointer inside *d_scene, d_out and d_guess_out are DEVICE pointers (the struct itself is read on the host);
 * asynchronous on `cuda_stream`.  Indices are not validated: one past the table gives HFB_PATH_UNSUPPORTED. */
int hfb_batch_distance_objects_device(hfb_ctx* ctx, const hfb_object_pairs* d_scene, const hfb_distance_request* req,
                                      hfb_distance_result* d_out, const hfb_guess_out* d_guess_out, void* cuda_stream);
int hfb_batch_collide_objects_device(hfb_ctx* ctx, const hfb_object_pairs* d_scene, const hfb_collision_request* req,
                                     hfb_contact* d_out, const hfb_guess_out* d_guess_out, void* cuda_stream);

/* ---- batched ConvexBase support function (the convex-support kernel):
 *      for each query i: argmax_v <dir_i, v> over the vertices of convex
 *      convex_ids[i]  (getShapeSupportLinear, support_functions.cpp:401-421;
 *      strict '>' => lowest index on ties).  index_out[i] = vertex index,
 *      support_out[i] = the vertex. */
int hfb_batch_convex_support(hfb_ctx* ctx, size_t n, const uint32_t* convex_ids,
                             const double* dirs, int32_t* index_out,
                             double* support_out);
int hfb_batch_convex_support_device(hfb_ctx* ctx, size_t n,
                                    const uint32_t* d_convex_ids,
                                    const double* d_dirs, int32_t* d_index_out,
                                    double* d_support_out, void* cuda_stream);

/* ---- multi-GPU: one context per GPU, pairs sharded over the ranks ---------------------------------------------
 * The path shards trivially (independent pairs, SURVEY 8e): there are exactly two collectives -- one broadcast of
 * the geometry arena per scene and one all-gather of the result records per batch -- and both live here, behind
 * the C-ABI, so that a C++ caller (hpp-fcl itself) can use a whole 8-GPU box.  NCCL is loaded with dlopen at the
 * first hfb_comm_* call (no link-time dependency).
 *   rank 0:      hfb_comm_unique_id(&id); hand `id` (128 bytes) to the other ranks by any means (MPI, a file, ...)
 *   every rank:  hfb_ctx_create(gpu, &ctx); hfb_comm_init(ctx, &id, rank, nranks);
 *   rank 0:      registers the geometry;      every rank: hfb_geom_broadcast(ctx, 0)   (commits on every rank)
 *   every rank:  hfb_batch_distance_sharded_device(ctx, n_local, rows of ITS pairs..., &d_all, stream)
 * d_all: the records of all ranks' pairs, rank-major (nranks * n_local), in one of two buffers the context owns;
 * the all-gather runs on the communicator's own stream and overlaps the next call's kernels; the buffer is complete
 * when `stream` has passed hfb_comm_wait(ctx, stream), and is reused by the next call but one. */
typedef struct hfb_comm_id {
  char bytes[128];
} hfb_comm_id;
int hfb_comm_unique_id(hfb_comm_id* id);
int hfb_comm_init(hfb_ctx* ctx, const hfb_comm_id* id, int rank, int nranks);
int hfb_comm_destroy(hfb_ctx* ctx);
int hfb_geom_broadcast(hfb_ctx* ctx, int root);
int hfb_batch_distance_sharded_device(hfb_ctx* ctx, size_t n_local, const uint32_t* d_h1, const hfb_transform* d_tf1,
                                      const uint32_t* d_h2, const hfb_transform* d_tf2, const hfb_distance_request* req,
                                      hfb_distance_result** d_all, void* cuda_stream);
int hfb_batch_collide_sharded_device(hfb_ctx* ctx, size_t n_local, const uint32_t* d_h1, const hfb_transform* d_tf1,
                                     const uint32_t* d_h2, const hfb_transform* d_tf2, const hfb_collision_request* req,
                                     hfb_contact** d_all, void* cuda_stream);
int hfb_comm_wait(hfb_ctx* ctx, void* cuda_stream);

/* ---- counters (mirror enable_statistics num_bv_tests / num_leaf_tests,
 *      traversal_node_bvh_shape.h:91-93) and launch accounting ------------ */
typedef struct hfb_stats {
  uint64_t kernel_launches; /* kernels launched by this ctx since creation */
  uint64_t pairs_processed;
  uint64_t epa_pairs;       /* pairs that went through the EPA kernel */
  uint64_t bv_tests;
  uint64_t leaf_tests;
  uint64_t watchdog_trips;  /* must stay 0: a block of the mesh-shape walk gave up waiting for work (its results are incomplete) */
} hfb_stats;
int hfb_get_stats(hfb_ctx* ctx, hfb_stats* out);

/* optional per-kernel device timing (CUDA events recorded on the launching stream
 * around every kernel launch; the reference's counterpart is request.enable_timings
 * -> result.timings, collision.cpp:196-201).  Off by default. */
typedef struct hfb_kernel_times {
  double pairs_ms;   /* sum over launches of the GJK-routed primitive-pair kernel (phase 1) */
  double epa_ms;     /* sum over launches of the EPA kernel */
  double other_ms;   /* classify / support / clear */
  uint64_t pairs_launches;
  uint64_t epa_launches;
  uint64_t other_launches;
  double closed_ms;  /* closed-form pair kernel */
  double convex_ms;  /* lane-group kernel for pairs touching ConvexBase / TriangleP */
  uint64_t closed_launches;
  uint64_t convex_launches;
  double bvh_ms;     /* OBBRSS mesh-shape traversal kernel */
  uint64_t bvh_launches;
} hfb_kernel_times;
int hfb_set_profiling(hfb_ctx* ctx, int enable);
int hfb_get_kernel_times(hfb_ctx* ctx, hfb_kernel_times* out, int reset);

#ifdef __cplusplus
}
#endif
#endif /* HPPFCL_B200_H */
