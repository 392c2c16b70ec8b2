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

/* ---- broadphase between two object sets: BroadPhaseCollisionManager::collide(other_manager, callback) and
 * collide(obj, callback) (include/hpp/fcl/broadphase/broadphase_collision_manager.h:94-118) ----------------------
 * The candidates are every (i, j), i in set A, j in set B, whose boxes overlap (AABB::overlap, closed intervals) --
 * the set NaiveCollisionManager::collide(other) reports (src/broadphase/broadphase_bruteforce.cpp:150-170), with
 * first = i (index in A) and second = j (index in B): o1 from the manager called, o2 from `other`.  Objects without a
 * box take no part; halfspaces and planes take part with their unbounded boxes (DynamicAABBTreeCollisionManager's
 * tighter halfspace leaf test, AABB::overlap(const Halfspace&), is not reproduced, as in the self form).  In no
 * particular order; all counted in *n_pairs, at most `capacity` stored.
 * hfb_broadphase_cross_pairs: HOST function, no context.  hfb_broadphase_cross_pairs_device: DEVICE buffers,
 * asynchronous on `cuda_stream` (the count is a device word); only the A objects in [first_a, first_a + num_a) --
 * one GPU's share of the configurations -- report their pairs. */
int hfb_broadphase_cross_pairs(size_t n_a, const double* aabbs_a, size_t n_b, const double* aabbs_b, uint32_t* first,
                               uint32_t* second, size_t capacity, size_t* n_pairs);
int hfb_broadphase_cross_pairs_device(hfb_ctx* ctx, size_t n_a, const double* d_aabbs_a, size_t first_a, size_t num_a,
                                      size_t n_b, const double* d_aabbs_b, uint32_t* d_first, uint32_t* d_second,
                                      size_t capacity, uint32_t* d_n_pairs, void* cuda_stream);
/* Broadphase and narrow phase of set A against set B in ONE call, as hfb_scene_collide does for one set: HOST buffers,
 * blocking; boxes, cross pairs, collide() of every candidate (o1 from A, o2 from B, as hfb_batch_collide_objects over
 * the table [A; B]) and compaction on the device.  out->first = index in A, out->second = index in B; candidates and
 * colliding pairs are all counted.  [first_a, first_a + num_a) as in hfb_broadphase_cross_pairs_device. */
int hfb_scene_collide_sets(hfb_ctx* ctx, size_t n_a, const uint32_t* handles_a, const hfb_transform* tfs_a, size_t n_b,
                           const uint32_t* handles_b, const hfb_transform* tfs_b, size_t first_a, size_t num_a,
                           const hfb_collision_request* req, const hfb_scene_contacts* out);

/* ---- resident environment: set B kept on the device across hfb_scene_collide_sets-style queries -----------------
 * The reference's managers are set up once and queried many times (DynamicAABBTreeCollisionManager::setup(), then
 * update(obj) / update(objs) for the objects that moved: broadphase_dynamic_AABB_tree.cpp:587-647).  An hfb_env holds
 * set B's object table, its boxes and the cross grid over them on the device, so a query uploads only A.  B's boxes are
 * a snapshot taken at create / update time, as the reference's tree is; the narrow phase uses the current geometry
 * and B's stored poses.
 *   hfb_env_create:  HOST buffers; B's handles are validated as hfb_scene_collide_sets validates them.
 *   hfb_env_update:  new poses of m objects of B (indices into B, HOST buffers): the reference's update(objs).  An index
 *                    out of range or repeated is HFB_ERR_INVALID_ARGUMENT and changes nothing.
 *   hfb_env_collide: HOST buffers, blocking.  What hfb_scene_collide_sets(A, B) returns for the same inputs (o1 from A,
 *                    o2 from B, the same counts, [first_a, first_a + num_a) the same way).
 *   hfb_env_collide_device: A's handles and poses and every output in DEVICE memory, ordered on `cuda_stream`; the
 *                    call blocks once, for the candidate count that sizes the narrow phase, and once more, on
 *                    `cuda_stream`, when A has more objects than any query before and the env's table regrows.
 *   hfb_env_destroy: frees it; hfb_ctx_destroy frees the envs a context still owns.
 * After a later hfb_geom_commit, B's handles are checked again before the next query: a handle released since is
 * HFB_ERR_INVALID_ARGUMENT.  After hfb_geom_clear every env of the context is refused until it is destroyed. */
typedef struct hfb_env hfb_env;
/* hfb_scene_contacts plus `flags` (may be null): flags[i] = 1 iff A object i has at least one colliding candidate pair,
 * for all n_a objects (0 outside [first_a, first_a + num_a)) -- the batched verdict CollisionCallBackDefault leaves in
 * data.result.isCollision() (default_broadphase_callbacks.cpp:43-60).  With flags set and capacity == 0 no pair records
 * are compacted or downloaded; the counts are still written. */
typedef struct hfb_env_out {
  uint32_t* first;
  uint32_t* second;
  hfb_contact* contacts;
  uint32_t capacity;
  uint32_t* n_colliding;
  uint32_t* n_candidates;
  uint8_t* flags;
} hfb_env_out;
int hfb_env_create(hfb_ctx* ctx, size_t n_b, const uint32_t* handles_b, const hfb_transform* tfs_b, hfb_env** out);
int hfb_env_update(hfb_ctx* ctx, hfb_env* env, size_t m, const uint32_t* indices, const hfb_transform* tfs);
int hfb_env_collide(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* handles_a, const hfb_transform* tfs_a,
                    size_t first_a, size_t num_a, const hfb_collision_request* req, const hfb_env_out* out);
int hfb_env_collide_device(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* d_handles_a,
                           const hfb_transform* d_tfs_a, size_t first_a, size_t num_a, const hfb_collision_request* req,
                           const hfb_env_out* d_out, void* cuda_stream);
int hfb_env_destroy(hfb_ctx* ctx, hfb_env* env);

/* ---- each robot object's nearest environment object: distance queries against the resident environment ----------
 * For every A object i in [first_a, first_a + num_a) (clamped to n_a, as in hfb_env_collide) and every B object j, let
 * r_ij be distance(o1 = A_i, o2 = B_j) with a fresh DistanceResult: byte for byte the record hfb_batch_distance_objects
 * writes for the pair (i, n_a + j) over the table [A; B].  A pair is ELIGIBLE when r_ij.min_distance <= max_distance
 * (a NaN distance never is: DistanceResult::update compares with '>', collision_data.h:1099-1108) and its status does
 * not carry HFB_PATH_UNSUPPORTED (e.g. a plain BVHModel<OBB>, a plane against a mesh).
 *   nearest[i]:      the eligible j with the smallest min_distance, compared as doubles (-0.0 == +0.0); the lowest j on
 *                    a tie; -1 when no pair is eligible.
 *   min_distance[i]: r_ij.min_distance of that pair; DBL_MAX (DistanceResult's initial value) when there is none.
 *   results[i]:      the full record r_ij of that pair; when there is none a fresh record: min_distance DBL_MAX, NaN
 *                    points and normal, b1 = b2 = -1, status and iterations 0.
 *   Outside the range: -1, DBL_MAX and the fresh record.
 * This is what NaiveCollisionManager::distance(obj, callback) over B (broadphase_bruteforce.cpp:99-110) computes with
 * a callback that runs distance() with a fresh result on every pair and keeps the smallest, the first in B's order on
 * ties.  It is not DistanceCallBackDefault's result: that callback lets each shape pair overwrite min_distance and stops
 * at the first pair at distance <= 0, so it depends on the manager's visiting order.
 * max_distance must be >= 0 or +inf (+inf: the nearest object at any range); NaN or a negative value is
 * HFB_ERR_INVALID_ARGUMENT.  Boxes only skip pairs whose box gap, rounded outward, exceeds max_distance or the best
 * distance found, relying on a box enclosing its shape as the collide candidates do; B objects without a box take no
 * part.  The outputs are n_a long; each may be null but not all three.  n_candidates (may be null): the pairs whose
 * distance() was run, all rounds; n_unsupported (may be null): those of them that came back HFB_PATH_UNSUPPORTED.
 * Handles, the env's validity and the range are checked as hfb_env_collide checks them, the request as
 * hfb_batch_distance checks it; a malformed argument writes nothing.
 *   hfb_env_distance: HOST buffers, blocking.
 *   hfb_env_distance_device: A's handles and poses and every output in DEVICE memory, ordered on `cuda_stream`.  The
 *     candidates are found in rounds of growing radius, and the call blocks on `cuda_stream` for each round's candidate
 *     counts: once per round, and once per round more for every further chunk of the range when n_a' * n_b >= 2^32
 *     (n_a': the range's length; chunks of floor((2^32 - 1) / n_b) A objects keep the 32-bit counts from wrapping).  A
 *     round whose candidates outgrow the context's candidate lists counts, grows them and blocks a second time to
 *     store them.  Growing a context or env buffer (the candidate lists, the round's records, the per-object state,
 *     the env's table when A has more objects than any query before) allocates device memory, which waits for the
 *     whole device.  The host form blocks at the same points and at the end. */
typedef struct hfb_env_distance_out {
  int32_t* nearest;
  double* min_distance;
  hfb_distance_result* results;
  uint32_t* n_candidates;
  uint32_t* n_unsupported;
} hfb_env_distance_out;
int hfb_env_distance(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* handles_a, const hfb_transform* tfs_a,
                     size_t first_a, size_t num_a, const hfb_distance_request* req, double max_distance,
                     const hfb_env_distance_out* out);
int hfb_env_distance_device(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* d_handles_a,
                            const hfb_transform* d_tfs_a, size_t first_a, size_t num_a, const hfb_distance_request* req,
                            double max_distance, const hfb_env_distance_out* d_out, void* cuda_stream);

/* ---- a planner's validity check: robot configurations against the resident environment AND against themselves ----
 * Set A holds n_a = n_configs * links_per_config objects, configuration-major: object g * L + i is link i of
 * configuration g (L = links_per_config >= 1, n_a % L == 0).  The self-pair template is n_self_pairs pairs of link
 * indices (i, j), 2 uint32 each (HOST memory): an SRDF's enabled pairs, the collision pairs of a Pinocchio
 * GeometryModel.  A template with an index >= L, a pair (i, i) or the same unordered pair twice is
 * HFB_ERR_INVALID_ARGUMENT, and nothing is written; an empty template is allowed.  Only configurations
 * [first_config, first_config + num_configs) are checked; a range past n_configs is HFB_ERR_INVALID_ARGUMENT.
 *   Self candidates: per configuration g and template pair (i, j), the pair (g*L + i, g*L + j) when both boxes
 *     overlap (AABB::overlap, closed intervals; objects without a box take no part) -- the set
 *     DynamicAABBTreeCollisionManager::collide(callback) over configuration g's L objects hands to a callback that keeps
 *     only the template's pairs (broadphase_collision_manager.h:104-106).  collide() runs with o1 = g*L + i and
 *     o2 = g*L + j, in the template's order; a pair whose boxes are apart is never tested, whatever security_margin says.
 *   Environment candidates: those hfb_env_collide finds for the A objects of the range.
 *   verdicts (may be null): n_configs bytes, verdicts[g] = 1 iff configuration g has a colliding environment pair or
 *     a colliding self pair (0 outside the range) -- the OR of what CollisionCallBackDefault leaves in
 *     data.result.isCollision() (default_broadphase_callbacks.cpp:43-60) after the two reference queries of g.
 *   env: the colliding environment pairs, byte for byte what hfb_env_collide returns (first: index in A, second: index
 *     in B).  self: the colliding self pairs (both indices in A), byte for byte what hfb_batch_collide_objects returns
 *     for them over the table A.  Each kind has its own capacity and counts; all pairs are counted, at most capacity
 *     of each kind stored, in no particular order.  With verdicts set and both capacities 0, no pair records are
 *     compacted or downloaded.
 * An env with no objects still checks the self pairs.  Handles, the env's validity and the request are checked as
 * hfb_env_collide checks them; security_margin == -inf gives no contacts and all verdicts 0.
 *   hfb_env_collide_configs: HOST buffers, blocking.
 *   hfb_env_collide_configs_device: A's handles and poses and every output in DEVICE memory, ordered on `cuda_stream`
 *     (the template stays in host memory); it blocks as hfb_env_collide_device does.
 *   hfb_broadphase_config_pairs: the self candidates of boxes `aabbs` (n_a x 6), HOST function, no context: configuration
 *     by configuration in template order, all counted in *n_pairs, at most `capacity` stored. */
typedef struct hfb_configs_out {
  uint8_t* verdicts;
  hfb_scene_contacts env;
  hfb_scene_contacts self;
} hfb_configs_out;
int hfb_env_collide_configs(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* handles_a, const hfb_transform* tfs_a,
                            size_t links_per_config, size_t n_self_pairs, const uint32_t* self_pairs, size_t first_config,
                            size_t num_configs, const hfb_collision_request* req, const hfb_configs_out* out);
int hfb_env_collide_configs_device(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* d_handles_a,
                                   const hfb_transform* d_tfs_a, size_t links_per_config, size_t n_self_pairs,
                                   const uint32_t* self_pairs, size_t first_config, size_t num_configs,
                                   const hfb_collision_request* req, const hfb_configs_out* d_out, void* cuda_stream);
int hfb_broadphase_config_pairs(size_t n_a, const double* aabbs, size_t links_per_config, size_t n_self_pairs,
                                const uint32_t* self_pairs, size_t first_config, size_t num_configs, uint32_t* first,
                                uint32_t* second, size_t capacity, size_t* n_pairs);

/* ---- a planner's clearance: each configuration's nearest pair, environment or self ---------------------------------
 * A, the template and the configuration range are laid out and checked as in hfb_env_collide_configs; the distance
 * rules are those of hfb_env_distance (a fresh DistanceResult per pair; ELIGIBLE: min_distance <= max_distance and not
 * HFB_PATH_UNSUPPORTED, a NaN distance never is; max_distance >= 0 or +inf, NaN or negative is
 * HFB_ERR_INVALID_ARGUMENT, checked before the context is read).  For configuration g the pairs are, in this order:
 *   1. environment pairs (g*L + i, j), j in B: link order first, then B order; each record byte for byte what
 *      hfb_env_distance returns for that pair;
 *   2. self pairs (o1 = g*L + i, o2 = g*L + j) in template order; each record byte for byte what
 *      hfb_batch_distance_objects returns for that pair over the table A.
 * The winner is the eligible pair with the smallest min_distance (-0.0 == +0.0); on a tie the first in that order, so
 * an environment pair beats a self pair at the same distance.  This is OMPL's StateValidityChecker::clearance(state),
 * which MoveIt computes as the smaller of distanceRobot and distanceSelf.  Outputs, n_configs = n_a / L each:
 *   kind[g]:          0 environment pair, 1 self pair, -1 no eligible pair (int8).
 *   first[g]:         the winner's index in A; second[g]: its index in B (kind 0) or in A (kind 1); both UINT32_MAX
 *                     without a winner.
 *   min_distance[g]:  the winner's distance, DBL_MAX without one; results[g]: its record, a fresh record without one
 *                     (as hfb_env_distance writes them).  Configurations outside the range get these no-winner values.
 *   kind, min_distance and results may each be null but not all three; first and second may be null.
 *   n_env_candidates (may be null): the count hfb_env_distance gives for the range's links; n_self_candidates (may be
 *   null): the self pairs whose distance() ran; n_unsupported (may be null): pairs of both kinds that came back
 *   HFB_PATH_UNSUPPORTED.
 * Environment pairs run as in hfb_env_distance over the range's links.  A self pair is skipped only when both link
 * boxes exist and are finite and link j's box does not overlap link i's box widened by max_distance, rounded outward
 * (relying on a box enclosing its shape, as the other calls do); at +inf every template pair runs.  An env with no
 * objects still checks the self pairs, an empty template still checks the environment.  A refused call writes nothing.
 * Counts are 32 bits: the self pairs go through the range in chunks of floor((2^32 - 1) / n_self_pairs) configurations.
 *   hfb_env_distance_configs: HOST buffers, blocking.
 *   hfb_env_distance_configs_device: A's handles and poses and every output in DEVICE memory, ordered on `cuda_stream`
 *     (the template stays in host memory).  It blocks on `cuda_stream` where hfb_env_distance_device does (the rounds'
 *     candidate counts), plus once per chunk of configurations for the self candidate count (once more when they
 *     outgrow the candidate lists).  Growing a context or env buffer allocates device memory, which waits for the
 *     whole device.  Later host calls on the context wait for it.
 *   hfb_broadphase_config_distance_pairs: the self pairs that would run, for boxes `aabbs` (n_a x 6), HOST function, no
 *     context: configuration by configuration in template order, all counted in *n_pairs, at most `capacity` stored. */
typedef struct hfb_configs_distance_out {
  int8_t* kind;
  uint32_t* first;
  uint32_t* second;
  double* min_distance;
  hfb_distance_result* results;
  uint32_t* n_env_candidates;
  uint32_t* n_self_candidates;
  uint32_t* n_unsupported;
} hfb_configs_distance_out;
int hfb_env_distance_configs(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* handles_a, const hfb_transform* tfs_a,
                             size_t links_per_config, size_t n_self_pairs, const uint32_t* self_pairs, size_t first_config,
                             size_t num_configs, const hfb_distance_request* req, double max_distance,
                             const hfb_configs_distance_out* out);
int hfb_env_distance_configs_device(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* d_handles_a,
                                    const hfb_transform* d_tfs_a, size_t links_per_config, size_t n_self_pairs,
                                    const uint32_t* self_pairs, size_t first_config, size_t num_configs,
                                    const hfb_distance_request* req, double max_distance,
                                    const hfb_configs_distance_out* d_out, void* cuda_stream);
int hfb_broadphase_config_distance_pairs(size_t n_a, const double* aabbs, size_t links_per_config, size_t n_self_pairs,
                                         const uint32_t* self_pairs, size_t first_config, size_t num_configs,
                                         double max_distance, uint32_t* first, uint32_t* second, size_t capacity,
                                         size_t* n_pairs);

/* ---- a planner's motion validation: each motion's first colliding sample and the pair that collides there ---------
 * A, the template and the configuration layout are those of hfb_env_collide_configs (object g*L + i is link i of
 * configuration g), checked the same way.  The library does not interpolate: the caller samples each motion (forward
 * kinematics is the caller's) and lays its configurations out one after another, in walking order.  There are
 * n_motions motions; motion_offsets holds n_motions + 1 uint32 values in HOST memory (in both forms, as the template):
 * motion m is configurations [offsets[m], offsets[m+1]), and sample k of motion m is configuration offsets[m] + k.
 * offsets[0] != 0, decreasing offsets, offsets[n_motions] != n_configs or a motion of more than INT32_MAX samples is
 * HFB_ERR_INVALID_ARGUMENT.  An empty motion is allowed and is valid.  Only motions [first_motion, first_motion +
 * num_motions) are checked (one GPU's share); a range past n_motions is HFB_ERR_INVALID_ARGUMENT.  The configurations
 * checked are those of the range's motions, with exactly the candidates, collide() calls (o1, o2) and records
 * hfb_env_collide_configs has over that configuration range: a sample collides iff its verdict there would be 1.
 * Within a configuration the pairs are ordered as in hfb_env_distance_configs: environment pairs by link, then by B
 * index; then self pairs in template order.  Per motion m:
 *   first_invalid[m]: the smallest k whose sample collides, -1 when none does or the motion is empty (int32).  To
 *                     validate from the end (hpp-core's `reverse`), lay the samples out end first.
 *   kind[m]:          0 environment pair, 1 self pair, -1 none (int8).
 *   first[m], second[m]: the witness, the first colliding pair in the order above of sample first_invalid[m]: its index
 *                     in A, and its index in B (kind 0) or in A (kind 1); both UINT32_MAX without a witness.
 *   contacts[m]:      the witness's record, byte for byte the one hfb_env_collide_configs returns for that pair;
 *                     without a witness the cleared CollisionResult (collision_data.h:483-489): distance_lower_bound
 *                     DBL_MAX, distance, p1, p2, normal and pos quiet NaN, b1 = b2 = -1, status, num_contacts,
 *                     iterations and _pad 0.
 *   Motions outside the range get the no-witness values.  first_invalid, kind and contacts may each be null but not
 *   all three; first and second may be null.  With kind, first, second and contacts all null no witness is sought.
 *   n_env_candidates, n_env_colliding, n_self_candidates, n_self_colliding (may be null): what hfb_env_collide_configs
 *   reports for the same configuration range.  Every sample is checked (no early exit past a motion's first colliding
 *   sample), so the counts do not depend on scheduling.  Counts are 32 bits.
 * This is OMPL's DiscreteMotionValidator::checkMotion(s1, s2, lastValid) over the caller's samples, and hpp-core's
 * discretized path validation, whose PathValidationReport carries the colliding pair and its CollisionResult.
 * An env with no objects still checks the self pairs.  Handles, the env's validity and the request are checked as
 * hfb_env_collide checks them; security_margin == -inf gives no contacts and every motion valid.  A refused call
 * writes nothing.
 *   hfb_env_collide_motions: HOST buffers, blocking.
 *   hfb_env_collide_motions_device: A's handles and poses and every output in DEVICE memory, ordered on `cuda_stream`
 *     (the template and the offsets stay in host memory).  It blocks where hfb_env_collide_configs_device does: on
 *     `cuda_stream` for the candidate count (twice when the candidates outgrow the context's candidate lists, which
 *     then grow), and growing a context or env buffer (the candidate lists, the records, the per-motion state, the
 *     env's table when A has more objects than any query before) allocates device memory, which waits for the whole
 *     device.  Later host calls on the context wait for it. */
typedef struct hfb_motions_out {
  int32_t* first_invalid;
  int8_t* kind;
  uint32_t* first;
  uint32_t* second;
  hfb_contact* contacts;
  uint32_t* n_env_candidates;
  uint32_t* n_env_colliding;
  uint32_t* n_self_candidates;
  uint32_t* n_self_colliding;
} hfb_motions_out;
int hfb_env_collide_motions(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* handles_a, const hfb_transform* tfs_a,
                            size_t links_per_config, size_t n_self_pairs, const uint32_t* self_pairs, size_t n_motions,
                            const uint32_t* motion_offsets, size_t first_motion, size_t num_motions,
                            const hfb_collision_request* req, const hfb_motions_out* out);
int hfb_env_collide_motions_device(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* d_handles_a,
                                   const hfb_transform* d_tfs_a, size_t links_per_config, size_t n_self_pairs,
                                   const uint32_t* self_pairs, size_t n_motions, const uint32_t* motion_offsets,
                                   size_t first_motion, size_t num_motions, const hfb_collision_request* req,
                                   const hfb_motions_out* d_out, void* cuda_stream);

/* ---- a planner's continuous motion validation: each segment between two samples certified free -------------------
 * A, the template, the offsets, the motion range and the request are those of hfb_env_collide_motions, checked the
 * same way; the template and the offsets stay in HOST memory in both forms.  sweep holds n_a doubles (host memory in
 * the host form, device memory in the device form): sweep[g*L + i] is the caller's bound on the path length of every
 * point of link i from configuration g to configuration g+1, samples k and k+1 of one motion (hpp-core's
 * maximalVelocity times the step; the library does not interpolate).  The entry at a motion's last sample is never
 * read.  A value that is not finite and >= 0 (NaN, negative, +-inf) is not an error: it widens nothing, and every
 * segment it bounds is uncertified.
 * Sides.  At sample g a pair has a right threshold (segment g -> g+1) and a left one (g-1 -> g): an environment pair
 * (link i, B object j) has s_R = sweep[g*L+i] and s_L = sweep[(g-1)*L+i] (the environment does not move); a self pair
 * (i, j) has s_R = sweep[g*L+i] + sweep[g*L+j] rounded up, and s_L the same at g-1.  A side exists when g has a
 * successor (right) or predecessor (left) in its motion and its sweep values are valid.  A pair passes a side when the
 * side exists, its collide() record has num_contacts == 0, its status is not HFB_PATH_UNSUPPORTED (whose cleared record
 * carries distance_lower_bound = DBL_MAX) and 2 * distance_lower_bound > s (strict; NaN never passes).  A sample passes
 * a side when every candidate pair of it does.
 * Candidates.  w, the reach of a link or pair, is half the larger of its valid side thresholds, rounded up (0 with
 * none).  Environment candidates: link i's box widened by w, rounded outward, overlaps B's box (the grid query runs on
 * the widened boxes).  Self candidates: both links have a box, and unless both boxes are finite and link j's box does
 * not overlap link i's box widened by w, rounded outward (hfb_broadphase_sweep_pairs).  A pair that is not a candidate
 * passes both sides: its box gap, and so its distance, exceeds w.  At w = 0 the candidates include those of
 * hfb_env_collide_configs.  Objects without a box take no part.  Every candidate runs collide() with the caller's
 * request; its record is byte for byte what hfb_batch_collide_objects gives for that pair over the table [A; B].
 * Outputs, per motion m and configuration g:
 *   first_invalid[m]:     exactly what hfb_env_collide_motions returns: a sample collides iff one of its pairs whose
 *                         unwidened boxes overlap has contacts.  A contact of a pair found by the widening alone (e.g.
 *                         under a positive security_margin) does not invalidate the sample; it fails certification.
 *   certified[g]:         1 iff g and g+1 are samples k and k+1 of one motion of the range, g's right side passes and
 *                         g+1's left side passes; else 0 (a motion's last sample, configurations outside the range).
 *                         n_configs bytes.
 *   first_uncertified[m]: the smallest k with certified[offsets[m]+k] == 0 among the motion's n-1 segments, or -1
 *                         (empty and one-sample motions, motions outside the range).
 *   n_env_candidates, n_self_candidates: the widened candidates of the range; n_unsupported: the candidates that came
 *   back HFB_PATH_UNSUPPORTED; n_uncertified: the range's segments with certified = 0.  32-bit counts, may be null.
 *   first_invalid, first_uncertified and certified may each be null, but not all three.
 * security_margin == -inf: no collide() runs, every motion is valid and every segment with valid sweeps certified.
 * The guarantee.  If every point of each link travels at most its sweep along segment k and every
 * distance_lower_bound used is a true lower bound, no pair of the segment touches anywhere inside it: after a fraction
 * tau of the joint motion a pair's distance has dropped by at most (s_a + s_b) * tau from sample k, and by at most the
 * rest from sample k+1, so passing both half-tests covers tau in [0, 1/2] from the left end and [1/2, 1] from the
 * right.  For shape-shape leaves the reference subtracts security_margin from the lower bound: under a positive margin
 * the pair also stays outside the margin; under a negative one the lower bound exceeds the true distance by |margin|,
 * so the guarantee weakens to "no pair penetrates deeper than |margin|" (BVH pairs are unsupported there).  For GJK
 * pairs the reference's lower bound is the converged distance, good to
 * gjk_tolerance only: a caller who wants strict slack adds 2 * gjk_tolerance to each sweep.
 * Refinement of the segments with certified = 0 is hfb_env_validate_motions' (hpp-core's progressive validation), or
 * the caller's: resample them and call again.  Handles, the env's validity and the request are checked as hfb_env_collide checks them.  A refused
 * call (a null sweep or output, all three per-item outputs null, or a refusal of hfb_env_collide_motions) writes
 * nothing.
 *   hfb_env_certify_motions: HOST buffers, blocking.
 *   hfb_env_certify_motions_device: A's handles and poses, sweep and every output in DEVICE memory, ordered on
 *     `cuda_stream`; it blocks where hfb_env_collide_motions_device does.  Later host calls on the context wait for it.
 * hfb_broadphase_sweep_pairs: the self candidates above on the host (no context), for the configurations of the
 * motion range, from the boxes `aabbs` (n_a x 6, as hfb_scene_aabbs writes them) and the sweep bounds; configuration
 * by configuration in template order, all counted in *n_pairs, at most `capacity` stored.  Arguments are checked as
 * hfb_env_certify_motions checks them. */
typedef struct hfb_certify_out {
  int32_t* first_invalid;     /* n_motions */
  int32_t* first_uncertified; /* n_motions */
  uint8_t* certified;         /* n_configs */
  uint32_t* n_env_candidates;
  uint32_t* n_self_candidates;
  uint32_t* n_unsupported;
  uint32_t* n_uncertified;
} hfb_certify_out;
int hfb_env_certify_motions(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* handles_a, const hfb_transform* tfs_a,
                            const double* sweep, size_t links_per_config, size_t n_self_pairs, const uint32_t* self_pairs,
                            size_t n_motions, const uint32_t* motion_offsets, size_t first_motion, size_t num_motions,
                            const hfb_collision_request* req, const hfb_certify_out* out);
int hfb_env_certify_motions_device(hfb_ctx* ctx, hfb_env* env, size_t n_a, const uint32_t* d_handles_a,
                                   const hfb_transform* d_tfs_a, const double* d_sweep, size_t links_per_config,
                                   size_t n_self_pairs, const uint32_t* self_pairs, size_t n_motions,
                                   const uint32_t* motion_offsets, size_t first_motion, size_t num_motions,
                                   const hfb_collision_request* req, const hfb_certify_out* d_out, void* cuda_stream);
int hfb_broadphase_sweep_pairs(size_t n_a, const double* aabbs, const double* sweep, size_t links_per_config,
                               size_t n_self_pairs, const uint32_t* self_pairs, size_t n_motions,
                               const uint32_t* motion_offsets, size_t first_motion, size_t num_motions, uint32_t* first,
                               uint32_t* second, size_t capacity, size_t* n_pairs);

/* ---- a robot model on the device: forward kinematics, motion sampling and sweep bounds ---------------------------
 * What Pinocchio's forwardKinematics(model, data, q) followed by updateGeometryPlacements(model, data, geom_model,
 * geom_data) computes for a kinematic tree of 1-DoF joints, batched over configurations, with the results laid out as
 * the hfb_env_* calls above take set A: object g*L + i is link i of configuration g, so a planner chains these calls
 * with the env queries on one stream and uploads joint values instead of poses.
 * The model (hfb_robot_desc, validated on the host; a malformed one is HFB_ERR_INVALID_ARGUMENT and nothing is
 * created):
 *   num_joints J, 1..64, with nq = J: configuration g is q[g*J .. g*J + J).  Per joint j: parent[j] -1 (the world) or
 *   < j, so the joints come in topological order; type[j] HFB_JOINT_REVOLUTE or HFB_JOINT_PRISMATIC; axis[3j..3j+3),
 *   normalised at create (a zero or non-finite axis is refused); placement[j], the joint frame in its parent's frame at
 *   q = 0.  num_links L >= 1, with L * J <= UINT32_MAX.  Per link i: link_joint[i], -1 for fixed to the world or a joint index;
 *   link_placement[i]; link_handles[i], a committed geometry handle.  Null arrays are refused.
 * Semantics:
 *   joint frame   M_j = M_parent(j) o placement_j o X_j(q_j), M_parent = identity for a joint on the world; X_j is the
 *                 rotation by q_j about the unit axis (Rodrigues) for a revolute joint, the translation by q_j * axis
 *                 for a prismatic one;
 *   link pose     M_link_joint(i) o link_placement_i; link_placement_i for a link fixed to the world.
 *   sin and cos come from the library's own fdlibm restatement (csrc/hfb_kin.cuh), below 1 ulp for |q| <= 2^20 * pi/2
 *   (about 1.647e6 rad) and NaN beyond, so the device and a host build of the same code give the same bits.  A
 *   non-finite q is not an error: it propagates to NaN poses, which the narrow phase's rules for non-finite input handle.
 * The geometry: after a later hfb_geom_commit the handles are checked again (in range, not released) and the local
 * boxes the sweep bounds use are read again; after hfb_geom_clear every call on the robot is refused until it is
 * destroyed -- the rules of hfb_env.  hfb_ctx_destroy frees the robots a context still owns.
 * Counts: n_configs * L <= UINT32_MAX, as the env calls' n_a.
 *   hfb_robot_poses: n_configs x J joint values -> tfs (n_configs * L link poses) and, when handles is not null, the
 *     link handles tiled n_configs times.
 *   hfb_robot_sample_motions: motion m goes from q_from[m*J ..] to q_to[m*J ..]; motion_offsets (n_motions + 1 uint32,
 *     HOST memory in both forms) are checked as hfb_env_collide_motions checks them, n_configs = offsets[n_motions].
 *     Sample k of an n-sample motion, configuration offsets[m] + k, is q_from at k = 0, exactly q_to at k = n - 1 and
 *     q_from + (k / (n - 1)) * (q_to - q_from) in between: OMPL's RealVectorStateSpace::interpolate, linear in q.  A
 *     one-sample motion is q_from; an empty motion is allowed.  Outputs (hfb_robot_samples_out): tfs and handles as
 *     hfb_robot_poses writes them; q (may be null): the samples' joint values, n_configs x J; sweep (may be null): the
 *     bounds hfb_env_certify_motions takes.
 * Sweep bounds.  sweep[g*L + i] bounds the path length of every point of link i over the segment from sample g to g+1:
 *     s = sum over the joints k on the path from the root to link i of |q_{g+1,k} - q_{g,k}| * rho_k, with rho_k = 1 for
 *     a prismatic k and, for a revolute k, rho_k = the sum over the joints j strictly below k on that path of
 *     |translation(placement_j)|, plus max(|q_{g,j}|, |q_{g+1,j}|) for the prismatic ones among them, plus
 *     |translation(link_placement_i)| + r_i, where r_i is the largest corner norm of the geometry's committed local box
 *     (+inf for an unbounded geometry; a joint that does not move adds 0).  The argument: a point moves at the speed
 *     sum_k |dq_k/dt| * (its distance to k's axis) for revolute k, plus |dq_k/dt| for prismatic k.  k's axis passes
 *     through the origin of M_k, and the point's distance to that origin is at most rho_k by the triangle inequality
 *     down the path (a revolute joint does not move its own origin, a prismatic j moves it by |q_j|).  q is linear over
 *     the segment, so |q_j| is largest at an end point and the integral of |dq_k/dt| is |q_{g+1,k} - q_{g,k}|.  s is
 *     computed in round-to-nearest, then multiplied by 1 + J * 2^-46, far above the sum's rounding error, and rounded to
 *     the next double, so the host and the device give the same bits.  The entry at a motion's last sample is 0, as
 *     are those of links fixed to the world and of segments where no joint of the path moves.
 * Refusals: a null context, robot or array, malformed offsets, or a count past the 32-bit rule is
 * HFB_ERR_INVALID_ARGUMENT, and nothing is written.
 *   hfb_robot_poses / hfb_robot_sample_motions: HOST buffers, blocking.
 *   *_device: q (q_from, q_to) and every output in DEVICE memory, ordered on `cuda_stream`; the call does not block
 *     (the offsets are read on the host).  It orders itself after the context's previous *_device call as those do.
 * One kernel serves both: one thread per (configuration, link), walking the link's path from the root; every frame is
 * evaluated by the one formula above, so no result depends on scheduling. */
#define HFB_JOINT_REVOLUTE 0u
#define HFB_JOINT_PRISMATIC 1u
typedef struct hfb_robot_desc {
  uint32_t num_joints;
  const int32_t* parent;
  const uint32_t* type;
  const double* axis;
  const hfb_transform* placement;
  uint32_t num_links;
  const int32_t* link_joint;
  const hfb_transform* link_placement;
  const uint32_t* link_handles;
} hfb_robot_desc;
typedef struct hfb_robot hfb_robot;
typedef struct hfb_robot_samples_out {
  hfb_transform* tfs; /* n_configs * L */
  uint32_t* handles;  /* n_configs * L */
  double* q;          /* n_configs * J, may be null */
  double* sweep;      /* n_configs * L, may be null */
} hfb_robot_samples_out;
int hfb_robot_create(hfb_ctx* ctx, const hfb_robot_desc* desc, hfb_robot** out);
int hfb_robot_destroy(hfb_ctx* ctx, hfb_robot* robot);
int hfb_robot_poses(hfb_ctx* ctx, hfb_robot* robot, size_t n_configs, const double* q, hfb_transform* tfs,
                    uint32_t* handles);
int hfb_robot_poses_device(hfb_ctx* ctx, hfb_robot* robot, size_t n_configs, const double* d_q, hfb_transform* d_tfs,
                           uint32_t* d_handles, void* cuda_stream);
int hfb_robot_sample_motions(hfb_ctx* ctx, hfb_robot* robot, size_t n_motions, const double* q_from, const double* q_to,
                             const uint32_t* motion_offsets, const hfb_robot_samples_out* out);
int hfb_robot_sample_motions_device(hfb_ctx* ctx, hfb_robot* robot, size_t n_motions, const double* d_q_from,
                                    const double* d_q_to, const uint32_t* motion_offsets,
                                    const hfb_robot_samples_out* d_out, void* cuda_stream);

/* ---- a planner's progressive motion validation: each motion proven free, found colliding or left at its resolution --
 * hfb_env_certify_motions over samples that hfb_robot_sample_motions would make, with the segments that fail
 * certification split and checked again inside the call: hpp-core's continuous path validation
 * (continuousValidation::Dichotomy / Progressive).  Motion m of n_motions runs from q_from[m*J ..] to q_to[m*J ..] (J the
 * robot's joints), linear in q; the links are the robot's L links and the self-pair template is over link indices.
 * Positions.  With D = max_depth, a sample sits at an integer position k in [0, 2^D], t = k * 2^-D; its joint values are
 * q_from at k = 0, q_to at k = 2^D and q_from + t * (q_to - q_from) otherwise (hfb_robot_sample_motions' formula: t is an
 * exact dyadic, so the samples of depth d are bit for bit those of 2^d + 1 samples).  A segment [a, b] of depth d has
 * b - a = 2^(D-d); its sweep bounds are hfb_robot_sample_motions' bounds over q(a) -> q(b).
 * Round 0 opens the 2^d0 segments of depth d0 = initial_depth of each motion of the range [first_motion, first_motion
 * + num_motions).  A round:
 *   1. Runs: each motion's open segments form runs, maximal chains of contiguous open segments; a run of s segments has
 *      s + 1 samples.  Segments are admitted in (motion, position) order while the round's sample count stays <= the
 *      cap: min(max_samples, 2^29, floor((2^32 - 1 - n_b) / L)), the last keeping samples * L + n_b below 2^32 as the
 *      env calls' object counts are.
 *   2. Certify: the runs go through one hfb_env_certify_motions as its motions, with the robot's poses at the samples
 *      and the sweep bounds of the segments, the caller's request and template.
 *   3. Collisions: c_m <- min(c_m, the first colliding sample of each of m's runs).
 *   4. Segments: each open segment by the first rule that applies: certified -> closed; starts at or after c_m ->
 *      dropped; not admitted, of depth D, or a link's sweep bound not finite (halving cannot make it finite) -> stuck;
 *      otherwise split into two open halves.
 *   5. Frontier: with f_m the start of m's earliest stuck segment, every open segment of m from f_m on is dropped.
 * The call ends when no segment is open, after at most D - d0 + 1 rounds.  Per motion m of the range:
 *   t_valid[m]:   the end of the prefix of certified segments (1 when every segment is certified).
 *   t_collide[m]: c_m * 2^-D, -1 when no colliding sample was found.
 *   status[m]:    1 (collides) when a colliding sample was found, else 0 (valid) when t_valid = 1, else 2 (unresolved).
 *   kind, first, second, contacts: the witness at t_collide, what hfb_env_collide_motions returns for the one-sample
 *                 motion q(t_collide) (first, second: link indices, or a B index for kind 0); the no-witness values
 *                 without a colliding sample.  With all four null no witness is sought.
 *   Motions outside the range: status -1, t_valid 0, t_collide -1 and the no-witness values.
 *   n_rounds: the rounds that certified something; n_samples, n_env_candidates, n_self_candidates, n_unsupported: sums
 *   over the rounds of their samples and of hfb_env_certify_motions' counts (64 bits wide).  Each count may be null.
 * No output depends on scheduling.  For a colliding motion the first contact lies in (t_valid, t_collide].
 * The guarantee: a valid motion is certified whole, and [0, t_valid] is free when t_valid > 0, under hfb_env_certify_motions' guarantee
 * with its sweep bounds (including its weaker form under a negative security_margin and the gjk_tolerance caveat);
 * security_margin == -inf behaves as there (no collide() runs, every segment with finite sweeps certified).
 * Refusals, HFB_ERR_INVALID_ARGUMENT with nothing written: initial_depth > max_depth, max_depth > 30, max_samples < 2;
 * a null context, env, robot, request, params, output struct, status, t_valid or t_collide; a null self_pairs with
 * n_self_pairs > 0; null q_from / q_to with a non-empty range; a range past n_motions; then, under the context's lock,
 * the request as hfb_env_collide checks it, the robot's refusals (hfb_robot_poses'), the env's, and the template's
 * (hfb_env_collide_configs' with L the robot's link count).
 *   hfb_env_validate_motions: HOST buffers, blocking.
 *   hfb_env_validate_motions_device: q_from, q_to and every output in DEVICE memory (the template stays in host memory),
 *     ordered on `cuda_stream`.  It blocks on `cuda_stream` once per round (the round's sample count sizes its
 *     launches), where hfb_env_certify_motions_device blocks, and once more for the number of colliding motions;
 *     growing a context or env buffer allocates device memory, which waits for the whole device. */
typedef struct hfb_validate_params {
  uint32_t initial_depth; /* d0: round 0 checks 2^d0 equal segments per motion */
  uint32_t max_depth;     /* D, d0 <= D <= 30: no segment is shorter than 2^-D of its motion */
  uint64_t max_samples;   /* per round, >= 2 */
} hfb_validate_params;
typedef struct hfb_validate_out {
  int8_t* status;   /* n_motions: 0 valid, 1 collides, 2 unresolved; -1 outside the range */
  double* t_valid;  /* n_motions: end of the certified prefix, in [0, 1] */
  double* t_collide; /* n_motions: earliest colliding sample found, -1 if none */
  int8_t* kind;     /* n_motions each: the witness at t_collide (may be null) */
  uint32_t* first;
  uint32_t* second;
  hfb_contact* contacts;
  uint32_t* n_rounds;
  uint64_t* n_samples;
  uint64_t* n_env_candidates;
  uint64_t* n_self_candidates;
  uint64_t* n_unsupported;
} hfb_validate_out;
int hfb_env_validate_motions(hfb_ctx* ctx, hfb_env* env, hfb_robot* robot, size_t n_motions, const double* q_from,
                             const double* q_to, size_t n_self_pairs, const uint32_t* self_pairs, size_t first_motion,
                             size_t num_motions, const hfb_collision_request* req, const hfb_validate_params* p,
                             const hfb_validate_out* out);
int hfb_env_validate_motions_device(hfb_ctx* ctx, hfb_env* env, hfb_robot* robot, size_t n_motions,
                                    const double* d_q_from, const double* d_q_to, size_t n_self_pairs,
                                    const uint32_t* self_pairs, size_t first_motion, size_t num_motions,
                                    const hfb_collision_request* req, const hfb_validate_params* p,
                                    const hfb_validate_out* d_out, void* cuda_stream);

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
