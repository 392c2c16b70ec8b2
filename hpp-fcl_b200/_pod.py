"""POD layouts of include/hppfcl_b200.h as numpy structured dtypes + ctypes structs.

These are the flat forms of the reference's Transform3f (math/transform.h:56-216),
ShapeBase subclasses (shape/geometric_shapes.h:164-634), QueryRequest /
DistanceRequest / CollisionRequest (collision_data.h:171-274, 987-1050, 312-383),
DistanceResult (:1053-1096) and CollisionResult+Contact (:59-166, 391-509).
"""
import ctypes as C

import numpy as np

# NODE_TYPE values (collision_object.h:65-89)
BV_OBB = 2
BV_OBBRSS = 5
GEOM_BOX = 9
GEOM_SPHERE = 10
GEOM_CAPSULE = 11
GEOM_CONE = 12
GEOM_CYLINDER = 13
GEOM_CONVEX = 14
GEOM_PLANE = 15
GEOM_HALFSPACE = 16
GEOM_TRIANGLE = 17
GEOM_ELLIPSOID = 19

# data_types.h:85-98
DefaultGuess, CachedGuess, BoundingVolumeGuess = 0, 1, 2
DefaultGJK, PolyakAcceleration, NesterovAcceleration = 0, 1, 2
Default, DualityGap, Hybrid = 0, 1, 2
Relative, Absolute = 0, 1

# GJK::Status / EPA::Status (narrowphase/gjk.h:95-102, 330-341)
GJK_DidNotRun, GJK_Failed, GJK_NoCollisionEarlyStopped, GJK_NoCollision, \
    GJK_CollisionWithPenetrationInformation, GJK_Collision = range(6)
EPA_DidNotRun = 0xFF
EPA_Failed, EPA_Valid, EPA_AccuracyReached, EPA_Degenerated, EPA_NonConvex, \
    EPA_InvalidHull, EPA_OutOfFaces, EPA_OutOfVertices, EPA_FallBack = 0, 1, 3, 2, 4, 6, 8, 10, 12

PATH_GJK, PATH_CLOSED_FORM, PATH_BVH, PATH_UNSUPPORTED = 0, 1, 2, 0xEE

DBL_MAX = np.finfo(np.float64).max

transform_dtype = np.dtype([("R", "<f8", (9,)), ("T", "<f8", (3,))], align=True)
shape_dtype = np.dtype([("type", "<u4"), ("data", "<u4"), ("p", "<f8", (3,)), ("ssr", "<f8")], align=True)
distance_result_dtype = np.dtype(
    [("min_distance", "<f8"), ("p1", "<f8", (3,)), ("p2", "<f8", (3,)), ("normal", "<f8", (3,)),
     ("b1", "<i4"), ("b2", "<i4"), ("status", "<u4"), ("iterations", "<u4")], align=True)
contact_dtype = np.dtype(
    [("distance", "<f8"), ("p1", "<f8", (3,)), ("p2", "<f8", (3,)), ("normal", "<f8", (3,)),
     ("pos", "<f8", (3,)), ("distance_lower_bound", "<f8"), ("b1", "<i4"), ("b2", "<i4"),
     ("status", "<u4"), ("num_contacts", "<u4"), ("iterations", "<u4"), ("_pad", "<u4")], align=True)
bvh_node_dtype = np.dtype(
    [("first_child", "<i4"), ("first_primitive", "<u4"), ("num_primitives", "<u4"), ("_pad", "<u4"),
     ("obb_axes", "<f8", (9,)), ("obb_To", "<f8", (3,)), ("obb_extent", "<f8", (3,)),
     ("rss_axes", "<f8", (9,)), ("rss_Tr", "<f8", (3,)), ("rss_length", "<f8", (2,)),
     ("rss_radius", "<f8")], align=True)

assert transform_dtype.itemsize == 96
assert shape_dtype.itemsize == 40
assert distance_result_dtype.itemsize == 96
assert contact_dtype.itemsize == 136
assert bvh_node_dtype.itemsize == 256


class QueryRequest(C.Structure):
    _fields_ = [
        ("gjk_initial_guess", C.c_int32),
        ("gjk_variant", C.c_int32),
        ("gjk_convergence_criterion", C.c_int32),
        ("gjk_convergence_criterion_type", C.c_int32),
        ("gjk_max_iterations", C.c_uint32),
        ("epa_max_iterations", C.c_uint32),
        ("gjk_tolerance", C.c_double),
        ("epa_tolerance", C.c_double),
        ("collision_distance_threshold", C.c_double),
        ("cached_gjk_guess", C.c_void_p),
        ("cached_support_func_guess", C.c_void_p),
    ]


def _default_query(q):
    # collision_data.h:205-249 + narrowphase_defaults.h:47-62
    q.gjk_initial_guess = DefaultGuess
    q.gjk_variant = DefaultGJK
    q.gjk_convergence_criterion = Default
    q.gjk_convergence_criterion_type = Relative
    q.gjk_max_iterations = 128
    q.epa_max_iterations = 64
    q.gjk_tolerance = 1e-6
    q.epa_tolerance = 1e-6
    q.collision_distance_threshold = 1e-12
    q.cached_gjk_guess = None
    q.cached_support_func_guess = None


class DistanceRequestPOD(C.Structure):
    _fields_ = [("q", QueryRequest), ("enable_signed_distance", C.c_int32), ("enable_nearest_points", C.c_int32),
                ("rel_err", C.c_double), ("abs_err", C.c_double)]

    def __init__(self, **kw):
        super().__init__()
        _default_query(self.q)
        self.enable_signed_distance = 1
        self.enable_nearest_points = 1
        self.rel_err = 0.0
        self.abs_err = 0.0
        _apply_kw(self, kw)


class CollisionRequestPOD(C.Structure):
    _fields_ = [("q", QueryRequest), ("num_max_contacts", C.c_uint32), ("enable_contact", C.c_int32),
                ("security_margin", C.c_double), ("break_distance", C.c_double),
                ("distance_upper_bound", C.c_double)]

    def __init__(self, **kw):
        super().__init__()
        _default_query(self.q)
        self.num_max_contacts = 1
        self.enable_contact = 1
        self.security_margin = 0.0
        self.break_distance = 1e-3
        self.distance_upper_bound = DBL_MAX
        _apply_kw(self, kw)


def _apply_kw(req, kw):
    qnames = {f[0] for f in QueryRequest._fields_}
    for k, v in kw.items():
        if k in qnames:
            setattr(req.q, k, v)
        elif hasattr(req, k):
            setattr(req, k, v)
        else:
            raise TypeError("unknown request field %r" % k)


class GuessOut(C.Structure):
    _fields_ = [("cached_gjk_guess", C.c_void_p), ("cached_support_func_guess", C.c_void_p)]


class ObjectPairs(C.Structure):
    """hfb_object_pairs: an object table (handle + pose) and index pairs into it"""
    _fields_ = [("n_objects", C.c_size_t), ("object_handles", C.c_void_p), ("object_tfs", C.c_void_p),
                ("n_pairs", C.c_size_t), ("first", C.c_void_p), ("second", C.c_void_p)]


class CompactContacts(C.Structure):
    _fields_ = [("flags", C.c_void_p), ("n_colliding", C.c_void_p), ("pair_ids", C.c_void_p),
                ("contacts", C.c_void_p), ("capacity", C.c_uint32)]


class SceneContacts(C.Structure):
    _fields_ = [("first", C.c_void_p), ("second", C.c_void_p), ("contacts", C.c_void_p), ("capacity", C.c_uint32),
                ("n_colliding", C.c_void_p), ("n_candidates", C.c_void_p)]


class EnvOut(C.Structure):  # hfb_env_out: hfb_scene_contacts + one flag byte per A object
    _fields_ = SceneContacts._fields_ + [("flags", C.c_void_p)]


class ConfigsOut(C.Structure):  # hfb_configs_out: one verdict byte per configuration, the two kinds of pairs
    _fields_ = [("verdicts", C.c_void_p), ("env", SceneContacts), ("self", SceneContacts)]


class EnvDistanceOut(C.Structure):  # hfb_env_distance_out: per A object the nearest B object, its distance and record
    _fields_ = [("nearest", C.c_void_p), ("min_distance", C.c_void_p), ("results", C.c_void_p),
                ("n_candidates", C.c_void_p), ("n_unsupported", C.c_void_p)]


class ConfigsDistanceOut(C.Structure):  # hfb_configs_distance_out: per configuration its nearest pair, environment or self
    _fields_ = [("kind", C.c_void_p), ("first", C.c_void_p), ("second", C.c_void_p), ("min_distance", C.c_void_p),
                ("results", C.c_void_p), ("n_env_candidates", C.c_void_p), ("n_self_candidates", C.c_void_p),
                ("n_unsupported", C.c_void_p)]


class MotionsOut(C.Structure):  # hfb_motions_out: per motion its first colliding sample and the first pair colliding there
    _fields_ = [("first_invalid", C.c_void_p), ("kind", C.c_void_p), ("first", C.c_void_p), ("second", C.c_void_p),
                ("contacts", C.c_void_p), ("n_env_candidates", C.c_void_p), ("n_env_colliding", C.c_void_p),
                ("n_self_candidates", C.c_void_p), ("n_self_colliding", C.c_void_p)]


class CertifyOut(C.Structure):  # hfb_certify_out: per motion its first colliding and first uncertified sample, per
    # configuration whether the segment to the next sample is certified free
    _fields_ = [("first_invalid", C.c_void_p), ("first_uncertified", C.c_void_p), ("certified", C.c_void_p),
                ("n_env_candidates", C.c_void_p), ("n_self_candidates", C.c_void_p), ("n_unsupported", C.c_void_p),
                ("n_uncertified", C.c_void_p)]


JOINT_REVOLUTE, JOINT_PRISMATIC = 0, 1  # HFB_JOINT_*


class RobotDesc(C.Structure):  # hfb_robot_desc: a kinematic tree of 1-DoF joints and the links on it
    _fields_ = [("num_joints", C.c_uint32), ("parent", C.c_void_p), ("type", C.c_void_p), ("axis", C.c_void_p),
                ("placement", C.c_void_p), ("num_links", C.c_uint32), ("link_joint", C.c_void_p),
                ("link_placement", C.c_void_p), ("link_handles", C.c_void_p)]


class RobotSamplesOut(C.Structure):  # hfb_robot_samples_out: the samples' poses and handles, joint values, sweep bounds
    _fields_ = [("tfs", C.c_void_p), ("handles", C.c_void_p), ("q", C.c_void_p), ("sweep", C.c_void_p)]


class ValidateParams(C.Structure):  # hfb_validate_params: the initial and the largest depth, the samples per round
    _fields_ = [("initial_depth", C.c_uint32), ("max_depth", C.c_uint32), ("max_samples", C.c_uint64)]


class ValidateOut(C.Structure):  # hfb_validate_out: per motion its status, certified prefix, first collision and witness
    _fields_ = [("status", C.c_void_p), ("t_valid", C.c_void_p), ("t_collide", C.c_void_p), ("kind", C.c_void_p),
                ("first", C.c_void_p), ("second", C.c_void_p), ("contacts", C.c_void_p), ("n_rounds", C.c_void_p),
                ("n_samples", C.c_void_p), ("n_env_candidates", C.c_void_p), ("n_self_candidates", C.c_void_p),
                ("n_unsupported", C.c_void_p)]


class Stats(C.Structure):
    _fields_ = [("kernel_launches", C.c_uint64), ("pairs_processed", C.c_uint64),
                ("epa_pairs", C.c_uint64), ("bv_tests", C.c_uint64), ("leaf_tests", C.c_uint64),
                ("watchdog_trips", C.c_uint64)]


class KernelTimes(C.Structure):
    _fields_ = [("pairs_ms", C.c_double), ("epa_ms", C.c_double), ("other_ms", C.c_double),
                ("pairs_launches", C.c_uint64), ("epa_launches", C.c_uint64), ("other_launches", C.c_uint64),
                ("closed_ms", C.c_double), ("convex_ms", C.c_double),
                ("closed_launches", C.c_uint64), ("convex_launches", C.c_uint64),
                ("bvh_ms", C.c_double), ("bvh_launches", C.c_uint64)]


def status_gjk(s):
    return np.asarray(s) & 0xFF


def status_epa(s):
    return (np.asarray(s) >> 8) & 0xFF


def status_path(s):
    return (np.asarray(s) >> 16) & 0xFF


def make_transforms(R, T):
    """R: (n,3,3) rotation matrices (row-major numpy), T: (n,3) -> transform_dtype array.
    The POD stores R column-major like Eigen (transform.h:57)."""
    R = np.asarray(R, dtype=np.float64).reshape(-1, 3, 3)
    T = np.asarray(T, dtype=np.float64).reshape(-1, 3)
    out = np.zeros(R.shape[0], dtype=transform_dtype)
    out["R"] = np.transpose(R, (0, 2, 1)).reshape(-1, 9)
    out["T"] = T
    return out


def make_shapes(types, params, ssr=None, data=None):
    types = np.asarray(types, dtype=np.uint32).reshape(-1)
    out = np.zeros(types.shape[0], dtype=shape_dtype)
    out["type"] = types
    out["p"] = np.asarray(params, dtype=np.float64).reshape(-1, 3)
    if ssr is not None:
        out["ssr"] = ssr
    if data is not None:
        out["data"] = data
    return out
