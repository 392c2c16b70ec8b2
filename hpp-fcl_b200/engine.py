"""ctypes binding of the C-ABI (include/hppfcl_b200.h) -- the drop-in boundary.

`Engine` owns one hfb_ctx (one CUDA device).  Everything that computes goes
through libhppfcl_b200.so; there is no Python or CPU fallback: a missing library
or a missing GPU raises EngineError.
"""
import ctypes as C
import os

import numpy as np

from . import _pod as P
from .build import library_path

_LIB = None


class EngineError(RuntimeError):
    pass


_ERR = {1: "invalid argument", 2: "no CUDA device", 3: "CUDA error", 4: "unsupported pair",
        5: "out of memory"}


def load_library(path=None):
    """dlopen the in-tree extension. Works without a GPU (symbols only)."""
    global _LIB
    if _LIB is not None and path is None:
        return _LIB
    path = path or library_path()
    if not os.path.exists(path):
        raise EngineError("CUDA extension %s is not built (run __graft_entry__.build())" % path)
    L = C.CDLL(path)
    vp, sz, u32 = C.c_void_p, C.c_size_t, C.c_uint32
    L.hfb_ctx_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.hfb_ctx_destroy.argtypes = [vp]
    L.hfb_last_error.argtypes = [vp]
    L.hfb_last_error.restype = C.c_char_p
    L.hfb_version.restype = C.c_char_p
    L.hfb_default_distance_request.argtypes = [vp]
    L.hfb_default_collision_request.argtypes = [vp]
    L.hfb_geom_register_shapes.argtypes = [vp, vp, sz, vp]
    L.hfb_geom_register_halfspaces.argtypes = [vp, C.c_uint32, vp, vp, sz, vp]
    L.hfb_geom_register_convex.argtypes = [vp, vp, u32, vp]
    L.hfb_geom_register_convex_batch.argtypes = [vp, vp, u32, u32, vp]
    L.hfb_geom_register_bvh_obbrss.argtypes = [vp, vp, u32, vp, u32, vp, u32, vp]
    L.hfb_bvh_build_obbrss.argtypes = [vp, u32, vp, u32, vp, u32]
    L.hfb_geom_commit.argtypes = [vp]
    L.hfb_geom_device_arena.argtypes = [vp, C.POINTER(vp), C.POINTER(sz)]
    L.hfb_geom_num_shapes.argtypes = [vp]
    L.hfb_geom_num_shapes.restype = sz
    L.hfb_geom_clear.argtypes = [vp]
    L.hfb_geom_update_shapes.argtypes = [vp, vp, vp, C.c_size_t]
    L.hfb_geom_update_convex.argtypes = [vp, C.c_uint32, vp, C.c_uint32]
    L.hfb_geom_release_shapes.argtypes = [vp, vp, C.c_size_t]
    for name in ("hfb_batch_distance", "hfb_batch_collide"):
        getattr(L, name).argtypes = [vp, sz, vp, vp, vp, vp, vp, vp, vp]
        getattr(L, name + "_device").argtypes = [vp, sz, vp, vp, vp, vp, vp, vp, vp, vp]
    L.hfb_batch_collide_contacts.argtypes = [vp, sz, vp, vp, vp, vp, vp, vp, u32, vp, vp, vp]
    L.hfb_scene_aabbs.argtypes = [vp, sz, vp, vp, vp]
    L.hfb_broadphase_pairs.argtypes = [sz, vp, vp, vp, sz, vp]
    L.hfb_scene_aabbs_device.argtypes = [vp, sz, vp, vp, vp, vp]
    L.hfb_broadphase_pairs_device.argtypes = [vp, sz, vp, sz, sz, vp, vp, sz, vp, vp]
    L.hfb_scene_collide.argtypes = [vp, sz, vp, vp, sz, sz, vp, vp]
    L.hfb_broadphase_cross_pairs.argtypes = [sz, vp, sz, vp, vp, vp, sz, vp]
    L.hfb_broadphase_cross_pairs_device.argtypes = [vp, sz, vp, sz, sz, sz, vp, vp, vp, sz, vp, vp]
    L.hfb_scene_collide_sets.argtypes = [vp, sz, vp, vp, sz, vp, vp, sz, sz, vp, vp]
    L.hfb_env_create.argtypes = [vp, sz, vp, vp, C.POINTER(vp)]
    L.hfb_env_update.argtypes = [vp, vp, sz, vp, vp]
    L.hfb_env_collide.argtypes = [vp, vp, sz, vp, vp, sz, sz, vp, vp]
    L.hfb_env_collide_device.argtypes = [vp, vp, sz, vp, vp, sz, sz, vp, vp, vp]
    L.hfb_env_destroy.argtypes = [vp, vp]
    L.hfb_env_collide_configs.argtypes = [vp, vp, sz, vp, vp, sz, sz, vp, sz, sz, vp, vp]
    L.hfb_env_collide_configs_device.argtypes = [vp, vp, sz, vp, vp, sz, sz, vp, sz, sz, vp, vp, vp]
    L.hfb_env_distance.argtypes = [vp, vp, sz, vp, vp, sz, sz, vp, C.c_double, vp]
    L.hfb_env_distance_device.argtypes = [vp, vp, sz, vp, vp, sz, sz, vp, C.c_double, vp, vp]
    L.hfb_broadphase_config_pairs.argtypes = [sz, vp, sz, sz, vp, sz, sz, vp, vp, sz, vp]
    L.hfb_env_distance_configs.argtypes = [vp, vp, sz, vp, vp, sz, sz, vp, sz, sz, vp, C.c_double, vp]
    L.hfb_env_distance_configs_device.argtypes = [vp, vp, sz, vp, vp, sz, sz, vp, sz, sz, vp, C.c_double, vp, vp]
    L.hfb_env_collide_motions.argtypes = [vp, vp, sz, vp, vp, sz, sz, vp, sz, vp, sz, sz, vp, vp]
    L.hfb_env_collide_motions_device.argtypes = [vp, vp, sz, vp, vp, sz, sz, vp, sz, vp, sz, sz, vp, vp, vp]
    L.hfb_broadphase_config_distance_pairs.argtypes = [sz, vp, sz, sz, vp, sz, sz, C.c_double, vp, vp, sz, vp]
    L.hfb_env_certify_motions.argtypes = [vp, vp, sz, vp, vp, vp, sz, sz, vp, sz, vp, sz, sz, vp, vp]
    L.hfb_env_certify_motions_device.argtypes = [vp, vp, sz, vp, vp, vp, sz, sz, vp, sz, vp, sz, sz, vp, vp, vp]
    L.hfb_broadphase_sweep_pairs.argtypes = [sz, vp, vp, sz, sz, vp, sz, vp, sz, sz, vp, vp, sz, vp]
    L.hfb_robot_create.argtypes = [vp, vp, C.POINTER(vp)]
    L.hfb_robot_destroy.argtypes = [vp, vp]
    L.hfb_robot_poses.argtypes = [vp, vp, sz, vp, vp, vp]
    L.hfb_robot_poses_device.argtypes = [vp, vp, sz, vp, vp, vp, vp]
    L.hfb_robot_sample_motions.argtypes = [vp, vp, sz, vp, vp, vp, vp]
    L.hfb_robot_sample_motions_device.argtypes = [vp, vp, sz, vp, vp, vp, vp, vp]
    L.hfb_env_validate_motions.argtypes = [vp, vp, vp, sz, vp, vp, sz, vp, sz, sz, vp, vp, vp]
    L.hfb_env_validate_motions_device.argtypes = [vp, vp, vp, sz, vp, vp, sz, vp, sz, sz, vp, vp, vp, vp]
    L.hfb_comm_unique_id.argtypes = [vp]
    L.hfb_comm_init.argtypes = [vp, vp, C.c_int, C.c_int]
    L.hfb_comm_destroy.argtypes = [vp]
    L.hfb_geom_broadcast.argtypes = [vp, C.c_int]
    L.hfb_comm_wait.argtypes = [vp, vp]
    for name in ("hfb_batch_distance_sharded_device", "hfb_batch_collide_sharded_device"):
        getattr(L, name).argtypes = [vp, sz, vp, vp, vp, vp, vp, vp, vp]
    L.hfb_batch_distance_objects.argtypes = [vp, vp, vp, vp, vp, vp]
    L.hfb_batch_collide_objects.argtypes = [vp, vp, vp, vp, vp, vp]
    L.hfb_batch_distance_objects_device.argtypes = [vp, vp, vp, vp, vp, vp]
    L.hfb_batch_collide_objects_device.argtypes = [vp, vp, vp, vp, vp, vp]
    L.hfb_batch_convex_support.argtypes = [vp, sz, vp, vp, vp, vp]
    L.hfb_batch_convex_support_device.argtypes = [vp, sz, vp, vp, vp, vp, vp]
    L.hfb_get_stats.argtypes = [vp, vp]
    L.hfb_set_profiling.argtypes = [vp, C.c_int]
    L.hfb_get_kernel_times.argtypes = [vp, vp, C.c_int]
    if path == library_path():
        _LIB = L
    return L


def build_bvh_obbrss(vertices, triangles):
    """Host-side OBBRSS tree of a triangle mesh (BVHModel<OBBRSS>::endModel, mean split): the node array
    hfb_geom_register_bvh_obbrss takes.  Needs no GPU."""
    L = load_library()
    v = np.ascontiguousarray(vertices, dtype=np.float64).reshape(-1, 3)
    t = np.ascontiguousarray(triangles, dtype=np.uint32).reshape(-1, 3)
    nodes = np.zeros(max(2 * t.shape[0] - 1, 0), dtype=P.bvh_node_dtype)
    rc = L.hfb_bvh_build_obbrss(_ptr(v), v.shape[0], _ptr(t), t.shape[0], _ptr(nodes), nodes.shape[0])
    if rc != 0:
        raise EngineError("hfb_bvh_build_obbrss: %s" % _ERR.get(rc, rc))
    return nodes


def broadphase_pairs(aabbs, capacity=None):
    """every pair i < j of overlapping boxes (n x 6: min xyz, max xyz), in no particular order -> (first, second).
    Host function of the library: needs neither a context nor a GPU."""
    L = load_library()
    bb = np.ascontiguousarray(aabbs, dtype=np.float64).reshape(-1, 6)
    n = bb.shape[0]
    cap = int(capacity) if capacity is not None else max(16 * n, 1024)
    while True:
        first = np.empty(cap, dtype=np.uint32)
        second = np.empty(cap, dtype=np.uint32)
        cnt = C.c_size_t(0)
        rc = L.hfb_broadphase_pairs(n, _ptr(bb), _ptr(first), _ptr(second), cap, C.byref(cnt))
        if rc != 0:
            raise EngineError("hfb_broadphase_pairs: %s" % _ERR.get(rc, rc))
        if cnt.value <= cap or capacity is not None:
            k = min(cnt.value, cap)
            return first[:k], second[:k]
        cap = cnt.value


def broadphase_cross_pairs(aabbs_a, aabbs_b, capacity=None):
    """every (i, j), i a box of A, j a box of B (n x 6 each), whose boxes overlap, in no particular order -> (first =
    index in A, second = index in B).  Host function of the library: needs neither a context nor a GPU."""
    L = load_library()
    ba = np.ascontiguousarray(aabbs_a, dtype=np.float64).reshape(-1, 6)
    bb = np.ascontiguousarray(aabbs_b, dtype=np.float64).reshape(-1, 6)
    cap = int(capacity) if capacity is not None else max(16 * (ba.shape[0] + bb.shape[0]), 1024)
    while True:
        first = np.empty(cap, dtype=np.uint32)
        second = np.empty(cap, dtype=np.uint32)
        cnt = C.c_size_t(0)
        rc = L.hfb_broadphase_cross_pairs(ba.shape[0], _ptr(ba), bb.shape[0], _ptr(bb), _ptr(first), _ptr(second), cap,
                                          C.byref(cnt))
        if rc != 0:
            raise EngineError("hfb_broadphase_cross_pairs: %s" % _ERR.get(rc, rc))
        if cnt.value <= cap or capacity is not None:
            k = min(cnt.value, cap)
            return first[:k], second[:k]
        cap = cnt.value


def _template(self_pairs):
    """a self-pair template as the C ABI takes it: (P, 2) uint32, contiguous"""
    return np.ascontiguousarray(np.asarray(self_pairs, dtype=np.uint32).reshape(-1, 2))


def broadphase_config_pairs(aabbs, links_per_config, self_pairs, first_config=0, num_configs=None, capacity=None):
    """the self candidates of configurations: boxes (n x 6) of n_configs x links_per_config objects, configuration-major;
    for every configuration g of [first_config, first_config + num_configs) (default: to the end) and template pair
    (i, j) whose boxes overlap, (g * L + i, g * L + j) -> (first, second), configuration by configuration in template
    order.  Host function of the library: needs neither a context nor a GPU."""
    L = load_library()
    bb = np.ascontiguousarray(aabbs, dtype=np.float64).reshape(-1, 6)
    tpl = _template(self_pairs)
    n, lpc = bb.shape[0], int(links_per_config)
    if num_configs is None:
        num_configs = max(n // lpc - first_config, 0) if lpc else 0
    cap = int(capacity) if capacity is not None else max(tpl.shape[0] * int(num_configs), 1)
    first = np.empty(max(cap, 1), dtype=np.uint32)
    second = np.empty(max(cap, 1), dtype=np.uint32)
    cnt = C.c_size_t(0)
    rc = L.hfb_broadphase_config_pairs(n, _ptr(bb), lpc, tpl.shape[0], _ptr(tpl), int(first_config), int(num_configs),
                                       _ptr(first), _ptr(second), cap, C.byref(cnt))
    if rc != 0:
        raise EngineError("hfb_broadphase_config_pairs: %s" % _ERR.get(rc, rc))
    k = min(cnt.value, cap)
    return first[:k], second[:k]


def broadphase_config_distance_pairs(aabbs, links_per_config, self_pairs, max_distance=np.inf, first_config=0,
                                     num_configs=None, capacity=None):
    """the self pairs whose distance() the configurations distance query runs: boxes (n x 6) of n_configs x
    links_per_config objects, configuration-major; for every configuration g of [first_config, first_config +
    num_configs) (default: to the end) and template pair (i, j), (g * L + i, g * L + j) unless both boxes exist and are
    finite and j's box does not overlap i's box widened by max_distance (rounded outward) -> (first, second),
    configuration by configuration in template order.  Host function of the library: needs neither a context nor a GPU."""
    L = load_library()
    bb = np.ascontiguousarray(aabbs, dtype=np.float64).reshape(-1, 6)
    tpl = _template(self_pairs)
    n, lpc = bb.shape[0], int(links_per_config)
    if num_configs is None:
        num_configs = max(n // lpc - first_config, 0) if lpc else 0
    cap = int(capacity) if capacity is not None else max(tpl.shape[0] * int(num_configs), 1)
    first = np.empty(max(cap, 1), dtype=np.uint32)
    second = np.empty(max(cap, 1), dtype=np.uint32)
    cnt = C.c_size_t(0)
    rc = L.hfb_broadphase_config_distance_pairs(n, _ptr(bb), lpc, tpl.shape[0], _ptr(tpl), int(first_config),
                                                int(num_configs), float(max_distance), _ptr(first), _ptr(second), cap,
                                                C.byref(cnt))
    if rc != 0:
        raise EngineError("hfb_broadphase_config_distance_pairs: %s" % _ERR.get(rc, rc))
    k = min(cnt.value, cap)
    return first[:k], second[:k]


def broadphase_sweep_pairs(aabbs, sweep, links_per_config, self_pairs, offsets, first_motion=0, num_motions=None,
                           capacity=None):
    """the self pairs whose collide() the motion certification runs: boxes (n x 6) and sweep bounds (n) of n_configs x
    links_per_config objects, configuration-major, motion m being configurations [offsets[m], offsets[m+1]); for every
    configuration g of the motion range and template pair (i, j), (g * L + i, g * L + j) when both boxes exist and,
    unless both are finite, j's box overlaps i's box widened by the pair's reach: half the larger of its right and left
    thresholds (the sums of its links' sweeps, rounded up), rounded up (hfb_broadphase_sweep_pairs) -> (first, second),
    configuration by configuration in template order.  Host function of the library: needs neither a context nor a
    GPU."""
    L = load_library()
    bb = np.ascontiguousarray(aabbs, dtype=np.float64).reshape(-1, 6)
    sw = np.ascontiguousarray(sweep, dtype=np.float64).reshape(-1)
    tpl = _template(self_pairs)
    off = _offsets(offsets)
    n, lpc, n_motions = bb.shape[0], int(links_per_config), off.shape[0] - 1
    if sw.shape[0] != n:
        raise ValueError("sweep: one bound per object")
    if num_motions is None:
        num_motions = n_motions - first_motion
    cap = int(capacity) if capacity is not None else max(tpl.shape[0] * (n // lpc if lpc else 0), 1)
    first = np.empty(max(cap, 1), dtype=np.uint32)
    second = np.empty(max(cap, 1), dtype=np.uint32)
    cnt = C.c_size_t(0)
    rc = L.hfb_broadphase_sweep_pairs(n, _ptr(bb), _ptr(sw), lpc, tpl.shape[0], _ptr(tpl), n_motions, _ptr(off),
                                      int(first_motion), int(num_motions), _ptr(first), _ptr(second), cap, C.byref(cnt))
    if rc != 0:
        raise EngineError("hfb_broadphase_sweep_pairs: %s" % _ERR.get(rc, rc))
    k = min(cnt.value, cap)
    return first[:k], second[:k]


def _offsets(offsets):
    """motion offsets as the C ABI takes them: n_motions + 1 uint32, contiguous"""
    off = np.asarray(offsets).reshape(-1)
    if off.shape[0] == 0:
        raise ValueError("motion offsets: n_motions + 1 values, at least one")
    if off.dtype.kind not in "ui" or (off.dtype.kind == "i" and (off < 0).any()) or (off > 0xFFFFFFFF).any():
        raise ValueError("motion offsets: integers in [0, 2^32)")
    return np.ascontiguousarray(off, dtype=np.uint32)


def robot_desc(parent, types, axis, placement, link_joint, link_placement, link_handles):
    """an hfb_robot_desc over contiguous copies of the arrays -> (desc, the arrays it points into: keep them alive)"""
    par = np.ascontiguousarray(parent, dtype=np.int32).reshape(-1)
    typ = np.ascontiguousarray(types, dtype=np.uint32).reshape(-1)
    ax = np.ascontiguousarray(axis, dtype=np.float64).reshape(-1, 3)
    pl = np.ascontiguousarray(placement, dtype=P.transform_dtype).reshape(-1)
    lj = np.ascontiguousarray(link_joint, dtype=np.int32).reshape(-1)
    lp = np.ascontiguousarray(link_placement, dtype=P.transform_dtype).reshape(-1)
    lh = np.ascontiguousarray(link_handles, dtype=np.uint32).reshape(-1)
    J, L = par.shape[0], lj.shape[0]
    if typ.shape[0] != J or ax.shape[0] != J or pl.shape[0] != J:
        raise ValueError("robot model: one type, axis and placement per joint")
    if lp.shape[0] != L or lh.shape[0] != L:
        raise ValueError("robot model: one placement and geometry handle per link")
    keep = (par, typ, ax, pl, lj, lp, lh)
    desc = P.RobotDesc(J, *[a.ctypes.data for a in keep[:4]], L, *[a.ctypes.data for a in keep[4:]])
    return desc, keep


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    return a.ctypes.data_as(C.c_void_p)


class Engine:
    """One device context + geometry arena (ctx_create / geom_register_* / batch_*)."""

    def __init__(self, device=0):
        self.L = load_library()
        h = C.c_void_p()
        rc = self.L.hfb_ctx_create(int(device), C.byref(h))
        if rc != 0:
            raise EngineError("hfb_ctx_create(device=%d) failed: %s (no CPU fallback exists)"
                              % (device, _ERR.get(rc, rc)))
        self.h = h
        self.device = device

    # -- lifetime ---------------------------------------------------------
    def close(self):
        if getattr(self, "h", None):
            self.L.hfb_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            msg = self.L.hfb_last_error(self.h)
            raise EngineError("%s: %s" % (_ERR.get(rc, rc), msg.decode() if msg else ""))

    # -- geometry ---------------------------------------------------------
    def register_convex(self, points):
        pts = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        cid = C.c_uint32()
        self._check(self.L.hfb_geom_register_convex(self.h, _ptr(pts), pts.shape[0], C.byref(cid)))
        return cid.value

    def register_shapes(self, shapes):
        shapes = np.ascontiguousarray(shapes, dtype=P.shape_dtype)
        handles = np.zeros(shapes.shape[0], dtype=np.uint32)
        self._check(self.L.hfb_geom_register_shapes(self.h, _ptr(shapes), shapes.shape[0], _ptr(handles)))
        return handles

    def register_halfspaces(self, kind, n_d, ssr=None):
        """Halfspace (kind = GEOM_HALFSPACE) or Plane (GEOM_PLANE) geometries: n_d is (count, 4) rows
        (n.x, n.y, n.z, d), normalised by the library; ssr: count swept-sphere radii or None.  Returns the handles."""
        nd = np.ascontiguousarray(n_d, dtype=np.float64).reshape(-1, 4)
        r = None if ssr is None else np.ascontiguousarray(ssr, dtype=np.float64).reshape(-1)
        if r is not None and r.shape[0] != nd.shape[0]:
            raise ValueError("one swept-sphere radius per plane")
        handles = np.zeros(nd.shape[0], dtype=np.uint32)
        self._check(self.L.hfb_geom_register_halfspaces(self.h, int(kind), _ptr(nd), None if r is None else _ptr(r),
                                                        nd.shape[0], _ptr(handles)))
        return handles

    def register_convex_batch(self, points):
        """points: (count, nv, 3); returns the id of the first hull, the others follow"""
        pts = np.ascontiguousarray(points, dtype=np.float64)
        assert pts.ndim == 3 and pts.shape[2] == 3
        first = C.c_uint32()
        self._check(self.L.hfb_geom_register_convex_batch(self.h, _ptr(pts), pts.shape[1], pts.shape[0], C.byref(first)))
        return first.value

    def register_bvh_obbrss(self, nodes, vertices, triangles):
        """nodes: BVHModel<OBBRSS>::bvs as hfb_bvh_node records (the reference's own tree, or
        build_bvh_obbrss(vertices, triangles)); None builds it here."""
        if nodes is None:
            nodes = build_bvh_obbrss(vertices, triangles)
        nodes = np.ascontiguousarray(nodes, dtype=P.bvh_node_dtype)
        v = np.ascontiguousarray(vertices, dtype=np.float64).reshape(-1, 3)
        t = np.ascontiguousarray(triangles, dtype=np.uint32).reshape(-1, 3)
        bid = C.c_uint32()
        self._check(self.L.hfb_geom_register_bvh_obbrss(self.h, _ptr(nodes), nodes.shape[0], _ptr(v),
                                                        v.shape[0], _ptr(t), t.shape[0], C.byref(bid)))
        return bid.value  # use as `data` of a shape record of type BV_OBBRSS

    def register_bvh_obb(self, nodes, vertices, triangles):
        """a plain BVHModel<OBB> (collide() only): the same node records, RSS half ignored -- the OBB tree of a mesh is the
        OBB half of its OBBRSS tree, so build_bvh_obbrss serves both; use as `data` of a shape record of type BV_OBB"""
        if nodes is None:
            nodes = build_bvh_obbrss(vertices, triangles)
        nodes = np.ascontiguousarray(nodes, dtype=P.bvh_node_dtype)
        v = np.ascontiguousarray(vertices, dtype=np.float64).reshape(-1, 3)
        t = np.ascontiguousarray(triangles, dtype=np.uint32).reshape(-1, 3)
        bid = C.c_uint32()
        self._check(self.L.hfb_geom_register_bvh_obb(self.h, _ptr(nodes), nodes.shape[0], _ptr(v), v.shape[0], _ptr(t),
                                                     t.shape[0], C.byref(bid)))
        return bid.value

    def commit(self):
        self._check(self.L.hfb_geom_commit(self.h))

    def clear_geometry(self):
        """drops every registered shape / hull / mesh; all handles become invalid"""
        self._check(self.L.hfb_geom_clear(self.h))

    def update_shapes(self, handles, shapes):
        """replace the records of registered handles (e.g. new sizes); commit() before the next query"""
        handles = np.ascontiguousarray(handles, dtype=np.uint32)
        shapes = np.ascontiguousarray(shapes, dtype=P.shape_dtype)
        assert handles.shape[0] == shapes.shape[0]
        self._check(self.L.hfb_geom_update_shapes(self.h, _ptr(handles), _ptr(shapes), handles.shape[0]))

    def update_convex(self, convex_id, points):
        """replace the vertices of a registered hull by as many new ones"""
        pts = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        self._check(self.L.hfb_geom_update_convex(self.h, int(convex_id), _ptr(pts), pts.shape[0]))

    def release_shapes(self, handles):
        """retire handles: pairs that still name them come back as unsupported"""
        handles = np.ascontiguousarray(handles, dtype=np.uint32)
        self._check(self.L.hfb_geom_release_shapes(self.h, _ptr(handles), handles.shape[0]))

    def device_arena(self):
        base = C.c_void_p()
        n = C.c_size_t()
        self._check(self.L.hfb_geom_device_arena(self.h, C.byref(base), C.byref(n)))
        return base.value, n.value

    # -- host-buffer queries (H2D + kernels + D2H inside the call) ----------
    def _host_call(self, fn, out_dtype, h1, tf1, h2, tf2, req, want_guess, out=None):
        h1 = np.ascontiguousarray(h1, dtype=np.uint32)
        h2 = np.ascontiguousarray(h2, dtype=np.uint32)
        tf1 = np.ascontiguousarray(tf1, dtype=P.transform_dtype)
        tf2 = np.ascontiguousarray(tf2, dtype=P.transform_dtype)
        n = h1.shape[0]
        if not (h2.shape[0] == n and tf1.shape[0] == n and tf2.shape[0] == n):
            raise ValueError("batch arrays must have equal length")
        if out is None:
            out = np.empty(n, dtype=out_dtype)
        g = None
        gg = gh = None
        if want_guess:
            gg = np.zeros((n, 3), dtype=np.float64)
            gh = np.zeros((n, 2), dtype=np.int32)
            g = P.GuessOut(_ptr(gg), _ptr(gh))
        self._check(fn(self.h, n, _ptr(h1), _ptr(tf1), _ptr(h2), _ptr(tf2), C.byref(req), _ptr(out),
                       C.byref(g) if g is not None else None))
        if want_guess:
            return out, gg, gh
        return out

    def batch_distance(self, h1, tf1, h2, tf2, req=None, want_guess=False, out=None):
        req = req or P.DistanceRequestPOD()
        return self._host_call(self.L.hfb_batch_distance, P.distance_result_dtype, h1, tf1, h2, tf2,
                               req, want_guess, out)

    def batch_collide(self, h1, tf1, h2, tf2, req=None, want_guess=False, out=None):
        req = req or P.CollisionRequestPOD()
        return self._host_call(self.L.hfb_batch_collide, P.contact_dtype, h1, tf1, h2, tf2, req,
                               want_guess, out)

    def batch_collide_contacts(self, h1, tf1, h2, tf2, req=None, max_extra=3):
        """collide() keeping up to 1 + max_extra contacts of a mesh pair: -> (out, extra[n, max_extra], counts);
        contacts[k] of pair i, 1 <= k < min(counts[i], max_extra + 1), is extra[i, k - 1]"""
        req = req or P.CollisionRequestPOD()
        h1 = np.ascontiguousarray(h1, dtype=np.uint32)
        h2 = np.ascontiguousarray(h2, dtype=np.uint32)
        tf1 = np.ascontiguousarray(tf1, dtype=P.transform_dtype)
        tf2 = np.ascontiguousarray(tf2, dtype=P.transform_dtype)
        n = h1.shape[0]
        out = np.zeros(n, dtype=P.contact_dtype)
        extra = np.zeros((n, max(max_extra, 1)), dtype=P.contact_dtype)
        counts = np.zeros(n, dtype=np.uint32)
        self._check(self.L.hfb_batch_collide_contacts(self.h, n, _ptr(h1), _ptr(tf1), _ptr(h2), _ptr(tf2), C.byref(req),
                                                      _ptr(out), max_extra, _ptr(extra), _ptr(counts), None))
        return out, extra[:, :max_extra], counts

    # -- broadphase feed ---------------------------------------------------------------------------------
    def scene_aabbs(self, obj_handles, obj_tfs):
        """CollisionObject::computeAABB of every object -> n x 6 (min xyz, max xyz); host function"""
        oh = np.ascontiguousarray(obj_handles, dtype=np.uint32)
        ot = np.ascontiguousarray(obj_tfs, dtype=P.transform_dtype)
        bb = np.empty((oh.shape[0], 6), dtype=np.float64)
        self._check(self.L.hfb_scene_aabbs(self.h, oh.shape[0], _ptr(oh), _ptr(ot), _ptr(bb)))
        return bb

    def scene_aabbs_device(self, n, d_handles, d_tfs, d_aabbs, stream=0):
        self._check(self.L.hfb_scene_aabbs_device(self.h, n, _ptr(d_handles), _ptr(d_tfs), _ptr(d_aabbs), _ptr(stream)))

    def broadphase_pairs_device(self, n, d_aabbs, d_first, d_second, capacity, d_n_pairs, stream=0, first_object=0,
                                num_first_objects=None):
        """pairs (i, j), i < j, with i in [first_object, first_object + num_first_objects) (default: all)"""
        self._check(self.L.hfb_broadphase_pairs_device(self.h, n, _ptr(d_aabbs), first_object,
                                                       n if num_first_objects is None else num_first_objects, _ptr(d_first),
                                                       _ptr(d_second), capacity, _ptr(d_n_pairs), _ptr(stream)))

    def scene_collide(self, obj_handles, obj_tfs, req=None, capacity=None, first_object=0, num_first_objects=None, bufs=None):
        """broadphase + narrow phase of a scene in one call (hfb_scene_collide)
        -> (first, second, contacts, n_candidates, n_colliding): the colliding pairs, in no particular order"""
        req = req or P.CollisionRequestPOD()
        oh = np.ascontiguousarray(obj_handles, dtype=np.uint32)
        ot = np.ascontiguousarray(obj_tfs, dtype=P.transform_dtype)
        n = oh.shape[0]
        cap = int(capacity) if capacity is not None else max(4 * n, 1024)
        if bufs is None:
            bufs = (np.empty(cap, dtype=np.uint32), np.empty(cap, dtype=np.uint32), np.empty(cap, dtype=P.contact_dtype))
        f, s2, rec = bufs
        nc = np.zeros(2, dtype=np.uint32)
        out = P.SceneContacts(f.ctypes.data, s2.ctypes.data, rec.ctypes.data, cap, nc[0:1].ctypes.data, nc[1:2].ctypes.data)
        self._check(self.L.hfb_scene_collide(self.h, n, _ptr(oh), _ptr(ot), first_object,
                                             n if num_first_objects is None else num_first_objects, C.byref(req), C.byref(out)))
        k = min(int(nc[0]), cap)
        return f[:k], s2[:k], rec[:k], int(nc[1]), int(nc[0])

    def broadphase_cross_pairs_device(self, n_a, d_aabbs_a, n_b, d_aabbs_b, d_first, d_second, capacity, d_n_pairs,
                                      stream=0, first_a=0, num_a=None):
        """pairs (i in A, j in B) with overlapping boxes, i in [first_a, first_a + num_a) (default: all of A)"""
        self._check(self.L.hfb_broadphase_cross_pairs_device(self.h, n_a, _ptr(d_aabbs_a), first_a,
                                                             n_a if num_a is None else num_a, n_b, _ptr(d_aabbs_b),
                                                             _ptr(d_first), _ptr(d_second), capacity, _ptr(d_n_pairs),
                                                             _ptr(stream)))

    def scene_collide_sets(self, handles_a, tfs_a, handles_b, tfs_b, req=None, capacity=None, first_a=0, num_a=None,
                           bufs=None):
        """broadphase + narrow phase of set A against set B in one call (hfb_scene_collide_sets)
        -> (first = index in A, second = index in B, contacts, n_candidates, n_colliding), in no particular order"""
        req = req or P.CollisionRequestPOD()
        ha, ta = self._objects(handles_a, tfs_a)
        hb, tb = self._objects(handles_b, tfs_b)
        na, nb = ha.shape[0], hb.shape[0]
        cap = int(capacity) if capacity is not None else max(4 * (na + nb), 1024)
        if bufs is None:
            bufs = (np.empty(cap, dtype=np.uint32), np.empty(cap, dtype=np.uint32), np.empty(cap, dtype=P.contact_dtype))
        f, s2, rec = bufs
        nc = np.zeros(2, dtype=np.uint32)
        out = P.SceneContacts(f.ctypes.data, s2.ctypes.data, rec.ctypes.data, cap, nc[0:1].ctypes.data, nc[1:2].ctypes.data)
        self._check(self.L.hfb_scene_collide_sets(self.h, na, _ptr(ha), _ptr(ta), nb, _ptr(hb), _ptr(tb), first_a,
                                                  na if num_a is None else num_a, C.byref(req), C.byref(out)))
        k = min(int(nc[0]), cap)
        return f[:k], s2[:k], rec[:k], int(nc[1]), int(nc[0])

    # -- resident environment (hfb_env_*): set B's table, boxes and grid kept on the device across queries -------
    def env_create(self, handles_b, tfs_b):
        """set B on the device (its boxes as of now and the cross grid over them) -> an opaque env handle"""
        hb, tb = self._objects(handles_b, tfs_b)
        env = C.c_void_p()
        self._check(self.L.hfb_env_create(self.h, hb.shape[0], _ptr(hb), _ptr(tb), C.byref(env)))
        return env

    def env_update(self, env, indices, tfs):
        """new poses of the B objects `indices` (the reference's update(objs)); their boxes and the grid are redone"""
        idx = np.ascontiguousarray(indices, dtype=np.uint32)
        t = np.ascontiguousarray(tfs, dtype=P.transform_dtype)
        if idx.shape[0] != t.shape[0]:
            raise ValueError("index and pose arrays must have equal length")
        self._check(self.L.hfb_env_update(self.h, env, idx.shape[0], _ptr(idx), _ptr(t)))

    def env_collide(self, env, handles_a, tfs_a, req=None, capacity=None, first_a=0, num_a=None, flags=False, bufs=None):
        """set A against the env (hfb_env_collide): what scene_collide_sets(A, B) returns -> (first = index in A, second =
        index in B, contacts, n_candidates, n_colliding), plus one flag byte per A object (1: it collides) with
        flags=True.  capacity=0 with flags=True: no pair records at all"""
        req = req or P.CollisionRequestPOD()
        ha, ta = self._objects(handles_a, tfs_a)
        na = ha.shape[0]
        cap = int(capacity) if capacity is not None else max(4 * na, 1024)
        if bufs is None:
            bufs = (np.empty(cap, dtype=np.uint32), np.empty(cap, dtype=np.uint32), np.empty(cap, dtype=P.contact_dtype))
        f, s2, rec = bufs
        fl = np.empty(na, dtype=np.uint8) if flags else None
        nc = np.zeros(2, dtype=np.uint32)
        out = P.EnvOut(f.ctypes.data, s2.ctypes.data, rec.ctypes.data, cap, nc[0:1].ctypes.data, nc[1:2].ctypes.data,
                       None if fl is None else fl.ctypes.data)
        self._check(self.L.hfb_env_collide(self.h, env, na, _ptr(ha), _ptr(ta), first_a, na if num_a is None else num_a,
                                           C.byref(req), C.byref(out)))
        k = min(int(nc[0]), cap)
        res = (f[:k], s2[:k], rec[:k], int(nc[1]), int(nc[0]))
        return res + (fl,) if flags else res

    def env_collide_device(self, env, n_a, d_handles_a, d_tfs_a, d_first, d_second, d_contacts, capacity, d_n_colliding,
                           d_n_candidates, d_flags=None, req=None, stream=0, first_a=0, num_a=None):
        """hfb_env_collide_device: A's handles and poses and every output are device pointers, ordered on `stream`"""
        req = req or P.CollisionRequestPOD()
        out = P.EnvOut(d_first, d_second, d_contacts, capacity, d_n_colliding, d_n_candidates, d_flags)
        self._check(self.L.hfb_env_collide_device(self.h, env, n_a, _ptr(d_handles_a), _ptr(d_tfs_a), first_a,
                                                  n_a if num_a is None else num_a, C.byref(req), C.byref(out), _ptr(stream)))

    def env_destroy(self, env):
        self._check(self.L.hfb_env_destroy(self.h, env))

    def env_collide_configs(self, env, handles_a, tfs_a, links_per_config, self_pairs, req=None, env_capacity=None,
                            self_capacity=None, first_config=0, num_configs=None, verdicts=True):
        """configurations of links_per_config objects each (A, configuration-major) against the env and against
        themselves (the template's link pairs), hfb_env_collide_configs -> (verdicts: one byte per configuration, 1 iff
        it collides, or None with verdicts=False; env = (first = index in A, second = index in B, contacts, n_candidates,
        n_colliding); self = (first, second: indices in A, contacts, n_candidates, n_colliding)).  Both capacities 0 with
        verdicts=True: no pair records at all"""
        req = req or P.CollisionRequestPOD()
        ha, ta = self._objects(handles_a, tfs_a)
        tpl = _template(self_pairs)
        na, lpc = ha.shape[0], int(links_per_config)
        n_configs = na // lpc if lpc else 0
        caps = [int(c) if c is not None else max(4 * na, 1024) for c in (env_capacity, self_capacity)]
        bufs = [(np.empty(c, dtype=np.uint32), np.empty(c, dtype=np.uint32), np.empty(c, dtype=P.contact_dtype)) for c in caps]
        nc = np.zeros(4, dtype=np.uint32)  # env colliding, env candidates, self colliding, self candidates
        v = np.empty(n_configs, dtype=np.uint8) if verdicts else None
        kinds = [P.SceneContacts(f.ctypes.data, s2.ctypes.data, rec.ctypes.data, c, nc[2 * k:].ctypes.data,
                                 nc[2 * k + 1:].ctypes.data) for k, ((f, s2, rec), c) in enumerate(zip(bufs, caps))]
        out = P.ConfigsOut(None if v is None else v.ctypes.data, kinds[0], kinds[1])
        self._check(self.L.hfb_env_collide_configs(self.h, env, na, _ptr(ha), _ptr(ta), lpc, tpl.shape[0], _ptr(tpl),
                                                   first_config, n_configs - first_config if num_configs is None else num_configs,
                                                   C.byref(req), C.byref(out)))
        res = []
        for k, ((f, s2, rec), c) in enumerate(zip(bufs, caps)):
            m = min(int(nc[2 * k]), c)
            res.append((f[:m], s2[:m], rec[:m], int(nc[2 * k + 1]), int(nc[2 * k])))
        return v, res[0], res[1]

    def env_collide_configs_device(self, env, n_a, d_handles_a, d_tfs_a, links_per_config, self_pairs, d_verdicts, env_out,
                                   self_out, req=None, stream=0, first_config=0, num_configs=None):
        """hfb_env_collide_configs_device: A's handles and poses and every output are device pointers, ordered on
        `stream`; env_out / self_out = (d_first, d_second, d_contacts, capacity, d_n_colliding, d_n_candidates); the
        template is a host array"""
        req = req or P.CollisionRequestPOD()
        tpl = _template(self_pairs)
        lpc = int(links_per_config)
        n_configs = n_a // lpc if lpc else 0
        out = P.ConfigsOut(d_verdicts, P.SceneContacts(*env_out), P.SceneContacts(*self_out))
        self._check(self.L.hfb_env_collide_configs_device(self.h, env, n_a, _ptr(d_handles_a), _ptr(d_tfs_a), lpc,
                                                          tpl.shape[0], _ptr(tpl), first_config,
                                                          n_configs - first_config if num_configs is None else num_configs,
                                                          C.byref(req), C.byref(out), _ptr(stream)))

    def env_distance(self, env, handles_a, tfs_a, req=None, max_distance=np.inf, first_a=0, num_a=None, records=True):
        """each A object's nearest B object (hfb_env_distance) -> (nearest: index in B or -1, min_distance, records or
        None with records=False, n_candidates, n_unsupported)"""
        req = req or P.DistanceRequestPOD()
        ha, ta = self._objects(handles_a, tfs_a)
        na = ha.shape[0]
        nearest = np.empty(na, dtype=np.int32)
        dist = np.empty(na, dtype=np.float64)
        rec = np.empty(na, dtype=P.distance_result_dtype) if records else None
        nc = np.zeros(2, dtype=np.uint32)
        out = P.EnvDistanceOut(nearest.ctypes.data, dist.ctypes.data, None if rec is None else rec.ctypes.data,
                               nc[0:1].ctypes.data, nc[1:2].ctypes.data)
        self._check(self.L.hfb_env_distance(self.h, env, na, _ptr(ha), _ptr(ta), first_a, na if num_a is None else num_a,
                                            C.byref(req), float(max_distance), C.byref(out)))
        return nearest, dist, rec, int(nc[0]), int(nc[1])

    def env_distance_device(self, env, n_a, d_handles_a, d_tfs_a, d_nearest, d_min_distance, d_results, d_n_candidates=None,
                            d_n_unsupported=None, req=None, max_distance=np.inf, stream=0, first_a=0, num_a=None):
        """hfb_env_distance_device: A's handles and poses and every output are device pointers, ordered on `stream`"""
        req = req or P.DistanceRequestPOD()
        out = P.EnvDistanceOut(d_nearest, d_min_distance, d_results, d_n_candidates, d_n_unsupported)
        self._check(self.L.hfb_env_distance_device(self.h, env, n_a, _ptr(d_handles_a), _ptr(d_tfs_a), first_a,
                                                   n_a if num_a is None else num_a, C.byref(req), float(max_distance),
                                                   C.byref(out), _ptr(stream)))

    def env_distance_configs(self, env, handles_a, tfs_a, links_per_config, self_pairs, req=None, max_distance=np.inf,
                             first_config=0, num_configs=None, records=True):
        """each configuration's nearest pair, environment or self (hfb_env_distance_configs) -> (kind: 0 environment,
        1 self, -1 none; first: index in A; second: index in B for kind 0, in A for kind 1, UINT32_MAX for none;
        min_distance; records or None with records=False; n_env_candidates, n_self_candidates, n_unsupported)"""
        req = req or P.DistanceRequestPOD()
        ha, ta = self._objects(handles_a, tfs_a)
        tpl = _template(self_pairs)
        na, lpc = ha.shape[0], int(links_per_config)
        n_configs = na // lpc if lpc else 0
        kind = np.empty(n_configs, dtype=np.int8)
        first = np.empty(n_configs, dtype=np.uint32)
        second = np.empty(n_configs, dtype=np.uint32)
        dist = np.empty(n_configs, dtype=np.float64)
        rec = np.empty(n_configs, dtype=P.distance_result_dtype) if records else None
        nc = np.zeros(3, dtype=np.uint32)
        out = P.ConfigsDistanceOut(kind.ctypes.data, first.ctypes.data, second.ctypes.data, dist.ctypes.data,
                                   None if rec is None else rec.ctypes.data, nc[0:].ctypes.data, nc[1:].ctypes.data,
                                   nc[2:].ctypes.data)
        self._check(self.L.hfb_env_distance_configs(self.h, env, na, _ptr(ha), _ptr(ta), lpc, tpl.shape[0], _ptr(tpl),
                                                    first_config,
                                                    n_configs - first_config if num_configs is None else num_configs,
                                                    C.byref(req), float(max_distance), C.byref(out)))
        return kind, first, second, dist, rec, int(nc[0]), int(nc[1]), int(nc[2])

    def env_distance_configs_device(self, env, n_a, d_handles_a, d_tfs_a, links_per_config, self_pairs, d_kind, d_first,
                                    d_second, d_min_distance, d_results, d_n_env_candidates=None, d_n_self_candidates=None,
                                    d_n_unsupported=None, req=None, max_distance=np.inf, stream=0, first_config=0,
                                    num_configs=None):
        """hfb_env_distance_configs_device: A's handles and poses and every output are device pointers, ordered on
        `stream`; the template is a host array"""
        req = req or P.DistanceRequestPOD()
        tpl = _template(self_pairs)
        lpc = int(links_per_config)
        n_configs = n_a // lpc if lpc else 0
        out = P.ConfigsDistanceOut(d_kind, d_first, d_second, d_min_distance, d_results, d_n_env_candidates,
                                   d_n_self_candidates, d_n_unsupported)
        self._check(self.L.hfb_env_distance_configs_device(self.h, env, n_a, _ptr(d_handles_a), _ptr(d_tfs_a), lpc,
                                                           tpl.shape[0], _ptr(tpl), first_config,
                                                           n_configs - first_config if num_configs is None else num_configs,
                                                           C.byref(req), float(max_distance), C.byref(out), _ptr(stream)))

    def env_collide_motions(self, env, handles_a, tfs_a, links_per_config, self_pairs, offsets, req=None, first_motion=0,
                            num_motions=None, witness=True):
        """motions of configurations (A: configurations of links_per_config objects each, configuration-major, motion m
        is configurations [offsets[m], offsets[m+1])) against the env and against themselves (hfb_env_collide_motions)
        -> (first_invalid: per motion the first colliding sample, -1 for none; kind: 0 environment, 1 self, -1 none;
        first: index in A; second: index in B for kind 0, in A for kind 1, UINT32_MAX for none; contacts: the witness's
        record; counts = (n_env_candidates, n_env_colliding, n_self_candidates, n_self_colliding)).  witness=False:
        first_invalid alone, kind, first, second and contacts None"""
        req = req or P.CollisionRequestPOD()
        ha, ta = self._objects(handles_a, tfs_a)
        tpl = _template(self_pairs)
        off = _offsets(offsets)
        na, n_motions = ha.shape[0], off.shape[0] - 1
        first_invalid = np.empty(n_motions, dtype=np.int32)
        kind = np.empty(n_motions, dtype=np.int8) if witness else None
        first = np.empty(n_motions, dtype=np.uint32) if witness else None
        second = np.empty(n_motions, dtype=np.uint32) if witness else None
        contacts = np.empty(n_motions, dtype=P.contact_dtype) if witness else None
        nc = np.zeros(4, dtype=np.uint32)
        out = P.MotionsOut(first_invalid.ctypes.data, *[None if a is None else a.ctypes.data for a in (kind, first, second, contacts)],
                           *[nc[k:].ctypes.data for k in range(4)])
        self._check(self.L.hfb_env_collide_motions(self.h, env, na, _ptr(ha), _ptr(ta), int(links_per_config), tpl.shape[0],
                                                   _ptr(tpl), n_motions, _ptr(off), first_motion,
                                                   n_motions - first_motion if num_motions is None else num_motions,
                                                   C.byref(req), C.byref(out)))
        return first_invalid, kind, first, second, contacts, tuple(int(c) for c in nc)

    def env_collide_motions_device(self, env, n_a, d_handles_a, d_tfs_a, links_per_config, self_pairs, offsets,
                                   d_first_invalid, d_kind, d_first, d_second, d_contacts, d_counts=(None,) * 4, req=None,
                                   stream=0, first_motion=0, num_motions=None):
        """hfb_env_collide_motions_device: A's handles and poses and every output are device pointers, ordered on
        `stream`; d_counts = (d_n_env_candidates, d_n_env_colliding, d_n_self_candidates, d_n_self_colliding); the
        template and the offsets are host arrays"""
        req = req or P.CollisionRequestPOD()
        tpl = _template(self_pairs)
        off = _offsets(offsets)
        n_motions = off.shape[0] - 1
        out = P.MotionsOut(d_first_invalid, d_kind, d_first, d_second, d_contacts, *d_counts)
        self._check(self.L.hfb_env_collide_motions_device(self.h, env, n_a, _ptr(d_handles_a), _ptr(d_tfs_a),
                                                          int(links_per_config), tpl.shape[0], _ptr(tpl), n_motions,
                                                          _ptr(off), first_motion,
                                                          n_motions - first_motion if num_motions is None else num_motions,
                                                          C.byref(req), C.byref(out), _ptr(stream)))

    def env_certify_motions(self, env, handles_a, tfs_a, sweep, links_per_config, self_pairs, offsets, req=None,
                            first_motion=0, num_motions=None):
        """motions of configurations laid out as in env_collide_motions, each segment between consecutive samples
        certified free from the collide() lower bounds of its end samples and the sweep bounds (sweep: n_a float64,
        sweep[g * L + i] bounding link i's points' path from configuration g to g + 1; hfb_env_certify_motions) ->
        (first_invalid: per motion the first colliding sample, -1 for none; first_uncertified: per motion the first
        segment not certified, -1 for none; certified: per configuration 1 when the segment to the next sample is;
        counts = (n_env_candidates, n_self_candidates, n_unsupported, n_uncertified))"""
        req = req or P.CollisionRequestPOD()
        ha, ta = self._objects(handles_a, tfs_a)
        sw = np.ascontiguousarray(sweep, dtype=np.float64).reshape(-1)
        if sw.shape[0] != ha.shape[0]:
            raise ValueError("sweep: one bound per object of A")
        tpl = _template(self_pairs)
        off = _offsets(offsets)
        na, n_motions, lpc = ha.shape[0], off.shape[0] - 1, int(links_per_config)
        first_invalid = np.empty(n_motions, dtype=np.int32)
        first_uncertified = np.empty(n_motions, dtype=np.int32)
        certified = np.empty(na // lpc if lpc else 0, dtype=np.uint8)
        nc = np.zeros(4, dtype=np.uint32)
        out = P.CertifyOut(first_invalid.ctypes.data, first_uncertified.ctypes.data, certified.ctypes.data,
                           *[nc[k:].ctypes.data for k in range(4)])
        self._check(self.L.hfb_env_certify_motions(self.h, env, na, _ptr(ha), _ptr(ta), _ptr(sw), lpc, tpl.shape[0],
                                                   _ptr(tpl), n_motions, _ptr(off), first_motion,
                                                   n_motions - first_motion if num_motions is None else num_motions,
                                                   C.byref(req), C.byref(out)))
        return first_invalid, first_uncertified, certified, tuple(int(c) for c in nc)

    def env_certify_motions_device(self, env, n_a, d_handles_a, d_tfs_a, d_sweep, links_per_config, self_pairs, offsets,
                                   d_first_invalid, d_first_uncertified, d_certified, d_counts=(None,) * 4, req=None,
                                   stream=0, first_motion=0, num_motions=None):
        """hfb_env_certify_motions_device: A's handles and poses, the sweep bounds and every output are device
        pointers, ordered on `stream`; d_counts = (d_n_env_candidates, d_n_self_candidates, d_n_unsupported,
        d_n_uncertified); the template and the offsets are host arrays"""
        req = req or P.CollisionRequestPOD()
        tpl = _template(self_pairs)
        off = _offsets(offsets)
        n_motions = off.shape[0] - 1
        out = P.CertifyOut(d_first_invalid, d_first_uncertified, d_certified, *d_counts)
        self._check(self.L.hfb_env_certify_motions_device(self.h, env, n_a, _ptr(d_handles_a), _ptr(d_tfs_a),
                                                          _ptr(d_sweep), int(links_per_config), tpl.shape[0], _ptr(tpl),
                                                          n_motions, _ptr(off), first_motion,
                                                          n_motions - first_motion if num_motions is None else num_motions,
                                                          C.byref(req), C.byref(out), _ptr(stream)))

    # -- robot models (hfb_robot_*) -------------------------------------------------------------------------------
    def robot_create(self, parent, types, axis, placement, link_joint, link_placement, link_handles):
        """a robot model on the device (hfb_robot_create): joints (parent: -1 or an earlier joint; types:
        JOINT_REVOLUTE / JOINT_PRISMATIC; axis: 3 per joint; placement: hfb_transform per joint) and links (link_joint:
        -1 or a joint; link_placement; committed geometry handles) -> the robot"""
        desc, keep = robot_desc(parent, types, axis, placement, link_joint, link_placement, link_handles)
        r = C.c_void_p()
        self._check(self.L.hfb_robot_create(self.h, C.byref(desc), C.byref(r)))
        if not hasattr(self, "_robots"):
            self._robots = {}
        self._robots[r.value] = (desc.num_joints, desc.num_links)
        return r

    def robot_destroy(self, robot):
        self._check(self.L.hfb_robot_destroy(self.h, robot))
        self._robots.pop(robot.value, None)

    def robot_dims(self, robot):
        """(num_joints, num_links) of a robot of this engine"""
        return self._robots[robot.value]

    def robot_poses(self, robot, q, handles=True):
        """hfb_robot_poses: q (n_configs x J) -> (link poses, n_configs * L; the link handles tiled, or None)"""
        J, L = self.robot_dims(robot)
        qa = np.ascontiguousarray(q, dtype=np.float64).reshape(-1)
        if qa.shape[0] % J:
            raise ValueError("q: num_joints values per configuration")
        n = qa.shape[0] // J
        tfs = np.empty(n * L, dtype=P.transform_dtype)
        h = np.empty(n * L, dtype=np.uint32) if handles else None
        self._check(self.L.hfb_robot_poses(self.h, robot, n, _ptr(qa), _ptr(tfs), _ptr(h)))
        return tfs, h

    def robot_poses_device(self, robot, n_configs, d_q, d_tfs, d_handles=None, stream=0):
        """hfb_robot_poses_device: q, the poses and the handles are device pointers, ordered on `stream`"""
        self._check(self.L.hfb_robot_poses_device(self.h, robot, int(n_configs), _ptr(d_q), _ptr(d_tfs), _ptr(d_handles),
                                                  _ptr(stream)))

    def robot_sample_motions(self, robot, q_from, q_to, offsets, q=False, sweep=True):
        """hfb_robot_sample_motions: motion m from q_from[m] to q_to[m] (n_motions x J each), sampled
        offsets[m+1] - offsets[m] times, linear in q -> (poses and handles, n_configs * L; the samples' q, n_configs x J,
        or None; the sweep bounds, n_configs * L, or None)"""
        J, L = self.robot_dims(robot)
        off = _offsets(offsets)
        n_motions = off.shape[0] - 1
        qf = np.ascontiguousarray(q_from, dtype=np.float64).reshape(-1)
        qt = np.ascontiguousarray(q_to, dtype=np.float64).reshape(-1)
        if qf.shape[0] != n_motions * J or qt.shape[0] != n_motions * J:
            raise ValueError("q_from, q_to: num_joints values per motion")
        n = int(off[-1])
        tfs = np.empty(n * L, dtype=P.transform_dtype)
        h = np.empty(n * L, dtype=np.uint32)
        qo = np.empty((n, J)) if q else None
        sw = np.empty(n * L) if sweep else None
        out = P.RobotSamplesOut(tfs.ctypes.data, h.ctypes.data, None if qo is None else qo.ctypes.data,
                                None if sw is None else sw.ctypes.data)
        self._check(self.L.hfb_robot_sample_motions(self.h, robot, n_motions, _ptr(qf), _ptr(qt), _ptr(off),
                                                    C.byref(out)))
        return tfs, h, qo, sw

    def robot_sample_motions_device(self, robot, offsets, d_q_from, d_q_to, d_tfs, d_handles, d_q=None, d_sweep=None,
                                    stream=0):
        """hfb_robot_sample_motions_device: the end points and every output are device pointers, ordered on `stream`;
        the offsets are a host array"""
        off = _offsets(offsets)
        out = P.RobotSamplesOut(d_tfs, d_handles, d_q, d_sweep)
        self._check(self.L.hfb_robot_sample_motions_device(self.h, robot, off.shape[0] - 1, _ptr(d_q_from), _ptr(d_q_to),
                                                           _ptr(off), C.byref(out), _ptr(stream)))

    def env_validate_motions(self, env, robot, q_from, q_to, self_pairs, initial_depth, max_depth, max_samples, req=None,
                             first_motion=0, num_motions=None):
        """motion m from q_from[m] to q_to[m] ((n_motions, J) each) sampled by the robot, certified segment by segment
        and the uncertified segments split until each motion is proven free, found colliding or at depth max_depth
        (hfb_env_validate_motions) -> dict: status (0 valid, 1 collides, 2 unresolved, -1 outside the range), t_valid,
        t_collide, the witness (kind, first, second, contacts) and the counts n_rounds, n_samples, n_env_candidates,
        n_self_candidates, n_unsupported"""
        req = req or P.CollisionRequestPOD()
        J, _ = self.robot_dims(robot)
        qf = np.ascontiguousarray(q_from, dtype=np.float64).reshape(-1)
        qt = np.ascontiguousarray(q_to, dtype=np.float64).reshape(-1)
        if qf.shape[0] % J or qt.shape[0] != qf.shape[0]:
            raise ValueError("q_from, q_to: num_joints values per motion, as many motions in each")
        tpl = _template(self_pairs)
        n = qf.shape[0] // J
        r = {"status": np.empty(n, dtype=np.int8), "t_valid": np.empty(n), "t_collide": np.empty(n),
             "kind": np.empty(n, dtype=np.int8), "first": np.empty(n, dtype=np.uint32),
             "second": np.empty(n, dtype=np.uint32), "contacts": np.empty(n, dtype=P.contact_dtype)}
        rounds = np.zeros(1, dtype=np.uint32)
        nc = np.zeros(4, dtype=np.uint64)
        out = P.ValidateOut(*[r[k].ctypes.data for k in ("status", "t_valid", "t_collide", "kind", "first", "second",
                                                         "contacts")], rounds.ctypes.data,
                            *[nc[k:].ctypes.data for k in range(4)])
        p = P.ValidateParams(int(initial_depth), int(max_depth), int(max_samples))
        self._check(self.L.hfb_env_validate_motions(self.h, env, robot, n, _ptr(qf), _ptr(qt), tpl.shape[0], _ptr(tpl),
                                                    first_motion, n - first_motion if num_motions is None else num_motions,
                                                    C.byref(req), C.byref(p), C.byref(out)))
        r["n_rounds"] = int(rounds[0])
        for k, name in enumerate(("n_samples", "n_env_candidates", "n_self_candidates", "n_unsupported")):
            r[name] = int(nc[k])
        return r

    def env_validate_motions_device(self, env, robot, n_motions, d_q_from, d_q_to, self_pairs, initial_depth, max_depth,
                                    max_samples, d_status, d_t_valid, d_t_collide, d_kind=None, d_first=None,
                                    d_second=None, d_contacts=None, d_counts=(None,) * 5, req=None, stream=0,
                                    first_motion=0, num_motions=None):
        """hfb_env_validate_motions_device: the end points and every output are device pointers, ordered on `stream`;
        d_counts = (d_n_rounds (uint32), d_n_samples, d_n_env_candidates, d_n_self_candidates, d_n_unsupported
        (uint64)); the template is a host array"""
        req = req or P.CollisionRequestPOD()
        tpl = _template(self_pairs)
        out = P.ValidateOut(d_status, d_t_valid, d_t_collide, d_kind, d_first, d_second, d_contacts, *d_counts)
        p = P.ValidateParams(int(initial_depth), int(max_depth), int(max_samples))
        self._check(self.L.hfb_env_validate_motions_device(self.h, env, robot, int(n_motions), _ptr(d_q_from),
                                                           _ptr(d_q_to), tpl.shape[0], _ptr(tpl), first_motion,
                                                           n_motions - first_motion if num_motions is None
                                                           else num_motions, C.byref(req), C.byref(p), C.byref(out),
                                                           _ptr(stream)))

    @staticmethod
    def _objects(handles, tfs):
        """an object set as the C ABI takes it: handles and poses, contiguous and of equal length"""
        h = np.ascontiguousarray(handles, dtype=np.uint32)
        t = np.ascontiguousarray(tfs, dtype=P.transform_dtype)
        if h.shape[0] != t.shape[0]:
            raise ValueError("handle and pose arrays must have equal length")
        return h, t

    # -- object-table queries: the batched form of the CollisionObject overloads (collision.h:58-61) -----
    @staticmethod
    def _scene(obj_handles, obj_tfs, first, second):
        oh = np.ascontiguousarray(obj_handles, dtype=np.uint32)
        ot = np.ascontiguousarray(obj_tfs, dtype=P.transform_dtype)
        pi = np.ascontiguousarray(first, dtype=np.uint32)
        pj = np.ascontiguousarray(second, dtype=np.uint32)
        if oh.shape[0] != ot.shape[0] or pi.shape[0] != pj.shape[0]:
            raise ValueError("object table / pair list arrays must have equal length")
        sc = P.ObjectPairs(oh.shape[0], oh.ctypes.data, ot.ctypes.data, pi.shape[0], pi.ctypes.data, pj.ctypes.data)
        return sc, (oh, ot, pi, pj)

    def batch_distance_objects(self, obj_handles, obj_tfs, first, second, req=None, out=None, min_only=False):
        """distance() of the object pairs (first[k], second[k]).  min_only: only DistanceResult::min_distance
        comes back (8 B per pair over PCIe instead of 96)"""
        req = req or P.DistanceRequestPOD()
        sc, keep = self._scene(obj_handles, obj_tfs, first, second)
        n = sc.n_pairs
        if min_only:
            d = np.empty(n, dtype=np.float64) if out is None else out
            self._check(self.L.hfb_batch_distance_objects(self.h, C.byref(sc), C.byref(req), None, _ptr(d), None))
            return d
        if out is None:
            out = np.empty(n, dtype=P.distance_result_dtype)
        self._check(self.L.hfb_batch_distance_objects(self.h, C.byref(sc), C.byref(req), _ptr(out), None, None))
        return out

    def batch_collide_objects(self, obj_handles, obj_tfs, first, second, req=None, out=None, compact_capacity=None):
        """collide() of the object pairs.  compact_capacity = c: -> (flags bit per pair, n_colliding, pair_ids,
        contacts) with the records of at most c colliding pairs, in no particular order; else full records"""
        req = req or P.CollisionRequestPOD()
        sc, keep = self._scene(obj_handles, obj_tfs, first, second)
        n = sc.n_pairs
        if compact_capacity is not None:
            cap = int(compact_capacity)
            flags = np.zeros((n + 31) // 32, dtype=np.uint32)
            nhit = np.zeros(1, dtype=np.uint32)
            ids = np.zeros(max(cap, 1), dtype=np.uint32)
            recs = np.zeros(max(cap, 1), dtype=P.contact_dtype)
            cc = P.CompactContacts(flags.ctypes.data, nhit.ctypes.data, ids.ctypes.data, recs.ctypes.data, cap)
            self._check(self.L.hfb_batch_collide_objects(self.h, C.byref(sc), C.byref(req), None, C.byref(cc), None))
            k = min(int(nhit[0]), cap)
            return flags, int(nhit[0]), ids[:k], recs[:k]
        if out is None:
            out = np.empty(n, dtype=P.contact_dtype)
        self._check(self.L.hfb_batch_collide_objects(self.h, C.byref(sc), C.byref(req), _ptr(out), None, None))
        return out

    def batch_distance_objects_device(self, n_objects, d_handles, d_tfs, n_pairs, d_first, d_second, d_out, req=None,
                                      stream=0):
        req = req or P.DistanceRequestPOD()
        sc = P.ObjectPairs(n_objects, d_handles, d_tfs, n_pairs, d_first, d_second)
        self._check(self.L.hfb_batch_distance_objects_device(self.h, C.byref(sc), C.byref(req), _ptr(d_out), None,
                                                             _ptr(stream)))

    def batch_collide_objects_device(self, n_objects, d_handles, d_tfs, n_pairs, d_first, d_second, d_out, req=None,
                                     stream=0):
        req = req or P.CollisionRequestPOD()
        sc = P.ObjectPairs(n_objects, d_handles, d_tfs, n_pairs, d_first, d_second)
        self._check(self.L.hfb_batch_collide_objects_device(self.h, C.byref(sc), C.byref(req), _ptr(d_out), None,
                                                            _ptr(stream)))

    def batch_convex_support(self, convex_ids, dirs):
        ids = np.ascontiguousarray(convex_ids, dtype=np.uint32)
        d = np.ascontiguousarray(dirs, dtype=np.float64).reshape(-1, 3)
        idx = np.zeros(ids.shape[0], dtype=np.int32)
        sup = np.zeros((ids.shape[0], 3), dtype=np.float64)
        self._check(self.L.hfb_batch_convex_support(self.h, ids.shape[0], _ptr(ids), _ptr(d), _ptr(idx),
                                                    _ptr(sup)))
        return idx, sup

    # -- device-buffer queries (raw device pointers, async on `stream`) ------
    def batch_distance_device(self, n, d_h1, d_tf1, d_h2, d_tf2, d_out, req=None, stream=0, d_guess=None):
        req = req or P.DistanceRequestPOD()
        self._check(self.L.hfb_batch_distance_device(self.h, n, _ptr(d_h1), _ptr(d_tf1), _ptr(d_h2),
                                                     _ptr(d_tf2), C.byref(req), _ptr(d_out),
                                                     C.byref(d_guess) if d_guess is not None else None,
                                                     _ptr(stream)))

    def batch_collide_device(self, n, d_h1, d_tf1, d_h2, d_tf2, d_out, req=None, stream=0, d_guess=None):
        req = req or P.CollisionRequestPOD()
        self._check(self.L.hfb_batch_collide_device(self.h, n, _ptr(d_h1), _ptr(d_tf1), _ptr(d_h2),
                                                    _ptr(d_tf2), C.byref(req), _ptr(d_out),
                                                    C.byref(d_guess) if d_guess is not None else None,
                                                    _ptr(stream)))

    def batch_convex_support_device(self, n, d_ids, d_dirs, d_idx, d_sup, stream=0):
        self._check(self.L.hfb_batch_convex_support_device(self.h, n, _ptr(d_ids), _ptr(d_dirs),
                                                           _ptr(d_idx), _ptr(d_sup), _ptr(stream)))

    # -- multi-GPU: one context per rank (hfb_comm_*), NCCL behind the C-ABI -----------------------------------
    @staticmethod
    def comm_unique_id():
        """128 bytes rank 0 creates and hands to every rank (ncclGetUniqueId)"""
        L = load_library()
        buf = C.create_string_buffer(128)
        rc = L.hfb_comm_unique_id(buf)
        if rc != 0:
            raise EngineError("hfb_comm_unique_id: %s" % _ERR.get(rc, rc))
        return buf.raw

    def comm_init(self, comm_id, rank, nranks):
        self._check(self.L.hfb_comm_init(self.h, C.create_string_buffer(bytes(comm_id), 128), int(rank), int(nranks)))

    def comm_destroy(self):
        self._check(self.L.hfb_comm_destroy(self.h))

    def geom_broadcast(self, root=0):
        """the geometry registered on `root` replaces this context's, on every rank, committed"""
        self._check(self.L.hfb_geom_broadcast(self.h, int(root)))

    def batch_distance_sharded_device(self, n_local, d_h1, d_tf1, d_h2, d_tf2, req=None, stream=0):
        """-> device pointer of the records of all ranks' pairs (rank-major); complete after comm_wait(stream)"""
        req = req or P.DistanceRequestPOD()
        out = C.c_void_p()
        self._check(self.L.hfb_batch_distance_sharded_device(self.h, n_local, _ptr(d_h1), _ptr(d_tf1), _ptr(d_h2), _ptr(d_tf2),
                                                             C.byref(req), C.byref(out), _ptr(stream)))
        return out.value

    def batch_collide_sharded_device(self, n_local, d_h1, d_tf1, d_h2, d_tf2, req=None, stream=0):
        req = req or P.CollisionRequestPOD()
        out = C.c_void_p()
        self._check(self.L.hfb_batch_collide_sharded_device(self.h, n_local, _ptr(d_h1), _ptr(d_tf1), _ptr(d_h2), _ptr(d_tf2),
                                                            C.byref(req), C.byref(out), _ptr(stream)))
        return out.value

    def comm_wait(self, stream=0):
        self._check(self.L.hfb_comm_wait(self.h, _ptr(stream)))

    def set_profiling(self, on=True):
        self._check(self.L.hfb_set_profiling(self.h, int(on)))

    def kernel_times(self, reset=True):
        t = P.KernelTimes()
        self._check(self.L.hfb_get_kernel_times(self.h, C.byref(t), int(reset)))
        return {f[0]: getattr(t, f[0]) for f in P.KernelTimes._fields_}

    def stats(self):
        s = P.Stats()
        self._check(self.L.hfb_get_stats(self.h, C.byref(s)))
        return {f[0]: getattr(s, f[0]) for f in P.Stats._fields_}
