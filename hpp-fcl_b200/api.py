"""Host-side mirror of the hpp-fcl query interface for the accelerated path.

Same names, argument meaning and error behaviour as the reference's Python /
C++ surface for this path (python/collision.cc, python/distance.cc;
include/hpp/fcl/{collision,distance,collision_data}.h):

    collide(o1, tf1, o2, tf2, request, result) -> number of contacts
    distance(o1, tf1, o2, tf2, request, result) -> min distance
    ComputeCollision / ComputeDistance functors (collision.h:79-117)
    BatchQuery: the batched form (many (o1,tf1,o2,tf2) tuples, one launch)

Every call runs on the GPU through the C-ABI (engine.Engine); there is no CPU
path.  Single-pair calls are batches of one.
"""
import numpy as np

from . import _pod as P
from .engine import Engine

_NAN3 = np.full(3, np.nan)


# ---------------------------------------------------------------- geometry ---
class Transform3f:
    """math/transform.h:56-216 (rotation matrix + translation)."""

    def __init__(self, R=None, T=None):
        self.R = np.eye(3) if R is None else np.asarray(R, dtype=np.float64).reshape(3, 3)
        self.T = np.zeros(3) if T is None else np.asarray(T, dtype=np.float64).reshape(3)

    @staticmethod
    def from_quat(w, x, y, z, T=None):
        from .workloads import quat_to_rot
        return Transform3f(quat_to_rot(w, x, y, z), T)

    def transform(self, v):
        return self.R @ np.asarray(v, dtype=np.float64) + self.T

    def __mul__(self, o):  # transform.h:186-188
        return Transform3f(self.R @ o.R, self.R @ o.T + self.T)

    def getRotation(self):
        return self.R

    def getTranslation(self):
        return self.T

    def setTranslation(self, T):
        self.T = np.asarray(T, dtype=np.float64).reshape(3)

    def pod(self):
        return P.make_transforms(self.R[None], self.T[None])


class CollisionGeometry:
    node_type = None

    def __init__(self):
        self._ssr = 0.0

    def setSweptSphereRadius(self, r):  # geometric_shapes.h:77-85
        if r < 0:
            raise ValueError("Swept-sphere radius must be positive.")
        self._ssr = float(r)

    def getSweptSphereRadius(self):
        return self._ssr

    def getNodeType(self):
        return self.node_type

    def _params(self):
        return (0.0, 0.0, 0.0)

    def _points(self):
        return None


class Box(CollisionGeometry):
    node_type = P.GEOM_BOX

    def __init__(self, x, y=None, z=None):  # full side lengths; halfSide = side / 2 (geometric_shapes.h:164-187)
        super().__init__()
        side = np.asarray(x if y is None else (x, y, z), dtype=np.float64)
        self.halfSide = side / 2

    def _params(self):
        return tuple(self.halfSide)


class Sphere(CollisionGeometry):
    node_type = P.GEOM_SPHERE

    def __init__(self, radius):
        super().__init__()
        self.radius = float(radius)

    def _params(self):
        return (self.radius, 0.0, 0.0)


class Ellipsoid(CollisionGeometry):
    node_type = P.GEOM_ELLIPSOID

    def __init__(self, rx, ry=None, rz=None):
        super().__init__()
        self.radii = np.asarray(rx if ry is None else (rx, ry, rz), dtype=np.float64)

    def _params(self):
        return tuple(self.radii)


class _RadiusLength(CollisionGeometry):
    def __init__(self, radius, lz):  # halfLength = lz / 2 (geometric_shapes.h:386-400)
        super().__init__()
        self.radius = float(radius)
        self.halfLength = float(lz) / 2

    def _params(self):
        return (self.radius, self.halfLength, 0.0)


class Capsule(_RadiusLength):
    node_type = P.GEOM_CAPSULE


class Cone(_RadiusLength):
    node_type = P.GEOM_CONE


class Cylinder(_RadiusLength):
    node_type = P.GEOM_CYLINDER


class _PlaneBase(CollisionGeometry):
    """n . x <= d (Halfspace) or n . x = d (Plane); the constructor normalises (n, d) (unitNormalTest,
    src/shape/geometric_shapes.cpp:121-143)."""

    def __init__(self, a, b=None, c=None, d=None):  # (n, d) or (a, b, c, d): geometric_shapes.h:887-896, 979-988
        super().__init__()
        if c is None:
            n, off = np.asarray(a, dtype=np.float64).reshape(3).copy(), float(0.0 if b is None else b)
        else:
            n, off = np.array([a, b, c], dtype=np.float64), float(d)
        l = float(np.sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]))
        if l > 0:
            inv_l = 1.0 / l
            n, off = n * inv_l, off * inv_l
        else:
            n, off = np.array([1.0, 0.0, 0.0]), 0.0
        self.n, self.d = n, off

    def _params(self):
        return tuple(self.n)

    def _plane(self):
        return np.array([self.n[0], self.n[1], self.n[2], self.d], dtype=np.float64)


class Halfspace(_PlaneBase):  # geometric_shapes.h:885-961
    node_type = P.GEOM_HALFSPACE

    def signedDistance(self, p):
        return float(np.dot(self.n, p) - (self.d + self._ssr))


class Plane(_PlaneBase):  # geometric_shapes.h:977-1050
    node_type = P.GEOM_PLANE


class Convex(CollisionGeometry):
    """ConvexBase / Convex<Triangle> (geometric_shapes.h:638-872, shape/convex.h)."""
    node_type = P.GEOM_CONVEX

    def __init__(self, points, triangles=None):
        super().__init__()
        self.points = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        self.num_points = self.points.shape[0]
        self.triangles = None if triangles is None else np.ascontiguousarray(triangles, dtype=np.uint32)

    def _points(self):
        return self.points


class TriangleP(CollisionGeometry):
    node_type = P.GEOM_TRIANGLE

    def __init__(self, a, b, c):
        super().__init__()
        self.a, self.b, self.c = [np.asarray(v, dtype=np.float64).reshape(3) for v in (a, b, c)]

    def _points(self):
        return np.stack([self.a, self.b, self.c])


class BVHModelOBBRSS(CollisionGeometry):
    """BVHModel<OBBRSS> (include/hpp/fcl/BVH/BVH_model.h) with the reference's build protocol; the tree is
    built on the host by the library (hfb_bvh_build_obbrss, mean split), the queries walk it on the GPU."""
    node_type = P.BV_OBBRSS

    def __init__(self):
        super().__init__()
        self._verts, self._tris = [], []
        self.vertices = self.tri_indices = self.bvs = None
        self._begun = False

    def beginModel(self, num_tris=0, num_vertices=0):
        self._verts, self._tris = [], []
        self.vertices = self.tri_indices = self.bvs = None
        self._begun = True
        return 0

    def _need_begun(self):
        if not self._begun:
            raise ValueError("BVH construction does not follow correct sequence (beginModel first)")

    def addVertex(self, p):
        self._need_begun()
        self._verts.append(np.asarray(p, dtype=np.float64).reshape(3))
        return 0

    def addTriangle(self, p1, p2, p3):  # BVH_model.cpp:359-414: three new vertices
        self._need_begun()
        o = len(self._verts)
        for p in (p1, p2, p3):
            self.addVertex(p)
        self._tris.append((o, o + 1, o + 2))
        return 0

    def addSubModel(self, points, triangles):  # :470-538
        self._need_begun()
        o = len(self._verts)
        for p in np.asarray(points, dtype=np.float64).reshape(-1, 3):
            self._verts.append(p)
        for t in np.asarray(triangles, dtype=np.int64).reshape(-1, 3):
            self._tris.append((int(t[0]) + o, int(t[1]) + o, int(t[2]) + o))
        return 0

    def endModel(self):
        self._need_begun()
        if not self._tris:
            raise ValueError("BVH construction error: empty model")
        from .engine import build_bvh_obbrss
        self.vertices = np.ascontiguousarray(np.stack(self._verts), dtype=np.float64)
        self.tri_indices = np.ascontiguousarray(np.array(self._tris), dtype=np.uint32)
        self.bvs = build_bvh_obbrss(self.vertices, self.tri_indices)
        self.num_vertices, self.num_tris = len(self.vertices), len(self.tri_indices)
        self._begun = False
        return 0

    def getNumBVs(self):
        return 0 if self.bvs is None else len(self.bvs)


class BVHModelOBB(BVHModelOBBRSS):
    """BVHModel<OBB>: collide() only, as in the library (distance() on a plain OBB model is not offered, see
    hfb_geom_register_bvh_obb).  The plain OBB tree of a mesh is the OBB half of its OBBRSS tree, so the builder is shared."""
    node_type = P.BV_OBB


_MESH_TYPES = (P.BV_OBBRSS, P.BV_OBB)


# ---------------------------------------------------------- requests/results --
class _QueryRequest:
    _pod_cls = None

    def __init__(self, **kw):
        self._pod = self._pod_cls(**kw)

    def __getattr__(self, k):
        pod = object.__getattribute__(self, "_pod")
        if hasattr(pod.q, k):
            return getattr(pod.q, k)
        return getattr(pod, k)

    def __setattr__(self, k, v):
        if k == "_pod":
            object.__setattr__(self, k, v)
        elif hasattr(self._pod.q, k):
            setattr(self._pod.q, k, v)
        elif hasattr(self._pod, k):
            setattr(self._pod, k, v)
        else:
            raise AttributeError(k)


class CollisionRequest(_QueryRequest):  # collision_data.h:312-383
    _pod_cls = P.CollisionRequestPOD


class DistanceRequest(_QueryRequest):  # collision_data.h:987-1050
    _pod_cls = P.DistanceRequestPOD


class Contact:  # collision_data.h:59-166
    NONE = -1

    def __init__(self, o1, o2, rec):
        self.o1, self.o2 = o1, o2
        self.b1, self.b2 = int(rec["b1"]), int(rec["b2"])
        self.normal = rec["normal"].copy()
        self.nearest_points = [rec["p1"].copy(), rec["p2"].copy()]
        self.pos = rec["pos"].copy()
        self.penetration_depth = float(rec["distance"])


class CollisionResult:  # collision_data.h:391-509
    def __init__(self):
        self.clear()

    def clear(self):
        self.contacts = []
        self.distance_lower_bound = P.DBL_MAX
        self.normal = _NAN3.copy()
        self.nearest_points = [_NAN3.copy(), _NAN3.copy()]
        self.cached_gjk_guess = np.array([1.0, 0.0, 0.0])
        self.cached_support_func_guess = np.zeros(2, dtype=np.int32)

    def numContacts(self):
        return len(self.contacts)

    def isCollision(self):
        return len(self.contacts) > 0

    def getContact(self, i):
        if i >= len(self.contacts):
            raise IndexError("The index is out of range.")
        return self.contacts[i]


class DistanceResult:  # collision_data.h:1053-1174
    NONE = -1

    def __init__(self):
        self.clear()

    def clear(self):
        self.min_distance = P.DBL_MAX
        self.nearest_points = [_NAN3.copy(), _NAN3.copy()]
        self.normal = _NAN3.copy()
        self.o1 = self.o2 = None
        self.b1 = self.b2 = -1
        self.cached_gjk_guess = np.array([1.0, 0.0, 0.0])
        self.cached_support_func_guess = np.zeros(2, dtype=np.int32)


# ----------------------------------------------------------------- engine ----
_DEFAULT = {}


def default_engine(device=0):
    if device not in _DEFAULT:
        _DEFAULT[device] = _Scene(Engine(device))
    return _DEFAULT[device]


class _Scene:
    """Geometry handle cache keyed by object identity (the arena of SURVEY 8b)."""

    def __init__(self, engine):
        self.engine = engine
        self._handles = {}
        self._dirty = False

    @staticmethod
    def _content(geom):
        """what the arena holds for `geom` beyond its record: the vertices of a hull / triangle, the mesh of a model"""
        pts = geom._points()
        if geom.node_type in _MESH_TYPES:
            return (np.ascontiguousarray(geom.bvs).tobytes() if geom.bvs is not None else None,
                    np.ascontiguousarray(geom.vertices, dtype=np.float64).tobytes(),
                    np.ascontiguousarray(geom.tri_indices, dtype=np.uint32).tobytes())
        return np.ascontiguousarray(pts, dtype=np.float64).tobytes() if pts is not None else None

    def handle(self, geom):
        """the arena handle of `geom`, registered on first use.  A geometry changed in place since (new sizes, new
        swept-sphere radius, moved hull vertices) keeps its handle: the record / vertex set is updated
        (hfb_geom_update_shapes / hfb_geom_update_convex); only a change the arena cannot absorb -- another number of
        vertices, another mesh -- retires the handle and registers a new one."""
        key = id(geom)
        ent = self._handles.get(key)
        if geom.node_type in (P.GEOM_PLANE, P.GEOM_HALFSPACE):
            # (n, d) live outside the 40-byte record: a plane changed in place is registered anew
            sig = (geom.node_type, tuple(geom._plane().tolist()), geom.getSweptSphereRadius())
            if ent is not None and ent[2] is geom:
                if ent[1] == sig:
                    return ent[0]
                self.engine.release_shapes([ent[0]])
            h = int(self.engine.register_halfspaces(geom.node_type, geom._plane(), [geom.getSweptSphereRadius()])[0])
            self._handles[key] = (h, sig, geom, None, 0)
            self._dirty = True
            return h
        sig = (geom.node_type, tuple(np.asarray(geom._params(), dtype=np.float64).tolist()), geom.getSweptSphereRadius())
        content = self._content(geom)
        if ent is not None and ent[2] is geom:
            h, old_sig, _, old_content, data = ent
            if old_sig == sig and old_content == content:
                return h
            same_kind = old_sig[0] == sig[0]
            pts = geom._points()
            if same_kind and geom.node_type not in _MESH_TYPES and (
                    old_content == content or (pts is not None and old_content is not None and len(old_content) == len(content))):
                if old_content != content:
                    self.engine.update_convex(data, pts)
                rec = P.make_shapes([geom.node_type], [geom._params()], ssr=geom.getSweptSphereRadius(), data=data)
                self.engine.update_shapes([h], rec)
                self._handles[key] = (h, sig, geom, content, data)
                self._dirty = True
                return h
            self.engine.release_shapes([h])  # the storage of its vertices / mesh stays until hfb_geom_clear
        data = 0
        pts = geom._points()
        if geom.node_type in _MESH_TYPES:
            if geom.bvs is None:
                raise ValueError("BVHModel: endModel() was not called")
            reg = self.engine.register_bvh_obb if geom.node_type == P.BV_OBB else self.engine.register_bvh_obbrss
            data = reg(geom.bvs, geom.vertices, geom.tri_indices)
        elif pts is not None:
            data = self.engine.register_convex(pts)
        rec = P.make_shapes([geom.node_type], [geom._params()], ssr=geom.getSweptSphereRadius(), data=data)
        h = int(self.engine.register_shapes(rec)[0])
        self._handles[key] = (h, sig, geom, content, data)
        self._dirty = True
        return h

    def commit(self):
        if self._dirty:
            self.engine.commit()
            self._dirty = False


def _tf_array(tfs):
    if isinstance(tfs, np.ndarray) and tfs.dtype == P.transform_dtype:
        return tfs
    if isinstance(tfs, Transform3f):
        tfs = [tfs]
    R = np.stack([t.R for t in tfs])
    T = np.stack([t.T for t in tfs])
    return P.make_transforms(R, T)


class BatchQuery:
    """Batched collide()/distance(): the seam a broadphase CollisionCallBackCollect
    (broadphase/default_broadphase_callbacks.h:224-252) feeds."""

    def __init__(self, device=0):
        self.scene = default_engine(device)

    def handles(self, geoms):
        return np.array([self.scene.handle(g) for g in geoms], dtype=np.uint32)

    def distance(self, geoms1, tfs1, geoms2, tfs2, request=None):
        request = request or DistanceRequest()
        h1, h2 = self.handles(geoms1), self.handles(geoms2)
        self.scene.commit()
        return self.scene.engine.batch_distance(h1, _tf_array(tfs1), h2, _tf_array(tfs2), request._pod)

    def collide(self, geoms1, tfs1, geoms2, tfs2, request=None):
        request = request or CollisionRequest()
        if request.num_max_contacts == 0:  # collision.cpp:82-85
            raise ValueError("Invalid number of max contacts (current value is 0).")
        h1, h2 = self.handles(geoms1), self.handles(geoms2)
        self.scene.commit()
        return self.scene.engine.batch_collide(h1, _tf_array(tfs1), h2, _tf_array(tfs2), request._pod)


# ------------------------------------------------------------- broadphase seam --
class AABB:  # BV/AABB.h
    def __init__(self, min_=None, max_=None):
        self.min_ = np.full(3, np.inf) if min_ is None else np.asarray(min_, dtype=np.float64)
        self.max_ = np.full(3, -np.inf) if max_ is None else np.asarray(max_, dtype=np.float64)

    def overlap(self, other):  # :111-118, closed intervals
        return bool(np.all(self.min_ <= other.max_) and np.all(self.max_ >= other.min_))


class CollisionObject:  # collision_object.h:214-330 (geometry + pose + world-space box)
    def __init__(self, geom, tf=None):
        self.geom = geom
        self.tf = tf if tf is not None else Transform3f()
        self.aabb = AABB()

    def collisionGeometry(self):
        return self.geom

    def getTransform(self):
        return self.tf

    def setTransform(self, tf):
        self.tf = tf

    def getAABB(self):
        return self.aabb


class CollisionCallBackCollect:  # broadphase/default_broadphase_callbacks.h:224-252, .cpp:95-120
    def __init__(self, max_size=0):
        self.max_size = max_size
        self.collision_pairs = []

    def init(self):
        self.collision_pairs = []

    def collide(self, o1, o2):
        self.collision_pairs.append((o1, o2))
        return False

    __call__ = collide

    def numCollisionPairs(self):
        return len(self.collision_pairs)

    def getCollisionPairs(self):
        return self.collision_pairs

    def exist(self, o1, o2):
        return any(a is o1 and b is o2 for a, b in self.collision_pairs)


class DynamicAABBTreeCollisionManager:
    """BroadPhaseCollisionManager's interface (broadphase/broadphase_collision_manager.h:56-134) for the self-collision
    query: setup() / update() compute every object's box (CollisionObject::computeAABB, on the device), collide(callback)
    reports every pair of objects with overlapping boxes once -- the SET the reference's managers report
    (broadphase_dynamic_AABB_tree.cpp:336-407,716-721); the order is each manager's own.  No tree is kept: a uniform grid
    is rebuilt per query.  collide_batch() is what the seam is for: candidates + batched narrow phase in one go."""

    def __init__(self, device=0):
        self.scene = default_engine(device)
        self.objs = []
        self._stale = True
        self._handles = self._tfs = self._boxes = None

    def registerObject(self, obj):
        self.objs.append(obj)
        self._stale = True

    def registerObjects(self, objs):
        self.objs.extend(objs)
        self._stale = True

    def unregisterObject(self, obj):
        self.objs = [o for o in self.objs if o is not obj]
        self._stale = True

    def clear(self):
        self.objs = []
        self._stale = True

    def size(self):
        return len(self.objs)

    def empty(self):
        return not self.objs

    def getObjects(self):
        return list(self.objs)

    def _refresh(self):
        self._handles = np.array([self.scene.handle(o.geom) for o in self.objs], dtype=np.uint32)
        self.scene.commit()
        self._tfs = _tf_array([o.tf for o in self.objs]) if self.objs else np.zeros(0, dtype=P.transform_dtype)
        self._boxes = self.scene.engine.scene_aabbs(self._handles, self._tfs) if self.objs else np.zeros((0, 6))
        for o, b in zip(self.objs, self._boxes):
            o.aabb = AABB(b[:3].copy(), b[3:].copy())
        self._stale = False

    def setup(self):
        self._refresh()

    def update(self, objs=None):
        """update(): every object's box again; update(obj) / update(objs): the boxes of those objects from their current
        poses (broadphase_collision_manager.h:76-79)"""
        if objs is None or self._stale:
            self._refresh()
            return
        if isinstance(objs, CollisionObject):
            objs = [objs]
        where = {id(o): i for i, o in enumerate(self.objs)}
        objs = [o for o in objs if id(o) in where]  # an object the manager does not hold is skipped, as the reference does
        idx = np.array([where[id(o)] for o in objs], dtype=np.int64)
        if idx.size == 0:
            return
        self._tfs[idx] = _tf_array([o.tf for o in objs])
        bb = self.scene.engine.scene_aabbs(self._handles[idx], self._tfs[idx])
        self._boxes[idx] = bb
        for o, b in zip(objs, bb):
            o.aabb = AABB(b[:3].copy(), b[3:].copy())

    def _table(self, other):
        """(handles, poses, boxes, objects) of `other`: another manager (refreshed if stale) or one CollisionObject,
        whose box is computed here as setup() computes the manager's"""
        if isinstance(other, DynamicAABBTreeCollisionManager):
            if other._stale:
                other._refresh()
            return other._handles, other._tfs, other._boxes, other.objs
        h = np.array([self.scene.handle(other.geom)], dtype=np.uint32)
        self.scene.commit()
        tf = _tf_array([other.tf])
        bb = self.scene.engine.scene_aabbs(h, tf)
        other.aabb = AABB(bb[0, :3].copy(), bb[0, 3:].copy())
        return h, tf, bb, [other]

    def _cross(self, other):
        """-> (first, second, other's table): the cross candidates of this manager against `other` (a manager or a
        CollisionObject), first in this manager, second in `other`; other's table computed once"""
        if self._stale:
            self._refresh()
        from .engine import broadphase_cross_pairs
        table = self._table(other)
        first, second = broadphase_cross_pairs(self._boxes, table[2])
        return first, second, table

    def pairs(self, other=None):
        """the candidate pairs as object indices: first < second in this manager; or, with `other` (a manager or a
        CollisionObject), first in this manager and second in `other`"""
        if other is not None and other is not self:
            return self._cross(other)[:2]
        if self._stale:
            self._refresh()
        from .engine import broadphase_pairs
        return broadphase_pairs(self._boxes)

    def collide(self, other=None, callback=None):
        """collide(callback): every pair of this manager's objects with overlapping boxes.  collide(other, callback):
        o1 from this manager, o2 from `other`, another manager (collide(self, cb) is the self form) or one
        CollisionObject -- o2 is then that object, the order of DynamicAABBTreeCollisionManager::collide(obj)
        (broadphase_dynamic_AABB_tree.cpp:361-390; NaiveCollisionManager passes (obj, object) instead)"""
        if callback is None:  # collide(cb) / collide(callback=cb)
            other, callback = None, other
        callback.init()
        if other is None or other is self:
            first, second = self.pairs()
            objs_b = self.objs
        else:
            first, second, table = self._cross(other)
            objs_b = table[3]
        for a, b in zip(first.tolist(), second.tolist()):
            if callback(self.objs[a], objs_b[b]):
                return

    def collide_batch(self, request=None, other=None):
        """-> (first, second, contact records) of ALL candidate pairs: one hfb_batch_collide_objects call.  With
        `other` (a manager or a CollisionObject): the cross pairs, o1 from this manager, o2 from `other`, over the
        object table [this manager; other]"""
        request = request or CollisionRequest()
        if request.num_max_contacts == 0:
            raise ValueError("Invalid number of max contacts (current value is 0).")
        if other is None or other is self:
            first, second = self.pairs()
            rec = self.scene.engine.batch_collide_objects(self._handles, self._tfs, first, second, request._pod)
            return first, second, rec
        first, second, (hb, tb, _, _) = self._cross(other)
        n = len(self._handles)
        rec = self.scene.engine.batch_collide_objects(np.concatenate([self._handles, hb]), np.concatenate([self._tfs, tb]),
                                                      first, second + np.uint32(n), request._pod)
        return first, second, rec


class ResidentEnvironment:
    """A manager's objects kept on the device as set B of the two-set collide (hfb_env): its table, its boxes as of
    construction / update(objs) and the grid over them stay there between queries, as the reference's tree does between
    setup() and update().  Its queries (collide(), distance() and their forms per configuration) upload only the robot
    manager's poses.  close() (or leaving a `with` block) frees it."""

    def __init__(self, manager):
        if manager._stale:
            manager._refresh()
        self.engine = manager.scene.engine
        self._index = {id(o): i for i, o in enumerate(manager.objs)}
        self._env = self.engine.env_create(manager._handles, manager._tfs)

    def update(self, objs):
        """the current poses of these environment objects (one CollisionObject or several) pushed to the device"""
        if isinstance(objs, CollisionObject):
            objs = [objs]
        if any(id(o) not in self._index for o in objs):  # (the C++ mirror throws std::invalid_argument)
            raise ValueError("not an object of this environment")
        idx = np.array([self._index[id(o)] for o in objs], dtype=np.uint32)
        tfs = _tf_array([o.tf for o in objs]) if len(objs) else np.zeros(0, dtype=P.transform_dtype)
        self.engine.env_update(self._env, idx, tfs)

    @staticmethod
    def _robot(robot_manager, request):
        request = request or CollisionRequest()
        if request.num_max_contacts == 0 and request.security_margin != -np.inf:
            raise ValueError("Invalid number of max contacts (current value is 0).")
        if robot_manager._stale:
            robot_manager._refresh()
        return robot_manager._handles, robot_manager._tfs, request._pod

    def collide(self, robot_manager, request=None, capacity=None):
        """-> (first = index in the robot manager, second = index in the environment, contact records) of the colliding
        pairs, in no particular order"""
        h, t, req = self._robot(robot_manager, request)
        first, second, rec, _, hits = self.engine.env_collide(self._env, h, t, req, capacity=capacity)
        if capacity is None and hits > len(first):  # (all of them unless a capacity is given)
            first, second, rec, _, _ = self.engine.env_collide(self._env, h, t, req, capacity=hits)
        return first, second, rec

    def collide_flags(self, robot_manager, request=None):
        """-> one byte per robot object: 1 iff it collides with the environment (no pair records come back)"""
        h, t, req = self._robot(robot_manager, request)
        return self.engine.env_collide(self._env, h, t, req, capacity=0, flags=True)[5]

    def collide_configurations(self, robot_manager, links_per_config, self_pairs, request=None, capacity=None):
        """A planner's validity check: the robot manager holds configurations of links_per_config objects each,
        configuration-major (object g * L + i is link i of configuration g); self_pairs is the template of link pairs
        (i, j) each configuration checks against itself (an SRDF's enabled pairs).  -> (verdicts: one byte per
        configuration, 1 iff it collides with the environment or with itself; environment pairs (first = index in the
        robot manager, second = index in the environment, contact records); self pairs (first, second: indices in the
        robot manager, contact records)), the pairs in no particular order"""
        h, t, req = self._robot(robot_manager, request)
        v, e, s = self.engine.env_collide_configs(self._env, h, t, links_per_config, self_pairs, req, capacity, capacity)
        if capacity is None and (e[4] > len(e[0]) or s[4] > len(s[0])):  # (all of them unless a capacity is given)
            v, e, s = self.engine.env_collide_configs(self._env, h, t, links_per_config, self_pairs, req, e[4], s[4])
        return v, e[:3], s[:3]

    def configuration_flags(self, robot_manager, links_per_config, self_pairs, request=None):
        """-> one byte per configuration: 1 iff it collides with the environment or with itself (no pair records come
        back)"""
        h, t, req = self._robot(robot_manager, request)
        return self.engine.env_collide_configs(self._env, h, t, links_per_config, self_pairs, req, 0, 0)[0]

    def distance(self, robot_manager, request=None, max_distance=np.inf):
        """each robot object's nearest environment object -> (nearest: index in the environment, -1 when none is
        eligible; min_distance: DBL_MAX when none; the distance records).  distance() runs with a fresh DistanceResult on
        each pair; the eligible pairs are those at min_distance <= max_distance (>= 0 or inf) and not unsupported; the
        smallest distance wins, the lowest environment index on ties (include/hppfcl_b200.h, hfb_env_distance)"""
        h, t, req = self._distance_args(robot_manager, request, max_distance)
        return self.engine.env_distance(self._env, h, t, req, max_distance)[:3]

    def clearance(self, robot_manager, max_distance=np.inf, request=None):
        """-> min_distance of distance() alone: each robot object's distance to its nearest environment object (no
        records come back)"""
        h, t, req = self._distance_args(robot_manager, request, max_distance)
        return self.engine.env_distance(self._env, h, t, req, max_distance, records=False)[1]

    def distance_configurations(self, robot_manager, links_per_config, self_pairs, request=None, max_distance=np.inf):
        """A planner's clearance: the robot manager holds configurations of links_per_config objects each,
        configuration-major, and self_pairs is the template of link pairs (i, j) each configuration checks against
        itself.  -> per configuration its nearest pair over the environment pairs and the template's self pairs: (kind:
        0 environment, 1 self, -1 none eligible; first: index in the robot manager; second: index in the environment
        for kind 0, in the robot manager for kind 1; min_distance: DBL_MAX when none; the distance records).  The
        eligible pairs and the argmin are those of distance(); on a tie an environment pair beats a self pair, and
        earlier links and template entries beat later ones (include/hppfcl_b200.h, hfb_env_distance_configs)"""
        h, t, req = self._distance_args(robot_manager, request, max_distance)
        tpl = self._template_args(links_per_config, self_pairs)
        return self.engine.env_distance_configs(self._env, h, t, links_per_config, tpl, req, max_distance)[:5]

    def configuration_clearance(self, robot_manager, links_per_config, self_pairs, max_distance=np.inf, request=None):
        """-> min_distance of distance_configurations() alone: each configuration's clearance (no records come back)"""
        h, t, req = self._distance_args(robot_manager, request, max_distance)
        tpl = self._template_args(links_per_config, self_pairs)
        return self.engine.env_distance_configs(self._env, h, t, links_per_config, tpl, req, max_distance,
                                                records=False)[3]

    def collide_motions(self, robot_manager, links_per_config, self_pairs, motion_offsets, request=None, first_motion=0,
                        num_motions=None):
        """A planner's motion validation: the robot manager holds configurations laid out as in
        collide_configurations(), the samples of each motion one after another in walking order; motion m is
        configurations [motion_offsets[m], motion_offsets[m+1]).  -> per motion (first_invalid: the first sample that
        collides with the environment or with itself, -1 when none does; kind: 0 environment pair, 1 self pair, -1 none;
        first: index in the robot manager; second: index in the environment for kind 0, in the robot manager for kind 1;
        contacts: the pair's contact record).  The pair is the first colliding one of that sample: environment pairs by
        link, then by environment index, then self pairs in template order (include/hppfcl_b200.h,
        hfb_env_collide_motions).  Only motions [first_motion, first_motion + num_motions) are checked; the others
        get the no-witness values."""
        h, t, req = self._robot(robot_manager, request)
        tpl = self._template_args(links_per_config, self_pairs)
        off, first_motion, num_motions = self._motion_args(len(h), links_per_config, motion_offsets, first_motion,
                                                           num_motions)
        return self.engine.env_collide_motions(self._env, h, t, links_per_config, tpl, off, req, first_motion,
                                               num_motions)[:5]

    def first_invalid_samples(self, robot_manager, links_per_config, self_pairs, motion_offsets, request=None,
                              first_motion=0, num_motions=None):
        """-> first_invalid of collide_motions() alone (no pair records come back)"""
        h, t, req = self._robot(robot_manager, request)
        tpl = self._template_args(links_per_config, self_pairs)
        off, first_motion, num_motions = self._motion_args(len(h), links_per_config, motion_offsets, first_motion,
                                                           num_motions)
        return self.engine.env_collide_motions(self._env, h, t, links_per_config, tpl, off, req, first_motion,
                                               num_motions, witness=False)[0]

    def certify_motions(self, robot_manager, links_per_config, self_pairs, motion_offsets, sweep, request=None,
                        first_motion=0, num_motions=None):
        """A planner's continuous motion validation: the motions of collide_motions(), and sweep (one float64 per
        object of the robot manager): sweep[g * links_per_config + i] bounds the path length of every point of link i
        from configuration g to g + 1 (hpp-core's maximal velocity times the step; not finite and >= 0: the segment is
        not certified).  -> (first_invalid: per motion what collide_motions() returns; first_uncertified: per motion the
        first segment not certified free, -1 when all are; certified: per configuration 1 when the segment to the next
        sample of its motion is certified free).  A segment is certified when, at both its ends, every pair's collide()
        lower bound exceeds half its sweep (include/hppfcl_b200.h, hfb_env_certify_motions, states the rule and its
        guarantee).  Only motions [first_motion, first_motion + num_motions) are checked."""
        h, t, req = self._robot(robot_manager, request)
        tpl = self._template_args(links_per_config, self_pairs)
        off, first_motion, num_motions = self._motion_args(len(h), links_per_config, motion_offsets, first_motion,
                                                           num_motions)
        sw = np.asarray(sweep, dtype=np.float64).reshape(-1)
        if sw.shape[0] != len(h):
            raise ValueError("sweep: one bound per object of the robot manager")
        return self.engine.env_certify_motions(self._env, h, t, sw, links_per_config, tpl, off, req, first_motion,
                                               num_motions)[:3]

    def validate_motions(self, robot_model, q_from, q_to, self_pairs, *, initial_depth, max_depth, max_samples,
                         request=None, first_motion=0, num_motions=None):
        """A planner's progressive motion validation: motion m runs from q_from[m] to q_to[m] ((n_motions, nq) each)
        of the RobotModel, linear in q.  Each motion is cut into 2^initial_depth segments, certified as
        certify_motions() certifies them, and the uncertified segments are split again, down to 2^-max_depth of the
        motion, with at most max_samples samples per round (include/hppfcl_b200.h, hfb_env_validate_motions, states
        the rounds and their guarantee).  -> MotionValidation: per motion status (0 valid, 1 collides, 2 unresolved, -1
        outside the range), t_valid (the certified prefix is [0, t_valid]), t_collide (the earliest colliding sample
        found, -1 for none), the witness there (kind, first, second: link indices, or an environment index for kind 0;
        contacts), and the counts n_rounds, n_samples, n_env_candidates, n_self_candidates, n_unsupported."""
        request = request or CollisionRequest()
        if request.num_max_contacts == 0 and request.security_margin != -np.inf:
            raise ValueError("Invalid number of max contacts (current value is 0).")
        d0, d, cap = int(initial_depth), int(max_depth), int(max_samples)
        if d0 < 0 or d0 > d or d > 30 or cap < 2:
            raise ValueError("need 0 <= initial_depth <= max_depth <= 30 and max_samples >= 2")
        qf = np.asarray(q_from, dtype=np.float64)
        qt = np.asarray(q_to, dtype=np.float64)
        if qf.ndim != 2 or qf.shape[1] != robot_model.nq or qt.shape != qf.shape:
            raise ValueError("q_from, q_to: (n_motions, nq) each")
        n = qf.shape[0]
        num_motions = n - first_motion if num_motions is None else num_motions
        if first_motion < 0 or num_motions < 0 or first_motion + num_motions > n:
            raise ValueError("motion range past the end")
        tpl = self._template_args(robot_model.num_links, self_pairs)
        robot_model._sync()
        r = self.engine.env_validate_motions(self._env, robot_model._robot, qf, qt, tpl, d0, d, cap, request._pod,
                                             int(first_motion), int(num_motions))
        return MotionValidation(**r)

    @staticmethod
    def _motion_args(n_objects, links_per_config, motion_offsets, first_motion, num_motions):
        """the offsets and the motion range as the C ABI takes them; ones the C ABI refuses raise ValueError (the C++
        mirror throws std::invalid_argument)"""
        off = np.asarray(motion_offsets, dtype=np.int64).reshape(-1)
        lpc = int(links_per_config)
        if lpc < 1 or n_objects % lpc:
            raise ValueError("the robot manager's size is not a multiple of links_per_config")
        if off.shape[0] == 0 or off[0] != 0:
            raise ValueError("motion offsets must start at 0")
        if (np.diff(off) < 0).any():
            raise ValueError("motion offsets decrease")
        if off[-1] != n_objects // lpc:
            raise ValueError("motion offsets must end at the number of configurations")
        if (np.diff(off) > 0x7fffffff).any():
            raise ValueError("a motion has more than INT32_MAX samples")
        n_motions = off.shape[0] - 1
        num_motions = n_motions - first_motion if num_motions is None else num_motions
        if first_motion < 0 or num_motions < 0 or first_motion + num_motions > n_motions:
            raise ValueError("motion range past the end")
        return off.astype(np.uint32), int(first_motion), int(num_motions)

    @staticmethod
    def _template_args(links_per_config, self_pairs):
        """the template as the C ABI takes it; one the C ABI refuses raises ValueError (the C++ mirror throws
        std::invalid_argument)"""
        tpl = np.asarray(self_pairs, dtype=np.int64).reshape(-1, 2)
        lpc = int(links_per_config)
        key = np.sort(tpl, axis=1)
        if ((tpl < 0) | (tpl >= lpc)).any() or (tpl[:, 0] == tpl[:, 1]).any() or len(np.unique(key, axis=0)) != len(key):
            raise ValueError("self-pair template: a link index out of range, a link paired with itself or a pair listed "
                             "twice")
        return tpl.astype(np.uint32)

    @staticmethod
    def _distance_args(robot_manager, request, max_distance):
        if not max_distance >= 0:  # (the C++ mirror throws std::invalid_argument)
            raise ValueError("max_distance must be >= 0 or inf")
        if robot_manager._stale:
            robot_manager._refresh()
        return robot_manager._handles, robot_manager._tfs, (request or DistanceRequest())._pod

    def close(self):
        if getattr(self, "_env", None) is not None and getattr(self.engine, "h", None):
            self.engine.env_destroy(self._env)
        self._env = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class MotionValidation:
    """What ResidentEnvironment.validate_motions() returns: per motion status, t_valid, t_collide and the witness
    (kind, first, second, contacts), arrays of n_motions; the counts n_rounds, n_samples, n_env_candidates,
    n_self_candidates, n_unsupported, ints."""

    def __init__(self, **fields):
        self.__dict__.update(fields)


class RobotSamples:
    """Link poses of configurations from a RobotModel, in the form ResidentEnvironment's configuration and motion
    queries take a robot manager: object g * L + i is link i of configuration g.  tfs, handles: the objects; q: the
    configurations' joint values (n_configs x J) when asked; sweep: the sweep bounds certify_motions() takes, when
    asked; offsets: the motion offsets of sample_motions(), None for poses()."""
    _stale = False

    def __init__(self, tfs, handles, q=None, sweep=None, offsets=None):
        self._tfs, self._handles = tfs, handles
        self.q, self.sweep, self.offsets = q, sweep, offsets

    @property
    def tfs(self):
        return self._tfs

    @property
    def handles(self):
        return self._handles

    def size(self):
        return len(self._handles)


class RobotModel:
    """A kinematic tree of 1-DoF joints with a geometry per link, kept on the device (hfb_robot): Pinocchio's
    forwardKinematics + updateGeometryPlacements, batched.  joints: (parent, type, axis, placement) per joint, parent -1
    or an earlier joint, type JOINT_REVOLUTE or JOINT_PRISMATIC, placement a Transform3f (the joint frame in its
    parent's at q = 0); links: (joint, placement, geometry) per link, joint -1 for fixed to the world.  nq = the number
    of joints.  include/hppfcl_b200.h states the semantics and the sweep bounds.  close() (or leaving a `with` block)
    frees it."""

    def __init__(self, joints, links, device=0):
        self.scene = default_engine(device)
        self.engine = self.scene.engine
        parent = [j[0] for j in joints]
        types = [j[1] for j in joints]
        axis = np.array([j[2] for j in joints], dtype=np.float64).reshape(-1, 3)
        placement = _tf_array([j[3] for j in joints]) if joints else np.zeros(0, dtype=P.transform_dtype)
        link_joint = [l[0] for l in links]
        link_placement = _tf_array([l[1] for l in links]) if links else np.zeros(0, dtype=P.transform_dtype)
        self._geoms = [l[2] for l in links]
        handles = np.array([self.scene.handle(g) for g in self._geoms], dtype=np.uint32)
        self.scene.commit()
        self.nq, self.num_links = len(joints), len(links)
        self._robot = self.engine.robot_create(parent, types, axis, placement, link_joint, link_placement, handles)

    def _sync(self):
        """the links' geometry changed in place since: its records updated and committed, as a manager's setup() does"""
        for g in self._geoms:
            self.scene.handle(g)
        self.scene.commit()

    def poses(self, q):
        """q: (n_configs, nq) -> RobotSamples with the links' poses of every configuration"""
        self._sync()
        q = np.ascontiguousarray(q, dtype=np.float64).reshape(-1, self.nq)
        tfs, h = self.engine.robot_poses(self._robot, q)
        return RobotSamples(tfs, h, q=q)

    def sample_motions(self, q_from, q_to, offsets, sweep=True):
        """motion m from q_from[m] to q_to[m] ((n_motions, nq) each), offsets[m+1] - offsets[m] samples linear in q,
        end points included -> RobotSamples with the samples' poses, their q and (sweep=True) the sweep bounds"""
        self._sync()
        off = np.asarray(offsets, dtype=np.int64).reshape(-1)
        if off.shape[0] == 0 or off[0] != 0 or (np.diff(off) < 0).any() or (np.diff(off) > 0x7fffffff).any():
            raise ValueError("motion offsets must start at 0, not decrease, and hold motions of at most INT32_MAX samples")
        tfs, h, q, sw = self.engine.robot_sample_motions(self._robot, q_from, q_to, off.astype(np.uint32), q=True,
                                                         sweep=sweep)
        return RobotSamples(tfs, h, q=q, sweep=sw, offsets=off.astype(np.uint32))

    def close(self):
        if getattr(self, "_robot", None) is not None and getattr(self.engine, "h", None):
            self.engine.robot_destroy(self._robot)
        self._robot = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _unsupported(o1, o2, what, request=None):
    """the exception the reference throws for this pair (the record carries HFB_PATH_UNSUPPORTED)"""
    mesh = [o for o in (o1, o2) if o.node_type in _MESH_TYPES]
    shape = [o for o in (o1, o2) if o.node_type not in _MESH_TYPES]
    if len(mesh) == 1 and shape:
        if what == "Collision" and request is not None and request.security_margin < 0:
            # collision_func_matrix.cpp:109-112
            raise ValueError("Negative security margin are not handled yet for BVHModel")
        if getattr(shape[0], "getSweptSphereRadius", lambda: 0.0)() > 0:
            raise RuntimeError("Swept-sphere radius not yet supported.")  # geometric_shapes_utility.h:73-78
        if request is not None and request.gjk_initial_guess == P.BoundingVolumeGuess:
            raise RuntimeError("computeLocalAABB must have been called on the shapes before using "
                               "GJKInitialGuess::BoundingVolumeGuess.")  # narrowphase.h:368-377
    raise ValueError("%s function between node type %s and node type %s is not yet supported."
                     % (what, o1.node_type, o2.node_type))


def collide(o1, tf1, o2, tf2, request, result, device=0):
    """collide() of src/collision.cpp:69-130. Results accumulate: callers clear()."""
    if request.security_margin == -np.inf:  # :73-76
        result.clear()
        return 0
    if request.num_max_contacts == 0:
        raise ValueError("Invalid number of max contacts (current value is 0).")
    if result.isCollision() and request.num_max_contacts <= result.numContacts():  # isSatisfied
        return result.numContacts()
    bq = BatchQuery(device)
    scene = bq.scene
    h1, h2 = scene.handle(o1), scene.handle(o2)
    scene.commit()
    mesh = o1.node_type in _MESH_TYPES or o2.node_type in _MESH_TYPES
    more = []
    if mesh and request.num_max_contacts > 1:  # every contact of the pair, not only contacts[0]
        out, extra, counts = scene.engine.batch_collide_contacts([h1], _tf_array(tf1), [h2], _tf_array(tf2), request._pod,
                                                                 max_extra=int(request.num_max_contacts) - 1)
        more = [extra[0, k] for k in range(int(counts[0]) - 1)]
        gg, gh = [result.cached_gjk_guess], [result.cached_support_func_guess]
    else:
        out, gg, gh = scene.engine.batch_collide([h1], _tf_array(tf1), [h2], _tf_array(tf2), request._pod,
                                                 want_guess=True)
    rec = out[0]
    if P.status_path(rec["status"]) == P.PATH_UNSUPPORTED:
        _unsupported(o1, o2, "Collision", request)
    if rec["distance_lower_bound"] < result.distance_lower_bound:
        result.distance_lower_bound = float(rec["distance_lower_bound"])
        result.nearest_points = [rec["p1"].copy(), rec["p2"].copy()]
        result.normal = rec["normal"].copy()
    if rec["num_contacts"]:
        result.contacts.append(Contact(o1, o2, rec))
        for x in more:
            result.contacts.append(Contact(o1, o2, x))
    result.cached_gjk_guess = gg[0]
    result.cached_support_func_guess = gh[0]
    return result.numContacts() if rec["num_contacts"] else 0


def distance(o1, tf1, o2, tf2, request, result, device=0):
    """distance() of src/distance.cpp:60-109."""
    if result.min_distance <= 0:  # DistanceRequest::isSatisfied
        return result.min_distance
    bq = BatchQuery(device)
    scene = bq.scene
    h1, h2 = scene.handle(o1), scene.handle(o2)
    scene.commit()
    out, gg, gh = scene.engine.batch_distance([h1], _tf_array(tf1), [h2], _tf_array(tf2), request._pod,
                                              want_guess=True)
    rec = out[0]
    if P.status_path(rec["status"]) == P.PATH_UNSUPPORTED:
        _unsupported(o1, o2, "Distance", request)
    d = float(rec["min_distance"])
    closed = P.status_path(rec["status"]) == P.PATH_CLOSED_FORM
    if closed or result.min_distance > d:
        result.min_distance = d
        result.o1, result.o2 = o1, o2
        result.b1, result.b2 = int(rec["b1"]), int(rec["b2"])
        result.nearest_points = [rec["p1"].copy(), rec["p2"].copy()]
        result.normal = rec["normal"].copy()
    result.cached_gjk_guess = gg[0]
    result.cached_support_func_guess = gh[0]
    return d


class ComputeCollision:  # collision.h:79-117
    def __init__(self, o1, o2):
        self.o1, self.o2 = o1, o2

    def __call__(self, tf1, tf2, request, result):
        return collide(self.o1, tf1, self.o2, tf2, request, result)


class ComputeDistance:  # distance.h:74-112
    def __init__(self, o1, o2):
        self.o1, self.o2 = o1, o2

    def __call__(self, tf1, tf2, request, result):
        return distance(self.o1, tf1, self.o2, tf2, request, result)
