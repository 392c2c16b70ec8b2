"""CPU-only: the C-ABI library loads and exports every symbol include/*.h declares (no compute
calls), refuses to create a context without a GPU (no CPU fallback), and the host-side logic
(request PODs, sharding over ranks with gloo) behaves."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from tests.common import P, ROOT, hf, make_scenes
from hppfcl_b200 import workloads as W


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "hppfcl_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(hfb_[a-z_0-9]+)\s*\(", hdr)))


def test_library_exports_every_declared_symbol(built):
    L = hf.load_library()
    syms = declared_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(L, s), "missing export %s" % s
    assert b"sm_90a" in L.hfb_version()


def test_pod_layouts_match_header(built):
    # sizes the header documents; the defaults filled by the library equal the Python defaults
    L = hf.load_library()
    for cls, fn in ((P.DistanceRequestPOD, L.hfb_default_distance_request),
                    (P.CollisionRequestPOD, L.hfb_default_collision_request)):
        a, b = cls(), cls()
        C.memset(C.byref(b), 0xAB, C.sizeof(b))
        fn(C.byref(b))
        assert bytes(a) == bytes(b)
    assert C.sizeof(P.QueryRequest) == 64


def test_no_gpu_means_no_context(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(hf.EngineError) as e:
        hf.Engine(0)
    assert "no CUDA device" in str(e.value) and "no CPU fallback" in str(e.value)


def test_product_does_not_import_oracle():
    """the oracle is test infrastructure: nothing under hpp-fcl_b200/ may import, include, link or
    dlopen anything from oracle/ (comments may mention it)"""
    pkg = os.path.join(ROOT, "hpp-fcl_b200")
    pat = re.compile(r"(import\s+oracle|from\s+oracle|oracle_lib|liboracle|#include\s*[\"<][^\n]*oracle|oracle/)")
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(root, f)).read()
                assert not pat.search(txt), "%s references the oracle" % f


def test_shard_bounds():
    from hppfcl_b200.sharding import shard_bounds
    for n in (0, 1, 7, 8, 1000001):
        for world in (1, 2, 3, 8):
            b, per = shard_bounds(n, world)
            assert len(b) == world and b[0][0] == 0 and b[-1][1] == n
            assert all(b[i][1] == b[i + 1][0] for i in range(world - 1))
            assert all(hi - lo <= per for lo, hi in b)


_WORKER = r'''
import os, sys
sys.path.insert(0, %(root)r)
import numpy as np, torch, torch.distributed as dist
import hppfcl_b200 as hf
from hppfcl_b200 import _pod as P, workloads as W, sharding as S
from oracle import oracle_lib
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
n = 5001
w = W.config2_mixed_primitives(n, pool=256, seed=3)          # same seed on every rank: the batch
rng = np.random.default_rng(1)
pts = rng.normal(size=(12, 3))
shapes, cvx = S.broadcast_geometry(w["shapes"] if rank == 0 else None, [pts] if rank == 0 else None)
assert np.array_equal(shapes.view(np.uint8), w["shapes"].view(np.uint8)) and np.allclose(cvx[0], pts)
orc = oracle_lib.OracleScene(P)   # stand-in for the per-rank engine in this CPU test
orc.register_shapes(shapes)
def compute(lo, hi):
    return orc.batch_distance(w["h1"][lo:hi], w["tf1"][lo:hi], w["h2"][lo:hi], w["tf2"][lo:hi])
full = S.sharded_batch(compute, n, P.distance_result_dtype)
ref = orc.batch_distance(w["h1"], w["tf1"], w["h2"], w["tf2"])
assert full.shape == ref.shape
a, b = full.view(np.uint8).reshape(n, -1), ref.view(np.uint8).reshape(n, -1)
nan = np.isnan(ref["p1"][:, 0])
assert np.array_equal(a[~nan], b[~nan]) and np.array_equal(full["status"], ref["status"])
dist.barrier()
if rank == 0:
    print("SHARD-OK", world)
dist.destroy_process_group()
'''


def test_two_rank_gloo_sharding(tmp_path, built):
    """world_size 2 over gloo: geometry broadcast, pair-range sharding, result all-gather."""
    script = tmp_path / "worker.py"
    script.write_text(_WORKER % {"root": ROOT})
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29577", str(script)]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-3000:]
    assert "SHARD-OK 2" in res.stdout


def test_api_objects_without_gpu():
    """reference-shaped host objects (constructors, defaults) -- no compute"""
    b = hf.Box(6, 10, 2)
    assert np.allclose(b.halfSide, [3, 5, 1])                      # geometric_shapes.h:164-187
    c = hf.Capsule(2., 4.)
    assert c.radius == 2. and c.halfLength == 2.                   # :386-400
    r = hf.CollisionRequest()
    assert r.num_max_contacts == 1 and r.enable_contact == 1 and r.security_margin == 0 \
        and r.break_distance == 1e-3 and r.gjk_max_iterations == 128 and r.epa_max_iterations == 64 \
        and r.gjk_tolerance == 1e-6 and r.collision_distance_threshold == 1e-12   # collision_data.h:312-366
    d = hf.DistanceRequest()
    assert d.enable_signed_distance == 1 and d.rel_err == 0 and d.abs_err == 0       # :987-1030
    res = hf.CollisionResult()
    assert res.numContacts() == 0 and not res.isCollision() and res.distance_lower_bound == P.DBL_MAX
    dr = hf.DistanceResult()
    assert dr.min_distance == P.DBL_MAX and np.all(np.isnan(dr.normal)) and dr.b1 == -1
    t = hf.Transform3f.from_quat(1, 0, 0, 0, (1, 2, 3))
    assert np.allclose(t.transform([1, 1, 1]), [2, 3, 4])
    with pytest.raises(ValueError):
        hf.Sphere(1).setSweptSphereRadius(-1)
    cb = hf.CollisionCallBackCollect(10)                                             # default_broadphase_callbacks.cpp:95-120
    oa, ob = hf.CollisionObject(hf.Box(1, 1, 1)), hf.CollisionObject(hf.Sphere(1), hf.Transform3f(T=[1, 0, 0]))
    assert cb(oa, ob) is False and cb.numCollisionPairs() == 1 and cb.exist(oa, ob) and not cb.exist(ob, oa)
    cb.init()
    assert cb.numCollisionPairs() == 0
    assert hf.AABB([0, 0, 0], [1, 1, 1]).overlap(hf.AABB([1, 1, 1], [2, 2, 2]))     # closed intervals (AABB.h:111-118)
    assert not hf.AABB([0, 0, 0], [1, 1, 1]).overlap(hf.AABB([1.1, 0, 0], [2, 1, 1]))
    h = hf.Halfspace([0, 0, 2.0], 3.0)                                               # :887-890 + unitNormalTest
    assert np.allclose(h.n, [0, 0, 1]) and h.d == 1.5 and h.getNodeType() == P.GEOM_HALFSPACE
    assert h.signedDistance([0, 0, 2.0]) == 0.5
    pl = hf.Plane(0, 0, 0, 1.0)                                                      # zero normal -> (1, 0, 0), 0
    assert np.allclose(pl.n, [1, 0, 0]) and pl.d == 0 and pl.getNodeType() == P.GEOM_PLANE


def _update_scenario(dev, fresh):
    """register, query, change sizes / a hull / retire a handle, query again: `dev` after its updates must answer
    like `fresh` registered with the final geometry from scratch"""
    rng = np.random.default_rng(21)
    ALL = (P.GEOM_SPHERE, P.GEOM_CAPSULE, P.GEOM_BOX, P.GEOM_CYLINDER, P.GEOM_CONE, P.GEOM_ELLIPSOID)
    prim = W.random_primitive_shapes(rng, 40, ALL)
    hull_a, _ = W.ellipsoid_hull(rng, 20)
    hull_b = hull_a * np.array([1.5, 0.7, 1.1]) + 0.05
    cid = dev.register_convex(hull_a)
    rec = np.concatenate([prim, P.make_shapes([P.GEOM_CONVEX], [[0, 0, 0]], data=[cid])])
    h = dev.register_shapes(rec)
    dev.commit()
    n = 3000
    h1, h2 = h[rng.integers(0, len(h), n)], h[rng.integers(0, len(h), n)]
    tf1 = W.random_transforms(rng, n, (-1, -1, -1), (1, 1, 1))
    tf2 = W.random_transforms(rng, n, (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5))
    before = dev.batch_distance(h1, tf1, h2, tf2)
    # the changes
    rec2 = rec.copy()
    rec2["p"][:10] *= 1.7                      # ten shapes grow
    rec2[10] = P.make_shapes([P.GEOM_SPHERE], [[0.33, 0, 0]])[0]  # one changes its type
    rec2["ssr"][11] = 0.05
    dev.update_shapes(h[:12], rec2[:12])
    dev.update_convex(cid, hull_b)
    gone = h[12:14]
    if hasattr(dev, "release_shapes"):
        dev.release_shapes(gone)
    dev.commit()
    after = dev.batch_distance(h1, tf1, h2, tf2)
    fid = fresh.register_convex(hull_b, None) if type(fresh).__name__ == "OracleScene" else fresh.register_convex(hull_b)
    assert fid == cid
    assert np.array_equal(fresh.register_shapes(rec2), h)
    fresh.commit() if hasattr(fresh, "commit") else None
    kw = dict(nthreads=0) if type(fresh).__name__ == "OracleScene" else {}
    want = fresh.batch_distance(h1, tf1, h2, tf2, **kw)
    live = ~(np.isin(h1, gone) | np.isin(h2, gone)) if hasattr(dev, "release_shapes") else np.ones(n, dtype=bool)
    assert np.array_equal(after[live], want[live]) or all(
        np.array_equal(after[live][f], want[live][f], equal_nan=(after.dtype[f].kind == "f")) for f in after.dtype.names if f != "_pad")
    touched = np.isin(h1, h[:12]) | np.isin(h2, h[:12]) | (h1 == h[-1]) | (h2 == h[-1])
    assert (before["min_distance"][touched & live] != after["min_distance"][touched & live]).mean() > 0.5
    if hasattr(dev, "release_shapes"):
        assert np.all(P.status_path(after["status"][~live]) == P.PATH_UNSUPPORTED)
    # invalid updates leave everything as it was
    with pytest.raises(Exception):
        dev.update_convex(cid, hull_b[:5])
    with pytest.raises(Exception):
        dev.update_shapes([len(h) + 7], rec2[:1])


def test_geometry_updates_in_the_arena():
    """HostArena::set_shape / set_convex behind hfb_geom_update_* (shared by the library and tests/emu)"""
    from tests.common import EmuScene
    from oracle import oracle_lib
    _update_scenario(EmuScene(), oracle_lib.OracleScene(P))



def test_python_handle_cache_follows_in_place_changes():
    """api._Scene.handle: a geometry mutated in place keeps its handle and gets its record / vertices UPDATED (no
    stale answers for hulls and triangles, no handle leaked per change); only another vertex count re-registers"""
    from hppfcl_b200 import api

    class FakeEngine:
        def __init__(self):
            self.log, self.nshape, self.ncvx = [], 0, 0

        def register_convex(self, pts):
            self.log.append(("convex", len(pts)))
            self.ncvx += 1
            return self.ncvx - 1

        def register_shapes(self, rec):
            self.log.append(("shape", int(rec["type"][0])))
            self.nshape += 1
            return np.array([self.nshape - 1], dtype=np.uint32)

        def update_shapes(self, handles, rec):
            self.log.append(("update_shape", int(handles[0]), tuple(rec["p"][0].tolist()), float(rec["ssr"][0])))

        def update_convex(self, cid, pts):
            self.log.append(("update_convex", int(cid), len(pts)))

        def release_shapes(self, handles):
            self.log.append(("release", int(handles[0])))

        def commit(self):
            self.log.append(("commit",))

    e = FakeEngine()
    sc = api._Scene(e)
    box = hf.Box(2, 4, 6)
    h = sc.handle(box)
    assert sc.handle(box) == h and e.log == [("shape", P.GEOM_BOX)]
    box.halfSide[0] = 5.0  # in place
    assert sc.handle(box) == h and e.log[-1] == ("update_shape", h, (5.0, 2.0, 3.0), 0.0)
    box.setSweptSphereRadius(0.25)
    assert sc.handle(box) == h and e.log[-1][0] == "update_shape" and e.log[-1][3] == 0.25
    pts = np.random.default_rng(0).normal(size=(12, 3))
    cvx = hf.Convex(pts.copy())
    hc = sc.handle(cvx)
    n0 = len(e.log)
    assert sc.handle(cvx) == hc and len(e.log) == n0
    cvx.points[3] += 0.5  # a moved vertex: same handle, vertices updated
    assert sc.handle(cvx) == hc and ("update_convex", 0, 12) in e.log[n0:]
    assert sc.handle(cvx) == hc and e.log[-1][0] == "update_shape"
    n1 = len(e.log)
    assert sc.handle(cvx) == hc and len(e.log) == n1  # unchanged since: nothing to do
    tri = hf.TriangleP([0, 0, 0], [1, 0, 0], [0, 1, 0])
    ht = sc.handle(tri)
    tri.b[0] = 2.0
    assert sc.handle(tri) == ht and any(x[0] == "update_convex" and x[2] == 3 for x in e.log[n1:])
