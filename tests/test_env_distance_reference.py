"""The distance query's winners against the reference build (no GPU needed).  A sample of (A object, nearest B object)
pairs -- the robot workload and a scene of every kind of B object, each at a finite and an infinite cutoff -- is found
by brute force with the oracle under the contract of hfb_env_distance (include/hppfcl_b200.h).  The reference build's
distance() on those pairs must give the oracle's records bit for bit; tests/test_gpu_env_distance.py then checks that
the device finds the same winners with the same records."""
import gzip
import json
import os

import numpy as np

from tests import common
from tests.common import P, compare_distance, make_scenes
from oracle import oracle_lib
from hppfcl_b200 import workloads as W

# the reference's recorded outputs for the sample's call (HFB_RECORD_REFERENCE=<this file> records them), looked up
# with those of tests/golden/reference_outputs.json.gz where oracle/_ref is not built
REF_OUTPUTS = os.path.join(common.ROOT, "tests", "golden", "reference_outputs_env_distance.json.gz")
CUTOFFS = (0.05, np.inf)
# the fields the reference defines on every pair of the sample; a mesh's record also carries the oracle's own
# iteration counters and path byte (tests.common.ref_agrees)
FIELDS = ("min_distance", "p1", "p2", "normal", "b1", "b2")


def load_recorded():
    if os.path.exists(REF_OUTPUTS):
        common._load_recorded().update(json.load(gzip.open(REF_OUTPUTS, "rt")))


def contents_geometry(sc):
    """A and B of a scene with every kind of B object: duplicates, two spheres touching A's first sphere at exactly 0,
    a Halfspace floor, a Plane wall, an OBBRSS mesh, a plain OBB model (never eligible) and convex hulls"""
    rng = np.random.default_rng(5)
    sph, box, cap = (int(x) for x in sc.register_shapes(P.make_shapes([P.GEOM_SPHERE, P.GEOM_BOX, P.GEOM_CAPSULE],
                                                                         [[0.5, 0, 0], [0.2, 0.3, 0.1], [0.1, 0.2, 0]])))
    floor = sc.register_halfspaces(P.GEOM_HALFSPACE, [[0, 0, 1, -3.0]])[0]
    wall = sc.register_halfspaces(P.GEOM_PLANE, [[1, 0, 0, 6.0]])[0]
    verts, tris = W.sphere_mesh(0.4, 12, 6, noise=0.02, rng=rng)
    mesh = sc.register_shapes(P.make_shapes([P.BV_OBBRSS], [[0, 0, 0]], data=[sc.register_bvh(verts, tris)[0]]))[0]
    obb = sc.register_shapes(P.make_shapes([P.BV_OBB], [[0, 0, 0]], data=[sc.register_bvh_obb(verts, tris)[0]]))[0]
    hulls = []
    for _ in range(2):
        pts, ht = W.ellipsoid_hull(rng, 24, radii=(0.2, 0.3, 0.25))
        hulls.append(sc.register_shapes(P.make_shapes([P.GEOM_CONVEX], [[0, 0, 0]], data=[sc.register_convex(pts, ht)]))[0])
    hb = np.array([floor, sph, sph, sph, sph, wall, mesh, obb, hulls[0], hulls[1], box, box, cap], dtype=np.uint32)
    T = np.array([[0, 0, 0], [1.0, 0, 0], [0, 1.0, 0], [3, 3, 0], [3, 3, 0], [0, 0, 0], [0, -1.5, 0.5], [-0.2, -0.2, 0.1],
                  [2, -2, 0], [-2, 2, 1], [4, 4, 4], [4, 4, 4], [-3, -3, 0]], dtype=np.float64)
    ha = np.array([sph, box, cap, hulls[0], sph, box], dtype=np.uint32)
    TA = np.array([[0, 0, 0], [3, 3, 1], [-2.5, -3, 0.3], [1, -1.5, 0.8], [4, 4, 5.2], [-0.3, -0.2, 0.6]])
    return ha, W.identity_transforms(len(ha), T=TA), hb, W.identity_transforms(len(hb), T=T)


def oracle_nearest(orc, ha, tfa, hb, tfb, maxd):
    """-> (nearest, records of every pair) by the oracle's distance() on every pair and the header's argmin"""
    na, nb = len(ha), len(hb)
    i, j = np.repeat(np.arange(na), nb), np.tile(np.arange(nb), na)
    rec = orc.batch_distance(ha[i], tfa[i], hb[j], tfb[j], nthreads=0).reshape(na, nb)
    d = rec["min_distance"]
    elig = (d <= maxd) & (P.status_path(rec["status"]) != P.PATH_UNSUPPORTED)
    nearest = np.full(na, -1, dtype=np.int32)
    for a in range(na):
        c = np.flatnonzero(elig[a])
        if len(c):
            nearest[a] = c[d[a, c] == d[a, c].min()][0]
    return nearest, rec


def reference_sample(sc):
    """registers both scenes in every backend of sc (which holds the oracle) -> (scenes: [(ha, tfa, hb, tfb, {cutoff:
    oracle's nearest})], the sample's pairs as (h1, tf1, h2, tf2), the oracle's records of the sample).  The same
    wherever this runs: the oracle is the reference's restatement on the CPU."""
    w = W.robot_vs_environment(n_configs=4, n_env=300, room=1.2, seed=51)
    hs = w["register"](sc, oracle=True)
    robot = (hs[w["geom_a"]].astype(np.uint32), w["tf_a"], hs[w["geom_b"]].astype(np.uint32), w["tf_b"])
    contents = contents_geometry(sc)
    sc.commit()
    orc = sc.b["oracle"]
    scenes, pairs, recs = [], set(), []
    for ha, tfa, hb, tfb in (robot, contents):
        near = {}
        for maxd in CUTOFFS:
            n, rec = oracle_nearest(orc, ha, tfa, hb, tfb, maxd)
            near[maxd] = n
            for a in np.flatnonzero(n >= 0):
                if (len(scenes), a, n[a]) not in pairs:
                    pairs.add((len(scenes), a, n[a]))
                    recs.append((ha[a], tfa[a], hb[n[a]], tfb[n[a]], rec[a, n[a]]))
        scenes.append((ha, tfa, hb, tfb, near))
    h1 = np.array([r[0] for r in recs], dtype=np.uint32)
    tf1 = np.array([r[1] for r in recs], dtype=P.transform_dtype)
    h2 = np.array([r[2] for r in recs], dtype=np.uint32)
    tf2 = np.array([r[3] for r in recs], dtype=P.transform_dtype)
    return scenes, (h1, tf1, h2, tf2), np.array([r[4] for r in recs], dtype=P.distance_result_dtype)


def assert_fields(got, want, what):
    for f in FIELDS:
        x, y = got[f], want[f]
        ok = (x == y) | (np.isnan(x) & np.isnan(y)) if x.dtype.kind == "f" else x == y
        assert np.all(ok), "%s: field %s differs at rows %s" % (what, f, np.unique(np.nonzero(~ok)[0])[:8])


def test_winners_reference_sample():
    """the sample the GPU test compares the device's winners on: the reference build's distance() on every winning
    pair gives the oracle's record, and the sample holds found and not-found objects, ties and unbounded winners"""
    oracle_lib.build_ref()
    load_recorded()
    sc = make_scenes(ref=True, emu=False)
    scenes, args, orec = reference_sample(sc)
    rr = sc.b["ref"].batch_distance(*args)
    assert_fields(rr, orec, "winning pairs against the reference build")
    rows = P.status_path(orec["status"]) != P.PATH_BVH
    compare_distance(rr[rows], orec[rows], what="winning shape pairs against the reference build")
    assert len(orec) > 60
    robot, contents = scenes
    for near in (robot[4], contents[4]):
        assert (near[np.inf] >= 0).all() and (near[0.05] < 0).any() and (near[0.05] >= 0).any()
    # winners: the floor and other objects in the robot scene; the sphere touching at exactly 0 with the lower index
    # and the first of two duplicates in the other, never the OBB model
    assert 0 in robot[4][np.inf] and (robot[4][np.inf] >= 1).any()
    assert contents[4][np.inf][0] == 1 and 10 in contents[4][np.inf] and 11 not in contents[4][np.inf]
    assert 7 not in contents[4][np.inf]
