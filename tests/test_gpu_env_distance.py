"""Each robot object's nearest environment object (hfb_env_distance*).  The ground truth is brute force: distance() of
every (A object, B object) pair through hfb_batch_distance_objects over the table [A; B], then the argmin the header
defines -- eligible pairs (min_distance <= max_distance, not HFB_PATH_UNSUPPORTED), the smallest distance compared as
doubles, the lowest B index on ties.  nearest must match exactly, min_distance and the records byte for byte."""
import numpy as np
import pytest

from tests.common import P, hf
from tests.test_broadphase_sets import robot_scene
from hppfcl_b200 import workloads as W

pytestmark = pytest.mark.gpu

CUTOFFS = (0.0, 0.05, 0.3, np.inf)


def fresh(n):
    r = np.zeros(n, dtype=P.distance_result_dtype)
    r["min_distance"] = P.DBL_MAX
    for k in ("p1", "p2", "normal"):
        r[k] = np.nan
    r["b1"] = r["b2"] = -1
    return r


def brute(eng, ha, tfa, hb, tfb, maxd, req=None, first_a=0, num_a=None):
    """-> (nearest, min_distance, records, n_unsupported over all pairs of the range) by brute force"""
    na, nb = len(ha), len(hb)
    lo = min(first_a, na)
    hi = lo + min(na - lo if num_a is None else num_a, na - lo)
    nearest, rec = np.full(na, -1, dtype=np.int32), fresh(na)
    unsup = 0
    if hi > lo and nb:
        rows = np.arange(lo, hi, dtype=np.uint32)
        first = np.repeat(rows, nb)
        second = np.tile(np.arange(nb, dtype=np.uint32), len(rows)) + np.uint32(na)
        allr = eng.batch_distance_objects(np.concatenate([ha, hb]), np.concatenate([tfa, tfb]), first, second, req)
        allr = allr.reshape(len(rows), nb)
        d = allr["min_distance"]
        bad = P.status_path(allr["status"]) == P.PATH_UNSUPPORTED
        unsup = int(bad.sum())
        elig = (d <= maxd) & ~bad
        for k, i in enumerate(rows):
            c = np.flatnonzero(elig[k])
            if len(c):
                j = c[d[k, c] == d[k, c].min()][0]
                nearest[i], rec[i] = j, allr[k, j]
    return nearest, rec["min_distance"].copy(), rec, unsup


def assert_same(got, want):
    assert np.array_equal(got[0], want[0])
    assert got[1].tobytes() == want[1].tobytes()
    assert got[2].tobytes() == want[2].tobytes()


def test_robot_scene_matches_brute_force():
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = robot_scene(eng, n_configs=16, n_env=2000, room=1.4, seed=41)
    env = eng.env_create(hb, tfb)
    na, nb = len(ha), len(hb)
    for maxd in CUTOFFS:
        want = brute(eng, ha, tfa, hb, tfb, maxd)
        got = eng.env_distance(env, ha, tfa, max_distance=maxd)
        assert_same(got, want)
        if np.isfinite(maxd):
            assert got[3] < na * nb // 20
        if maxd == 0.3:
            assert (want[0] >= 0).sum() > na // 2 and (want[0] < 0).any()  # found and not found both occur
        if maxd == np.inf:
            assert (want[0] >= 0).all() and (want[1] > 0.05).any()
        # partial ranges add up to the whole; outside its range an object gets -1, DBL_MAX and a fresh record
        for lo, cnt in ((0, 37), (37, 1), (38, 0), (38, na)):
            r = eng.env_distance(env, ha, tfa, max_distance=maxd, first_a=lo, num_a=cnt)
            assert_same(r, brute(eng, ha, tfa, hb, tfb, maxd, first_a=lo, num_a=cnt))
        # clearance: the distances alone
        assert eng.env_distance(env, ha, tfa, max_distance=maxd, records=False)[1].tobytes() == want[1].tobytes()
    # A objects no longer in the table's first slots once a larger A came before: the same answers
    eng.env_distance(env, np.concatenate([ha, ha]), np.concatenate([tfa, tfa]))
    assert_same(eng.env_distance(env, ha, tfa, max_distance=0.3), brute(eng, ha, tfa, hb, tfb, 0.3))


def contents_scene(eng):
    """A: spheres and boxes near the origin; B: ties (duplicates, two spheres touching A's first sphere at exactly 0),
    a Halfspace floor, a Plane wall, an OBBRSS mesh, a plain OBB model and convex hulls"""
    rng = np.random.default_rng(5)
    prims = eng.register_shapes(P.make_shapes([P.GEOM_SPHERE, P.GEOM_BOX, P.GEOM_CAPSULE],
                                              [[0.5, 0, 0], [0.2, 0.3, 0.1], [0.1, 0.2, 0]]))
    floor = eng.register_halfspaces(P.GEOM_HALFSPACE, [[0, 0, 1, -3.0]])
    wall = eng.register_halfspaces(P.GEOM_PLANE, [[1, 0, 0, 6.0]])
    verts, tris = W.sphere_mesh(0.4, 12, 6, noise=0.02, rng=rng)
    nodes = hf.build_bvh_obbrss(verts, tris)
    mesh = eng.register_shapes(P.make_shapes([P.BV_OBBRSS], [[0, 0, 0]], data=[eng.register_bvh_obbrss(nodes, verts, tris)]))
    obb = eng.register_shapes(P.make_shapes([P.BV_OBB], [[0, 0, 0]], data=[eng.register_bvh_obb(nodes, verts, tris)]))
    hulls = []
    for _ in range(2):
        pts, _ = W.ellipsoid_hull(rng, 24, radii=(0.2, 0.3, 0.25))
        hulls.append(eng.register_shapes(P.make_shapes([P.GEOM_CONVEX], [[0, 0, 0]], data=[eng.register_convex(pts)]))[0])
    eng.commit()
    sph, box, cap = (int(x) for x in prims)
    hb = np.array([floor[0], sph, sph, sph, sph, wall[0], mesh[0], obb[0], hulls[0], hulls[1], box, box, cap], dtype=np.uint32)
    T = np.array([[0, 0, 0], [1.0, 0, 0], [0, 1.0, 0], [3, 3, 0], [3, 3, 0], [0, 0, 0], [0, -1.5, 0.5], [-0.2, -0.2, 0.1],
                  [2, -2, 0], [-2, 2, 1], [4, 4, 4], [4, 4, 4], [-3, -3, 0]], dtype=np.float64)
    tfb = W.identity_transforms(len(hb), T=T)
    ha = np.array([sph, box, cap, hulls[0], sph, box], dtype=np.uint32)
    TA = np.array([[0, 0, 0], [3, 3, 1], [-2.5, -3, 0.3], [1, -1.5, 0.8], [4, 4, 5.2], [-0.3, -0.2, 0.6]])
    tfa = W.identity_transforms(len(ha), T=TA)
    return ha, tfa, hb, tfb


def test_b_contents_ties_unbounded_meshes_hulls():
    eng = hf.Engine(0)
    ha, tfa, hb, tfb = contents_scene(eng)
    env = eng.env_create(hb, tfb)
    for maxd in CUTOFFS + (2.5,):
        want = brute(eng, ha, tfa, hb, tfb, maxd)
        got = eng.env_distance(env, ha, tfa, max_distance=maxd)
        assert_same(got, want)
        assert got[4] <= want[3]  # (the unsupported pairs among the candidates)
        assert 7 not in got[0]  # the plain OBB model is never nearest
    got = eng.env_distance(env, ha, tfa)
    assert got[0][0] == 1 and got[1][0] == 0.0  # the two spheres touching at exactly 0: the lower index wins
    assert got[4] >= 1  # distance() to the OBB model is unsupported, and the box next to it is a candidate
    assert got[0][4] in (10, 11) and got[0][4] == 10  # duplicates: the first one


def test_edges_far_points_displaced_nonfinite_empty():
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = robot_scene(eng, n_configs=4, n_env=600, room=1.2, seed=43, plane=False)
    env = eng.env_create(hb[1:], tfb[1:])  # no floor: nothing unbounded
    # a robot far outside B's bounds: the rounds stop once its box reaches all of B
    far = tfa.copy()
    far["T"] += [1e4, -3e3, 5e3]
    for maxd in (0.3, np.inf):
        assert_same(eng.env_distance(env, ha, far, max_distance=maxd), brute(eng, ha, far, hb[1:], tfb[1:], maxd))
    # NaN and infinite poses terminate, with what brute force says: such an object runs against all of B in one round,
    # and a pair is eligible only when distance() itself returns a distance within the cutoff
    bad = tfa.copy()
    bad["T"][3] = np.nan
    bad["R"][5, 0] = np.nan
    bad["T"][7, 1] = np.inf
    for maxd in (0.05, np.inf):
        got = eng.env_distance(env, ha, bad, max_distance=maxd)
        assert_same(got, brute(eng, ha, bad, hb[1:], tfb[1:], maxd))
        assert not np.isnan(got[1]).any()
    # scenes displaced by 1e100: A and B together
    for shift in (1e6, 1e100):
        ta, tb = tfa.copy(), tfb.copy()
        ta["T"] += shift
        tb["T"] += shift
        e2 = eng.env_create(hb[1:], tb[1:])
        for maxd in (0.05, np.inf):
            assert_same(eng.env_distance(e2, ha, ta, max_distance=maxd), brute(eng, ha, ta, hb[1:], tb[1:], maxd))
        eng.env_destroy(e2)
    # B of points only (spheres of radius 0)
    pts = eng.register_shapes(P.make_shapes([P.GEOM_SPHERE], [[0, 0, 0]]))
    eng.commit()
    rng = np.random.default_rng(2)
    hp = np.full(300, pts[0], dtype=np.uint32)
    tp = W.identity_transforms(300, T=rng.uniform(-1.5, 1.5, (300, 3)))
    e3 = eng.env_create(hp, tp)
    for maxd in CUTOFFS:
        assert_same(eng.env_distance(e3, ha, tfa, max_distance=maxd), brute(eng, ha, tfa, hp, tp, maxd))
    # an empty env, and no A objects
    e4 = eng.env_create(hb[:0], tfb[:0])
    got = eng.env_distance(e4, ha, tfa)
    assert (got[0] == -1).all() and got[2].tobytes() == fresh(len(ha)).tobytes() and got[3:] == (0, 0)
    got = eng.env_distance(env, ha[:0], tfa[:0])
    assert len(got[0]) == 0 and got[3:] == (0, 0)


def test_updates_and_lifetime():
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = robot_scene(eng, n_configs=8, n_env=1500, room=1.3, seed=47)
    env = eng.env_create(hb, tfb)
    rng = np.random.default_rng(9)
    idx = rng.choice(len(hb), 300, replace=False).astype(np.uint32)
    t2 = tfb.copy()
    t2["T"][idx] += rng.uniform(-0.4, 0.4, (len(idx), 3))
    eng.env_update(env, idx, t2[idx])
    for maxd in (0.05, np.inf):
        assert_same(eng.env_distance(env, ha, tfa, max_distance=maxd), brute(eng, ha, tfa, hb, t2, maxd))
    eng.release_shapes([hb[3]])
    eng.commit()
    with pytest.raises(hf.EngineError, match="invalid argument"):
        eng.env_distance(env, ha, tfa)
    env2 = eng.env_create(ha[:10], tfa[:10])
    eng.clear_geometry()
    w["register"](eng)
    eng.commit()
    for e in (env, env2):
        with pytest.raises(hf.EngineError, match="invalid argument"):
            eng.env_distance(e, ha, tfa)
        eng.env_destroy(e)


def test_winners_equal_the_reference():
    """the sample of tests/test_env_distance_reference.py: the device finds the oracle's winners at both cutoffs, and
    their records equal the reference build's (its recorded outputs where it is not built here)"""
    from tests.common import make_scenes
    from tests.test_env_distance_reference import assert_fields, load_recorded, reference_sample
    load_recorded()
    sc = make_scenes(gpu=True, emu=False, ref=True)
    eng = sc.b["gpu"]
    scenes, args, orec = reference_sample(sc)
    rr = sc.b["ref"].batch_distance(*args)
    at = {}  # (scene, A index, B index) -> row of the sample
    for s, (ha, tfa, hb, tfb, near) in enumerate(scenes):
        for n in near.values():
            for a in np.flatnonzero(n >= 0):
                at.setdefault((s, int(a), int(n[a])), len(at))
    assert len(at) == len(rr)
    for s, (ha, tfa, hb, tfb, near) in enumerate(scenes):
        env = eng.env_create(hb, tfb)
        for maxd, n in near.items():
            got = eng.env_distance(env, ha, tfa, max_distance=maxd)
            assert np.array_equal(got[0], n)
            rows = [at[(s, int(a), int(n[a]))] for a in np.flatnonzero(n >= 0)]
            mine = got[2][n >= 0]
            assert_fields(mine, rr[rows], "device winners against the reference build")
            assert mine.tobytes() == orec[rows].tobytes()  # (the oracle's whole records)
        eng.env_destroy(env)


def dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1)).cuda()


def test_device_form_and_unsynchronised_host_calls():
    """the device form equals the host form; a device call on a side stream followed by host env and scene calls on the
    same context, with no synchronisation in between: both results as each call alone gives them"""
    import torch
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = robot_scene(eng, n_configs=16, n_env=2000, room=1.4, seed=41)
    env = eng.env_create(hb, tfb)
    n = len(ha)
    t_other = tfa.copy()
    t_other["T"] += 0.2
    d_h, d_t = dev(ha), dev(tfa)
    d_near = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_min = torch.zeros(n, dtype=torch.float64, device="cuda")
    d_rec = torch.zeros(n * P.distance_result_dtype.itemsize, dtype=torch.uint8, device="cuda")
    d_cnt = torch.zeros(2, dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()

    def run(maxd, first_a=0, num_a=None):
        eng.env_distance_device(env, n, d_h.data_ptr(), d_t.data_ptr(), d_near.data_ptr(), d_min.data_ptr(), d_rec.data_ptr(),
                                d_cnt.data_ptr(), d_cnt.data_ptr() + 4, max_distance=maxd, stream=side.cuda_stream,
                                first_a=first_a, num_a=num_a)

    def fetch():
        side.synchronize()
        rec = d_rec.cpu().numpy().view(P.distance_result_dtype)
        c = d_cnt.cpu().numpy()
        return d_near.cpu().numpy(), d_min.cpu().numpy(), rec, int(c[0]), int(c[1])

    torch.cuda.synchronize()
    for maxd, lo, cnt in ((0.05, 0, None), (np.inf, 0, None), (0.3, 40, 100)):
        want = eng.env_distance(env, ha, tfa, max_distance=maxd, first_a=lo, num_a=cnt)
        run(maxd, lo, cnt)
        got = fetch()
        assert_same(got, want)
        assert got[3:] == want[3:]
    want_dev = eng.env_distance(env, ha, tfa, max_distance=0.3)
    want_env = eng.env_distance(env, ha, t_other, max_distance=np.inf)
    want_col = eng.env_collide(env, ha, t_other, capacity=1 << 20)
    want_sets = eng.scene_collide_sets(ha, t_other, hb, tfb, capacity=1 << 20)
    for host_call, want in ((lambda: eng.env_distance(env, ha, t_other, max_distance=np.inf), want_env),
                            (lambda: eng.env_collide(env, ha, t_other, capacity=1 << 20), want_col),
                            (lambda: eng.scene_collide_sets(ha, t_other, hb, tfb, capacity=1 << 20), want_sets)):
        run(0.3)
        got = host_call()  # no synchronisation in between
        if want is want_env:
            assert_same(got, want)
            assert got[3:] == want[3:]
        else:
            assert got[3:5] == want[3:5] and sorted(zip(got[0].tolist(), got[1].tolist())) == sorted(zip(want[0].tolist(), want[1].tolist()))
        g = fetch()
        assert_same(g, want_dev)
        assert g[3:] == want_dev[3:]


def test_python_and_cpp_mirror_scene():
    """ResidentEnvironment.distance / clearance on managers: the brute-force answer over the managers' tables"""
    rng = np.random.default_rng(23)

    def pose(lo=0, hi=4):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        return hf.Transform3f.from_quat(*q, T=rng.uniform(lo, hi, 3))

    geoms = [hf.Box(0.3, 0.2, 0.4), hf.Sphere(0.15), hf.Capsule(0.1, 0.3)]
    robot = [hf.CollisionObject(geoms[i % 3], pose()) for i in range(60)]
    env_objs = [hf.CollisionObject(hf.Halfspace(np.array([0.0, 0, 1]), -0.5))]
    env_objs += [hf.CollisionObject(geoms[i % 3], pose()) for i in range(400)]
    mr, me = hf.DynamicAABBTreeCollisionManager(), hf.DynamicAABBTreeCollisionManager()
    mr.registerObjects(robot)
    me.registerObjects(env_objs)
    mr.setup()
    me.setup()
    with hf.ResidentEnvironment(me) as re:
        eng = re.engine
        for maxd in (0.2, np.inf):
            nearest, dist, rec = re.distance(mr, max_distance=maxd)
            want = brute(eng, mr._handles, mr._tfs, me._handles, me._tfs, maxd)
            assert_same((nearest, dist, rec), want)
            assert re.clearance(mr, maxd).tobytes() == want[1].tobytes()
        for bad in (np.nan, -0.1):
            with pytest.raises(ValueError):
                re.distance(mr, max_distance=bad)
