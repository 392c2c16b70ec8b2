"""Broadphase between two object sets: BroadPhaseCollisionManager::collide(other_manager, callback) and collide(obj,
callback) (broadphase_collision_manager.h:94-118).  The reference's managers do not build here (boost::function), so the
check is the definition: every (i in A, j in B) whose boxes overlap (AABB::overlap, closed intervals), brute force."""
import ctypes as C

import numpy as np
import pytest

from tests.common import P, compare_distance, hf
from hppfcl_b200 import workloads as W

BIG = np.finfo(np.float64).max


def brute_cross(ba, bb):
    """the cross set; boxless markers (min = DBL_MAX, max = -DBL_MAX) take no part"""
    ov = np.all((ba[:, None, :3] <= bb[None, :, 3:]) & (ba[:, None, 3:] >= bb[None, :, :3]), axis=2)
    ov &= ~((ba[:, 0] == BIG) & (ba[:, 3] == -BIG))[:, None]
    ov &= ~((bb[:, 0] == BIG) & (bb[:, 3] == -BIG))[None, :]
    i, j = np.nonzero(ov)
    return set(zip(i.tolist(), j.tolist()))


def boxes(rng, n, scale, small=0.05, big=0.0, huge_frac=0.0, huge=10.0):
    c = scale * (2 * rng.random((n, 3)) - 1)
    e = small + big * rng.random((n, 3))
    e[rng.random(n) < huge_frac] = huge
    return np.concatenate([c - e, c + e], axis=1)


def check(ba, bb):
    f, s = hf.broadphase_cross_pairs(ba, bb)
    got = set(zip(f.tolist(), s.tolist()))
    assert len(got) == len(f)
    assert got == brute_cross(ba, bb)
    return got


@pytest.mark.parametrize("na,nb,seed", [(300, 2000, 1), (2000, 300, 2), (1000, 1000, 3)])
def test_host_cross_finder_random_sets(na, nb, seed):
    rng = np.random.default_rng(seed)
    # sizes: A large against small B, B spread over several octaves, and a few huge boxes in B
    check(boxes(rng, na, 5.0, 0.1, 0.6), boxes(rng, nb, 5.0, 0.02, 0.1))
    check(boxes(rng, na, 5.0, 0.01, 0.02), boxes(rng, nb, 5.0, 0.005, 1.0))
    got = check(boxes(rng, na, 20.0, 0.2, 0.3), boxes(rng, nb, 20.0, 0.1, 0.2, huge_frac=0.01, huge=8.0))
    assert got


def test_touching_boxes_overlap():
    a = np.array([[0, 0, 0, 1, 1, 1.0], [5, 5, 5, 6, 6, 6]])
    b = np.array([[1, 0, 0, 2, 1, 1.0], [1, 1, 1, 2, 2, 2], [1 + 1e-12, 0, 0, 2, 1, 1], [-1, -1, -1, 0, 0, 0],
                  [6, 6, 6, 6, 6, 6]])
    assert check(a, b) == {(0, 0), (0, 1), (0, 3), (1, 4)}
    rng = np.random.default_rng(9)  # touching on a lattice: every face, edge and corner contact
    g = np.stack(np.meshgrid(*[np.arange(6.0)] * 3, indexing="ij"), -1).reshape(-1, 3)
    check(np.concatenate([g, g + 1], 1)[rng.permutation(len(g))[:80]], np.concatenate([g + 1, g + 2], 1))


def test_huge_boxes_in_b():
    """a few walls and tables among thousands of 5 cm objects: they go on the oversize list"""
    rng = np.random.default_rng(4)
    bb = boxes(rng, 5000, 10.0, 0.02, 0.03)
    bb[:10] = boxes(rng, 10, 10.0, 2.0, 8.0)
    check(boxes(rng, 2000, 10.0, 0.05, 0.2), bb)


def test_unbounded_objects_and_boxless_markers():
    rng = np.random.default_rng(5)
    floor = [-BIG, -BIG, -BIG, BIG, BIG, 0.0]
    tilted = [-np.inf, -np.inf, -np.inf, np.inf, np.inf, np.inf]
    plane = [2.0, -BIG, -BIG, 2.0, BIG, BIG]
    none = [BIG, BIG, BIG, -BIG, -BIG, -BIG]
    ba0, bb0 = boxes(rng, 800, 4.0, 0.1, 0.3), boxes(rng, 1500, 4.0, 0.05, 0.1)
    for where in ("a", "b", "both"):
        ba, bb = ba0.copy(), bb0.copy()
        if where in ("a", "both"):
            ba[[3, 100, 400, 799]] = [floor, tilted, plane, none]
        if where in ("b", "both"):
            bb[[0, 7, 1499, 600]] = [floor, tilted, plane, none]
        got = check(ba, bb)
        if where == "both":
            assert (100, 7) in got and (3, 0) in got and (400, 1499) in got
            assert not any(a == 799 or b == 600 for a, b in got)


def point_sets(rng):
    """B mostly (or only) point boxes with distinct centres -- zero-size shapes, a point cloud: the 95th percentile of
    B's extents is zero, the cell must still be a positive size that keeps the grid within bounds"""
    a = boxes(rng, 400, 1.0, 0.01, 0.05)
    p = rng.random((3000, 3))
    mostly = np.concatenate([p, p], axis=1)
    mostly[:100] = boxes(rng, 100, 1.0, 0.002, 0.01)
    only = np.concatenate([p[:100], p[:100]], axis=1)
    far = np.concatenate([p * 1e6, p * 1e6], axis=1)  # points over a huge span
    return a, [mostly, only, far]


def test_point_boxes_in_b():
    rng = np.random.default_rng(12)
    a, bs = point_sets(rng)
    for bb in bs:
        check(a, bb)
        check(bb, a)  # and as A
    a2 = np.concatenate([bs[1][:, :3] - 1e-3, bs[1][:, 3:] + 1e-3], axis=1)
    assert len(check(a2, bs[1])) >= 100  # every point against the small box around it


@pytest.mark.parametrize("na,nb", [(0, 0), (0, 5), (5, 0), (1, 1), (1, 50), (50, 1)])
def test_empty_and_single_sets(na, nb):
    rng = np.random.default_rng(na * 100 + nb)
    check(boxes(rng, na, 1.0, 0.3, 0.3).reshape(-1, 6), boxes(rng, nb, 1.0, 0.3, 0.3).reshape(-1, 6))


def test_capacity_below_the_count():
    rng = np.random.default_rng(6)
    ba, bb = boxes(rng, 500, 3.0, 0.1, 0.3), boxes(rng, 800, 3.0, 0.05, 0.2)
    want = brute_cross(ba, bb)
    assert len(want) > 20
    L = hf.load_library()
    first, second = np.zeros(7, np.uint32), np.zeros(7, np.uint32)
    cnt = C.c_size_t(0)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    assert L.hfb_broadphase_cross_pairs(500, ptr(ba), 800, ptr(bb), ptr(first), ptr(second), 7, C.byref(cnt)) == 0
    assert cnt.value == len(want)
    assert set(zip(first.tolist(), second.tolist())) <= want
    f, s = hf.broadphase_cross_pairs(ba, bb, capacity=7)
    assert len(f) == 7 and set(zip(f.tolist(), s.tolist())) <= want


def test_cross_pairs_reject_null_buffers():
    L = hf.load_library()
    bb = np.zeros((4, 6))
    f, s = np.zeros(8, np.uint32), np.zeros(8, np.uint32)
    cnt = C.c_size_t(0)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    fn = L.hfb_broadphase_cross_pairs
    assert fn(4, None, 4, ptr(bb), ptr(f), ptr(s), 8, C.byref(cnt)) == 1
    assert fn(4, ptr(bb), 4, None, ptr(f), ptr(s), 8, C.byref(cnt)) == 1
    assert fn(4, ptr(bb), 4, ptr(bb), None, ptr(s), 8, C.byref(cnt)) == 1
    assert fn(4, ptr(bb), 4, ptr(bb), ptr(f), None, 8, C.byref(cnt)) == 1
    assert fn(4, ptr(bb), 4, ptr(bb), ptr(f), ptr(s), 8, None) == 1
    assert fn(0, None, 0, None, None, None, 0, C.byref(cnt)) == 0 and cnt.value == 0
    assert fn(4, ptr(bb), 4, ptr(bb), None, None, 0, C.byref(cnt)) == 0 and cnt.value == 16  # counted, none stored


def test_robot_workload_has_the_intended_density():
    """the benchmark's robot-vs-environment scene: about 10^6 candidates, every kind of object of B among them"""
    from tests.common import EmuScene
    w = W.robot_vs_environment()
    emu = EmuScene()
    hs = w["register"](emu)
    ba, bb = emu.scene_aabbs(hs[w["geom_a"]], w["tf_a"]), emu.scene_aabbs(hs[w["geom_b"]], w["tf_b"])
    f, s = hf.broadphase_cross_pairs(ba, bb)
    assert 7e5 < len(f) < 1.5e6
    gb = w["geom_b"][s]
    assert (gb == w["geom_b"][0]).sum() > 100 and (gb == w["geom_b"][1]).sum() > 100  # the floor and the meshes
    assert len(ba) == 1024 * 16 and len(bb) == 100_000


# ---------------------------------------------------------------------------------------------------------- GPU
def robot_scene(eng, n_configs=96, n_env=12_000, room=2.2, seed=21, plane=True):
    """a small robot-vs-environment scene with a Plane wall added to B; -> (ha, tfa, hb, tfb, handles)"""
    w = W.robot_vs_environment(n_configs=n_configs, n_env=n_env, room=room, seed=seed)
    hs = w["register"](eng)
    ha, tfa = hs[w["geom_a"]].astype(np.uint32), w["tf_a"]
    hb, tfb = hs[w["geom_b"]].astype(np.uint32), w["tf_b"].copy()
    if plane:
        wall = eng.register_halfspaces(P.GEOM_PLANE, [[1, 0, 0, 0.5 * room]])
        hb[-1] = wall[0]
        tfb[-1] = W.identity_transforms(1)[0]
    eng.commit()
    return w, ha, tfa, hb, tfb


@pytest.mark.gpu
def test_device_cross_finder():
    import torch
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = robot_scene(eng)
    ba, bb = eng.scene_aabbs(ha, tfa), eng.scene_aabbs(hb, tfb)
    f, s = hf.broadphase_cross_pairs(ba, bb)
    want = set(zip(f.tolist(), s.tolist()))
    assert len(want) == len(f) and len(want) > 20_000
    assert want == brute_cross(ba, bb[:3000]) | {p for p in want if p[1] >= 3000}  # brute force on a prefix of B
    assert any(p[1] == 0 for p in want) and any(p[1] == len(hb) - 1 for p in want)  # the floor and the wall

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()

    stream = torch.cuda.current_stream().cuda_stream
    d_a, d_b = dev(ba), dev(bb)
    cap = len(want) + 1000
    d_f = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_s = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int32, device="cuda")
    for _ in range(2):  # twice: the scratch is reused
        eng.broadphase_cross_pairs_device(len(ba), d_a.data_ptr(), len(bb), d_b.data_ptr(), d_f.data_ptr(), d_s.data_ptr(),
                                          cap, d_n.data_ptr(), stream)
        torch.cuda.synchronize()
        k = int(d_n.item())
        got = set(zip(d_f[:k].cpu().numpy().tolist(), d_s[:k].cpu().numpy().tolist()))
        assert k == len(want) and got == want
    eng.broadphase_cross_pairs_device(len(ba), d_a.data_ptr(), len(bb), d_b.data_ptr(), d_f.data_ptr(), d_s.data_ptr(),
                                      100, d_n.data_ptr(), stream)
    torch.cuda.synchronize()
    assert int(d_n.item()) == len(want)
    assert set(zip(d_f[:100].cpu().numpy().tolist(), d_s[:100].cpu().numpy().tolist())) <= want
    got = set()
    n = len(ba)
    for lo, cnt in ((0, 500), (500, 333), (833, n)):
        eng.broadphase_cross_pairs_device(n, d_a.data_ptr(), len(bb), d_b.data_ptr(), d_f.data_ptr(), d_s.data_ptr(), cap,
                                          d_n.data_ptr(), stream, first_a=lo, num_a=cnt)
        torch.cuda.synchronize()
        kk = int(d_n.item())
        part = set(zip(d_f[:kk].cpu().numpy().tolist(), d_s[:kk].cpu().numpy().tolist()))
        assert len(part) == kk and all(lo <= a < lo + cnt for a, _ in part) and not (part & got)
        got |= part
    assert got == want
    # an A box that spans the whole grid, an unbounded one and a boxless one: the brute-force paths
    ba2 = ba.copy()
    ba2[0] = [-1.0, -1.0, -1.0, 9.0, 9.0, 3.0]
    ba2[1] = [-BIG, -BIG, -BIG, BIG, BIG, 0.05]
    ba2[2] = [BIG, BIG, BIG, -BIG, -BIG, -BIG]
    f2, s2 = hf.broadphase_cross_pairs(ba2, bb)
    want2 = set(zip(f2.tolist(), s2.tolist()))
    d_a2 = dev(ba2)
    cap = len(want2) + 1000
    d_f = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_s = torch.empty(cap, dtype=torch.int32, device="cuda")
    eng.broadphase_cross_pairs_device(n, d_a2.data_ptr(), len(bb), d_b.data_ptr(), d_f.data_ptr(), d_s.data_ptr(), cap,
                                      d_n.data_ptr(), stream)
    torch.cuda.synchronize()
    k = int(d_n.item())
    assert k == len(want2) and set(zip(d_f[:k].cpu().numpy().tolist(), d_s[:k].cpu().numpy().tolist())) == want2
    assert sum(1 for a, _ in want2 if a == 0) > 5000
    # B made mostly or only of point boxes: the device grid equals the host one (cell from the first non-zero bin)
    pa, pbs = point_sets(np.random.default_rng(12))
    pa[:100] = np.concatenate([pbs[1][:, :3] - 1e-3, pbs[1][:, 3:] + 1e-3], axis=1)
    for pb in pbs:
        f3, s3 = hf.broadphase_cross_pairs(pa, pb)
        want3 = set(zip(f3.tolist(), s3.tolist()))
        d_pa, d_pb = dev(pa), dev(pb)
        eng.broadphase_cross_pairs_device(len(pa), d_pa.data_ptr(), len(pb), d_pb.data_ptr(), d_f.data_ptr(), d_s.data_ptr(),
                                          cap, d_n.data_ptr(), stream)
        torch.cuda.synchronize()
        k = int(d_n.item())
        assert k == len(want3) <= cap and (pb is not pbs[1] or len(want3) >= 100)
        assert set(zip(d_f[:k].cpu().numpy().tolist(), d_s[:k].cpu().numpy().tolist())) == want3


@pytest.mark.gpu
def test_scene_collide_sets():
    from oracle import oracle_lib
    eng, orc = hf.Engine(0), oracle_lib.OracleScene(P)
    w, ha, tfa, hb, tfb = robot_scene(eng)
    ho = w["register"](orc, oracle=True)  # the same geometry in the same order: the same handles
    assert np.array_equal(ho[w["geom_a"]], ha) and np.array_equal(ho[w["geom_b"][:-1]], hb[:-1])
    assert orc.register_halfspaces(P.GEOM_PLANE, [[1, 0, 0, 0.5 * w["room"]]])[0] == hb[-1]
    pf, ps = hf.broadphase_cross_pairs(eng.scene_aabbs(ha, tfa), eng.scene_aabbs(hb, tfb))
    f, s, rec, ncand, nhit = eng.scene_collide_sets(ha, tfa, hb, tfb, capacity=len(pf) + 10)
    assert ncand == len(pf) > 20_000
    rows = eng.batch_collide(ha[pf], tfa[pf], hb[ps], tfb[ps])
    hit = rows["num_contacts"] > 0
    assert nhit == int(hit.sum()) == len(f) and nhit > 500
    want = {(int(a), int(b)): rows[i].tobytes() for i, (a, b) in enumerate(zip(pf, ps)) if hit[i]}
    got = {(int(a), int(b)): rec[i].tobytes() for i, (a, b) in enumerate(zip(f, s))}
    assert got == want
    # a sample against the oracle in the same operand order, (shape, mesh) and (mesh, shape) pairs included
    is_mesh_b = hb[ps] == hb[1]
    rng = np.random.default_rng(3)
    k = np.concatenate([np.nonzero(is_mesh_b)[0][:200], rng.choice(len(pf), 3000, replace=False)])
    ro = orc.batch_collide(ha[pf[k]], tfa[pf[k]], hb[ps[k]], tfb[ps[k]], nthreads=0)
    compare_distance(ro, rows[k], what="(link, environment) sample")  # bit for bit; NaNs of either sign are equal
    assert is_mesh_b[k].sum() > 50
    hm = np.array([hb[1]], dtype=np.uint32)  # (mesh, shape): a mesh of B as o1 against robot links
    rg = eng.batch_collide(np.repeat(hm, 200), tfb[np.full(200, 1)], ha[:200], tfa[:200])
    rr = orc.batch_collide(np.repeat(hm, 200), tfb[np.full(200, 1)], ha[:200], tfa[:200], nthreads=0)
    compare_distance(rr, rg, what="(mesh, link) pairs")
    # ranges of A add up
    n = len(ha)
    tot_c = tot_h = 0
    for lo, cnt in ((0, 700), (700, n)):
        f2, s2, _, c2, h2 = eng.scene_collide_sets(ha, tfa, hb, tfb, first_a=lo, num_a=cnt)
        assert ((f2 >= lo) & (f2 < lo + cnt)).all()
        tot_c += c2
        tot_h += h2
    assert tot_c == ncand and tot_h == nhit
    # capacity below the count, -inf margin, num_max_contacts == 0, empty sets
    f3, _, _, _, h3 = eng.scene_collide_sets(ha, tfa, hb, tfb, capacity=50)
    assert h3 == nhit and len(f3) == 50
    req = P.CollisionRequestPOD()
    req.security_margin = -np.inf
    f4, _, _, c4, h4 = eng.scene_collide_sets(ha, tfa, hb, tfb, req=req)
    assert c4 == ncand and h4 == 0 and len(f4) == 0
    req = P.CollisionRequestPOD()
    req.num_max_contacts = 0
    with pytest.raises(hf.EngineError):
        eng.scene_collide_sets(ha, tfa, hb, tfb, req=req)
    for args in ((ha[:0], tfa[:0], hb, tfb), (ha, tfa, hb[:0], tfb[:0])):
        assert eng.scene_collide_sets(*args)[3:] == (0, 0)


@pytest.mark.gpu
def test_python_manager_cross_collide():
    rng = np.random.default_rng(41)
    geoms = [hf.Box(*(0.2 + rng.random(3))) for _ in range(4)] + [hf.Sphere(0.3), hf.Capsule(0.2, 0.6)]

    def objs(n, lo, hi):
        return [hf.CollisionObject(geoms[rng.integers(0, len(geoms))],
                                   hf.Transform3f.from_quat(*(lambda q: q / np.linalg.norm(q))(rng.normal(size=4)),
                                                            rng.uniform(lo, hi, 3))) for _ in range(n)]

    robot, env = hf.DynamicAABBTreeCollisionManager(), hf.DynamicAABBTreeCollisionManager()
    robot.registerObjects(objs(150, -3, 3))
    env.registerObjects(objs(300, -3, 3))
    env.registerObject(hf.CollisionObject(hf.Halfspace([0, 0, 1], -2.0)))
    robot.setup()
    env.setup()
    box = lambda m: np.array([np.concatenate([o.getAABB().min_, o.getAABB().max_]) for o in m.getObjects()])  # noqa: E731
    ba, bb = box(robot), box(env)
    want = brute_cross(ba, bb)
    cb = hf.CollisionCallBackCollect(100000)
    robot.collide(env, cb)
    ia = {id(o): k for k, o in enumerate(robot.getObjects())}
    ib = {id(o): k for k, o in enumerate(env.getObjects())}
    got = [(ia[id(a)], ib[id(b)]) for a, b in cb.getCollisionPairs()]  # o1 always from robot, o2 from env
    assert set(got) == want and len(got) == len(want) and any(b == 300 for _, b in got)
    # one object against a manager: the manager's object first
    q = hf.CollisionObject(hf.Box(1.5, 1.5, 1.5), hf.Transform3f(T=[0.2, 0.1, 0.0]))
    cb2 = hf.CollisionCallBackCollect(1000)
    env.collide(q, cb2)
    assert cb2.numCollisionPairs() > 0 and all(b is q and id(a) in ib for a, b in cb2.getCollisionPairs())
    qb = np.concatenate([q.getAABB().min_, q.getAABB().max_])[None]
    assert {ib[id(a)] for a, _ in cb2.getCollisionPairs()} == {j for _, j in brute_cross(qb, bb)}
    # m.collide(m, cb) is the self form
    cs, cs2 = hf.CollisionCallBackCollect(100000), hf.CollisionCallBackCollect(100000)
    env.collide(env, cs)
    env.collide(cs2)
    assert cs.getCollisionPairs() == cs2.getCollisionPairs() and cs.numCollisionPairs() > 0
    cs3 = hf.CollisionCallBackCollect(100000)
    env.collide(callback=cs3)  # the keyword form of the self query
    assert cs3.getCollisionPairs() == cs2.getCollisionPairs()
    f_self, s_self = env.pairs(env)
    assert (f_self < s_self).all() and len(f_self) == cs2.numCollisionPairs()
    # the batched form agrees with collide() on sampled pairs
    first, second, rec = robot.collide_batch(other=env)
    assert set(zip(first.tolist(), second.tolist())) == want
    req = hf.CollisionRequest()
    for k in rng.choice(len(first), 40, replace=False):
        a, b = robot.getObjects()[first[k]], env.getObjects()[second[k]]
        assert hf.collide(a.geom, a.tf, b.geom, b.tf, req, hf.CollisionResult()) == int(rec["num_contacts"][k])
    assert rec["num_contacts"].sum() > 10
