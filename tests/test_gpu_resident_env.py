"""The resident environment (hfb_env_*): set B's table, boxes and cross grid kept on the device across queries.  Every
query must return what hfb_scene_collide_sets returns for the same A and B (B's poses as of create / update), and the
flags must be the OR of the colliding pairs per A object."""
import numpy as np
import pytest

from tests.common import P, hf
from tests.test_broadphase_sets import robot_scene
from hppfcl_b200 import workloads as W

pytestmark = pytest.mark.gpu

BIG_CAP = 1 << 20


def scene(eng):
    # 64 configurations x 16 links against 5 000 objects: meshes, the halfspace floor (object 0) and a Plane wall (last)
    return robot_scene(eng, n_configs=64, n_env=5000, room=1.6, seed=33)


def by_pair(f, s, rec):
    d = {(int(a), int(b)): r.tobytes() for a, b, r in zip(f, s, rec)}
    assert len(d) == len(f)
    return d


def assert_same(got, want):
    """env result vs hfb_scene_collide_sets result: counts, pair set, records byte for byte per pair"""
    assert got[3:5] == want[3:5]
    assert by_pair(*got[:3]) == by_pair(*want[:3])


def flags_of(f, n_a):
    fl = np.zeros(n_a, dtype=np.uint8)
    fl[np.asarray(f, dtype=np.int64)] = 1
    return fl


def moved_a(rng, tfa, k):
    t = tfa.copy()
    t["T"] += rng.uniform(-0.3, 0.3, (1, 3)) * (k + 1) / 10 + rng.uniform(-0.02, 0.02, t["T"].shape)
    return t


def test_env_matches_sets_ranges_and_reuse():
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = scene(eng)
    env = eng.env_create(hb, tfb)
    want = eng.scene_collide_sets(ha, tfa, hb, tfb, capacity=BIG_CAP)
    assert want[4] > 100
    got = eng.env_collide(env, ha, tfa, capacity=BIG_CAP)
    assert_same(got, want)
    # A ranges add up to the whole
    n, parts, cand, hit = len(ha), {}, 0, 0
    for lo, cnt in ((0, 300), (300, 1), (301, n)):
        r = eng.env_collide(env, ha, tfa, capacity=BIG_CAP, first_a=lo, num_a=cnt)
        assert_same(r, eng.scene_collide_sets(ha, tfa, hb, tfb, capacity=BIG_CAP, first_a=lo, num_a=cnt))
        assert all(lo <= a < lo + cnt for a in r[0])
        parts.update(by_pair(*r[:3]))
        cand, hit = cand + r[3], hit + r[4]
    assert parts == by_pair(*want[:3]) and (cand, hit) == want[3:5]
    # ten configurations sets against the one env, between calls that reuse the context's scratch
    rng = np.random.default_rng(5)
    for k in range(10):
        t = moved_a(rng, tfa, k)
        if k % 2:
            eng.scene_collide(np.concatenate([ha[:200], hb[:800]]), np.concatenate([t[:200], tfb[:800]]), capacity=BIG_CAP)
        else:
            eng.batch_distance(ha[:500], t[:500], hb[1:501], tfb[1:501])
        assert_same(eng.env_collide(env, ha, t, capacity=BIG_CAP), eng.scene_collide_sets(ha, t, hb, tfb, capacity=BIG_CAP))
    # a larger A than any before: the table regrows in front of B
    ha2, tfa2 = np.concatenate([ha, ha, ha]), np.concatenate([tfa, moved_a(rng, tfa, 3), moved_a(rng, tfa, 7)])
    assert_same(eng.env_collide(env, ha2, tfa2, capacity=BIG_CAP), eng.scene_collide_sets(ha2, tfa2, hb, tfb, capacity=BIG_CAP))
    assert_same(eng.env_collide(env, ha, tfa, capacity=BIG_CAP), want)
    eng.env_destroy(env)


def cross_cell(bb):
    """the cell of the cross grid over boxes bb (cross_cell / cross_grid_fit of hfb_broadphase.cuh): the top of the log2
    bin that holds the 95th percentile of the extents of the bounded, non-empty boxes"""
    big = np.finfo(np.float64).max
    live = ~((bb[:, 0] == big) & (bb[:, 3] == -big)) & np.all(np.abs(bb) < 1e300, axis=1)
    ext = np.max(bb[live, 3:] - bb[live, :3], axis=1)
    bins = np.where(ext > 0, np.clip(np.frexp(ext)[1] - 1 + 64, 1, 127), 0)
    hist = np.bincount(bins, minlength=128)
    b = int(np.argmax(np.cumsum(hist[:127]) >= len(ext) - len(ext) // 20))
    if b == 0:
        b = 1 + int(np.argmax(hist[1:] > 0))
    centres = 0.5 * (bb[live, :3] + bb[live, 3:])
    return max(2.0 ** (b - 63), float(np.max(centres.max(0) - centres.min(0))) * 2.0 ** -21)


def box_extent(eng, h, t):
    b = eng.scene_aabbs(np.array([h], dtype=np.uint32), t.reshape(1))[0]
    return float(np.max(b[3:] - b[:3]))


def test_env_update():
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = scene(eng)
    hb, tfb = hb.copy(), tfb.copy()
    # a thin square plate at a link's centre: 0.9 cells wide axis-aligned, 1.27 cells once turned 45 degrees about z
    cell = cross_cell(eng.scene_aabbs(hb, tfb))
    plate = eng.register_shapes(P.make_shapes([P.GEOM_BOX], [[0.45 * cell, 0.45 * cell, 0.002]]))[0]
    eng.commit()
    k_plate = 20
    hb[k_plate] = plate
    tfb[k_plate] = W.identity_transforms(1, T=tfa["T"][3:4])[0]
    cell = cross_cell(eng.scene_aabbs(hb, tfb))
    assert box_extent(eng, plate, tfb[k_plate]) <= cell  # in the grid
    env = eng.env_create(hb, tfb)
    rng = np.random.default_rng(8)
    nb = len(hb)

    def check():
        assert_same(eng.env_collide(env, ha, tfa, capacity=BIG_CAP), eng.scene_collide_sets(ha, tfa, hb, tfb, capacity=BIG_CAP))

    def move(idx, t):
        tfb[idx] = t
        eng.env_update(env, idx, t)
        check()

    # far outside the original bounds, and some of those back into the robot's reach
    idx = rng.choice(np.setdiff1d(np.arange(10, nb - 1), [k_plate]), 60, replace=False)
    t = tfb[idx].copy()
    t["T"] += [40.0, -25.0, 9.0]
    move(idx, t)
    t = tfb[idx[:20]].copy()
    t["T"] = tfa["T"][rng.choice(len(tfa), 20)]
    move(idx[:20], t)
    # the plate turned so that its box outgrows the cell: on the oversize list now
    c, sn = np.cos(np.pi / 4), np.sin(np.pi / 4)
    t = tfb[[k_plate]].copy()
    t["R"] = np.array([[c, -sn, 0.0], [sn, c, 0.0], [0.0, 0.0, 1.0]]).reshape(1, 9)
    tb = tfb.copy()
    tb[k_plate] = t[0]
    assert box_extent(eng, plate, t[0]) > cross_cell(eng.scene_aabbs(hb, tb))
    move(np.array([k_plate]), t)
    assert any(b == k_plate for b in eng.env_collide(env, ha, tfa, capacity=BIG_CAP)[1])
    # the floor raised by 30 cm
    t = tfb[[0]].copy()
    t["T"] = [0.0, 0.0, 0.3]
    move(np.array([0]), t)
    move(np.zeros(0, dtype=np.int64), tfb[:0])  # an empty update
    # repeated and out-of-range indices: refused, nothing moves
    before = eng.env_collide(env, ha, tfa, capacity=BIG_CAP)
    far = tfb[[5, 6]].copy()
    far["T"] = 1e3
    for bad in ([5, 5], [5, nb], [nb + 10, 6]):
        with pytest.raises(hf.EngineError, match="invalid argument"):
            eng.env_update(env, np.array(bad), far)
    assert_same(eng.env_collide(env, ha, tfa, capacity=BIG_CAP), before)


def test_env_flags_and_edge_cases():
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = scene(eng)
    env = eng.env_create(hb, tfb)
    n = len(ha)
    want = eng.scene_collide_sets(ha, tfa, hb, tfb, capacity=BIG_CAP)
    got = eng.env_collide(env, ha, tfa, capacity=BIG_CAP, flags=True)
    assert_same(got[:5], want)
    assert np.array_equal(got[5], flags_of(want[0], n)) and 0 < got[5].sum() < n
    only = eng.env_collide(env, ha, tfa, capacity=0, flags=True)  # flags alone: no records
    assert len(only[0]) == 0 and only[3:5] == want[3:5] and np.array_equal(only[5], got[5])
    lo, cnt = 200, 333
    part = eng.env_collide(env, ha, tfa, capacity=0, flags=True, first_a=lo, num_a=cnt)
    inside = np.zeros(n, dtype=bool)
    inside[lo:lo + cnt] = True
    assert np.array_equal(part[5], np.where(inside, got[5], 0))
    # security_margin = -inf: candidates counted, nothing collides
    req = P.CollisionRequestPOD()
    req.security_margin = -np.inf
    r = eng.env_collide(env, ha, tfa, req, capacity=BIG_CAP, flags=True)
    s = eng.scene_collide_sets(ha, tfa, hb, tfb, req, capacity=BIG_CAP)
    assert r[3:5] == s[3:5] == (want[3], 0) and not r[5].any() and len(r[0]) == 0
    # num_max_contacts = 0: refused by both
    req = P.CollisionRequestPOD()
    req.num_max_contacts = 0
    for call in (lambda: eng.env_collide(env, ha, tfa, req), lambda: eng.scene_collide_sets(ha, tfa, hb, tfb, req)):
        with pytest.raises(hf.EngineError, match="invalid argument"):
            call()
    # capacity below the count: all counted, `capacity` of them stored
    r = eng.env_collide(env, ha, tfa, capacity=50, flags=True)
    assert r[3:5] == want[3:5] and len(r[0]) == 50 and np.array_equal(r[5], got[5])
    wd = by_pair(*want[:3])
    assert all(wd[p] == rec for p, rec in by_pair(*r[:3]).items())
    # empty A, empty B
    r = eng.env_collide(env, ha[:0], tfa[:0], capacity=BIG_CAP, flags=True)
    assert r[3:5] == (0, 0) and len(r[5]) == 0
    empty = eng.env_create(hb[:0], tfb[:0])
    r = eng.env_collide(empty, ha, tfa, capacity=BIG_CAP, flags=True)
    assert r[3:5] == (0, 0) == eng.scene_collide_sets(ha, tfa, hb[:0], tfb[:0])[3:5] and not r[5].any()
    eng.env_update(empty, [], tfb[:0])
    eng.env_destroy(empty)


def test_env_device_form_equals_host_form():
    import torch
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = scene(eng)
    env = eng.env_create(hb, tfb)
    n = len(ha)

    def dev(x):
        return torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1)).cuda()

    stream = torch.cuda.Stream()
    cap = 200_000
    d_f = torch.zeros(cap, dtype=torch.int32, device="cuda")
    d_s = torch.zeros(cap, dtype=torch.int32, device="cuda")
    d_rec = torch.zeros(cap * P.contact_dtype.itemsize, dtype=torch.uint8, device="cuda")
    d_cnt = torch.zeros(2, dtype=torch.int32, device="cuda")
    d_fl = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
    rng = np.random.default_rng(2)
    for k, (lo, cnt, c) in enumerate(((0, n, cap), (100, 400, cap), (0, n, 0), (0, n, 60))):
        t = moved_a(rng, tfa, k)
        d_h, d_t = dev(ha), dev(t)
        torch.cuda.synchronize()
        eng.env_collide_device(env, n, d_h.data_ptr(), d_t.data_ptr(), d_f.data_ptr(), d_s.data_ptr(), d_rec.data_ptr(), c,
                               d_cnt.data_ptr(), d_cnt.data_ptr() + 4, d_fl.data_ptr(), stream=stream.cuda_stream,
                               first_a=lo, num_a=cnt)
        stream.synchronize()
        host = eng.env_collide(env, ha, t, capacity=c, flags=True, first_a=lo, num_a=cnt)
        hits, cand = (int(x) for x in d_cnt.cpu().numpy())
        assert (cand, hits) == host[3:5] and hits > 0
        assert np.array_equal(d_fl.cpu().numpy(), host[5])
        kk = min(hits, c)
        rec = d_rec[:kk * P.contact_dtype.itemsize].cpu().numpy().view(P.contact_dtype)
        got = by_pair(d_f[:kk].cpu().numpy(), d_s[:kk].cpu().numpy(), rec)
        if kk == hits:
            assert got == by_pair(*host[:3])
        else:  # a different subset of the colliding pairs may be kept: each as the full set has it
            full = by_pair(*eng.env_collide(env, ha, t, capacity=BIG_CAP, first_a=lo, num_a=cnt)[:3])
            assert all(full[p] == r for p, r in got.items())


def test_env_device_call_then_host_scene_calls_unsynchronised():
    """hfb_env_collide_device returns while its narrow phase and compaction still run on the caller's stream; the host
    scene calls that follow on the same context, with no synchronisation in between, share its candidate and counter
    buffers and must wait for it: both results as each call alone gives them"""
    import torch
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = scene(eng)
    env = eng.env_create(hb, tfb)
    n = len(ha)
    rng = np.random.default_rng(4)
    t_other = moved_a(rng, tfa, 5)
    want_dev = eng.env_collide(env, ha, tfa, capacity=BIG_CAP, flags=True)
    want_sets = eng.scene_collide_sets(ha, t_other, hb, tfb, capacity=BIG_CAP)
    tab_h, tab_t = np.concatenate([ha, hb[:3000]]), np.concatenate([t_other, tfb[:3000]])
    want_self = eng.scene_collide(tab_h, tab_t, capacity=BIG_CAP)
    assert want_dev[4] > 100 and want_sets[4] > 100 and want_self[4] > 100

    def dev(x):
        return torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1)).cuda()

    side = torch.cuda.Stream()
    cap = 200_000
    d_h, d_t = dev(ha), dev(tfa)
    d_f = torch.zeros(cap, dtype=torch.int32, device="cuda")
    d_s = torch.zeros(cap, dtype=torch.int32, device="cuda")
    d_rec = torch.zeros(cap * P.contact_dtype.itemsize, dtype=torch.uint8, device="cuda")
    d_cnt = torch.zeros(2, dtype=torch.int32, device="cuda")
    d_fl = torch.zeros(n, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    for host_call, want in ((lambda: eng.scene_collide_sets(ha, t_other, hb, tfb, capacity=BIG_CAP), want_sets),
                            (lambda: eng.scene_collide(tab_h, tab_t, capacity=BIG_CAP), want_self)):
        eng.env_collide_device(env, n, d_h.data_ptr(), d_t.data_ptr(), d_f.data_ptr(), d_s.data_ptr(), d_rec.data_ptr(), cap,
                               d_cnt.data_ptr(), d_cnt.data_ptr() + 4, d_fl.data_ptr(), stream=side.cuda_stream)
        got = host_call()  # no synchronisation in between
        side.synchronize()
        assert_same(got, want)
        hits, cand = (int(x) for x in d_cnt.cpu().numpy())
        assert (cand, hits) == want_dev[3:5]
        rec = d_rec[:hits * P.contact_dtype.itemsize].cpu().numpy().view(P.contact_dtype)
        assert by_pair(d_f[:hits].cpu().numpy(), d_s[:hits].cpu().numpy(), rec) == by_pair(*want_dev[:3])
        assert np.array_equal(d_fl.cpu().numpy(), want_dev[5])


def test_env_geometry_changes_and_lifetime():
    import torch
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = scene(eng)
    env = eng.env_create(hb, tfb)
    eng.env_collide(env, ha, tfa)
    eng.release_shapes([hb[3]])  # a handle of B released and committed
    eng.commit()
    with pytest.raises(hf.EngineError, match="invalid argument"):
        eng.env_collide(env, ha, tfa)
    with pytest.raises(hf.EngineError, match="invalid argument"):
        eng.env_update(env, [4], tfb[[4]])
    env2 = eng.env_create(ha[:10], tfa[:10])
    eng.clear_geometry()
    w["register"](eng)
    eng.commit()
    for e in (env, env2):
        with pytest.raises(hf.EngineError, match="invalid argument"):
            eng.env_collide(e, ha, tfa)
        eng.env_destroy(e)
    with pytest.raises(hf.EngineError, match="invalid argument"):
        eng.env_destroy(env)  # not an env of this context any more
    eng.close()
    # contexts destroyed with live envs: their memory comes back
    torch.cuda.synchronize()

    def cycle():
        e = hf.Engine(0)
        _, ha_, tfa_, hb_, tfb_ = scene(e)
        env_ = e.env_create(hb_, tfb_)
        e.env_collide(env_, ha_, tfa_)
        e.close()

    cycle()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        cycle()
    assert torch.cuda.mem_get_info()[0] > free0 - (64 << 20)


def test_python_resident_environment_and_manager_update():
    rng = np.random.default_rng(17)

    def pose():
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        return hf.Transform3f.from_quat(*q, T=rng.uniform(0, 6, 3))

    geoms = [hf.Box(0.6, 0.4, 0.8), hf.Sphere(0.3), hf.Capsule(0.2, 0.6)]
    robot = [hf.CollisionObject(geoms[i % 3], pose()) for i in range(150)]
    env_objs = [hf.CollisionObject(hf.Halfspace(np.array([0.0, 0, 1]), 0.2))]
    env_objs += [hf.CollisionObject(geoms[i % 3], pose()) for i in range(450)]
    mr, me = hf.DynamicAABBTreeCollisionManager(), hf.DynamicAABBTreeCollisionManager()
    mr.registerObjects(robot)
    me.registerObjects(env_objs)
    mr.setup()
    me.setup()
    with hf.ResidentEnvironment(me) as re:
        for _ in range(2):
            f, s, rec = mr.collide_batch(other=me)
            hit = rec["num_contacts"] > 0
            want = set(zip(f[hit].tolist(), s[hit].tolist()))
            assert len(want) > 20 and any(b == 0 for _, b in want)
            gf, gs, grec = re.collide(mr)
            assert set(zip(gf.tolist(), gs.tolist())) == want and len(gf) == len(want) and (grec["num_contacts"] > 0).all()
            assert np.array_equal(re.collide_flags(mr), flags_of(f[hit], len(robot)))
            moved = env_objs[10:60] + [env_objs[0]]
            for o in moved:
                o.setTransform(pose())
            me.update(moved[:-1])
            me.update(moved[-1])
            boxes = [(o.aabb.min_.copy(), o.aabb.max_.copy()) for o in env_objs]
            fresh = hf.DynamicAABBTreeCollisionManager()
            fresh.registerObjects(env_objs)
            fresh.setup()
            assert all(np.array_equal(a, o.aabb.min_) and np.array_equal(b, o.aabb.max_) for (a, b), o in zip(boxes, env_objs))
            re.update(moved)
        # an object the manager does not hold: skipped by the manager's update, as the reference does; refused by the env
        stray = robot[0]
        before = stray.aabb
        me.update(stray)
        me.update([stray, env_objs[5]])
        assert stray.aabb is before
        with pytest.raises(ValueError):
            re.update([stray])
