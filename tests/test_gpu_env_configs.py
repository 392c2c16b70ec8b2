"""The configurations query (hfb_env_collide_configs*): robot configurations against the resident environment and
against themselves in one call.  Its environment pairs must be what hfb_env_collide returns, its self pairs what
hfb_batch_collide_objects returns for the template's pairs whose boxes overlap (hfb_broadphase_config_pairs), and each
verdict the OR of the colliding pairs of its configuration."""
import numpy as np
import pytest

from tests.common import P, compare_distance, hf, make_scenes
from tests.test_config_pairs import brute_config, load_recorded, reference_sample
from tests.test_gpu_edge_inputs import NONFINITE_FIELDS, same_fields
from hppfcl_b200 import workloads as W

pytestmark = pytest.mark.gpu

BIG_CAP = 1 << 20
LINKS = 16
TPL = W.chain_self_pairs(LINKS)


def config_scene(eng, n_configs=256, n_env=500, room=3.0, seed=35, oracle=False):
    """the robot workload with the bending joints in +-2.8 rad, so that some configurations fold onto themselves, and a
    Plane wall added to B; the floor, the wall and the large boxes are moved out of the robot's reach, so that some
    configurations are free -> (w, ha, tfa, hb, tfb).  oracle: eng also registers in the oracle (a MultiScene)"""
    w = W.robot_vs_environment(n_configs=n_configs, n_env=n_env, room=room, seed=seed, joint_range=2.8)
    hs = w["register"](eng, oracle=oracle)
    ha, tfa = hs[w["geom_a"]].astype(np.uint32), w["tf_a"]
    hb, tfb = hs[w["geom_b"]].astype(np.uint32), w["tf_b"].copy()
    wall = eng.register_halfspaces(P.GEOM_PLANE, [[1, 0, 0, -0.5]])
    hb[-1] = wall[0]
    tfb[-1] = W.identity_transforms(1)[0]
    tfb[0] = W.identity_transforms(1, T=[[0.0, 0.0, -2.0]])[0]
    tfb["T"][(w["geom_b"] >= LINKS + 64) & (w["geom_b"] < LINKS + 80), 2] += 10.0  # the tables and shelves
    eng.commit()
    return w, ha, tfa, hb, tfb


def by_pair(f, s, rec):
    d = {(int(a), int(b)): r.tobytes() for a, b, r in zip(f, s, rec)}
    assert len(d) == len(f)
    return d


def expected(eng, env, ha, tfa, tpl=TPL, g0=0, ng=None, req=None):
    """what the existing calls give: (verdicts, env = hfb_env_collide's result, self = (first, second, records,
    n_candidates, n_colliding) from the host finder's candidates through hfb_batch_collide_objects)"""
    n_configs = len(ha) // LINKS
    ng = n_configs - g0 if ng is None else ng
    e = eng.env_collide(env, ha, tfa, req, capacity=BIG_CAP, first_a=g0 * LINKS, num_a=ng * LINKS)
    sf, ss = hf.broadphase_config_pairs(eng.scene_aabbs(ha, tfa), LINKS, tpl, g0, ng)
    if len(sf) and (req is None or req.security_margin != -np.inf):
        rec = eng.batch_collide_objects(ha, tfa, sf, ss, req)
    else:
        rec = np.zeros(len(sf), dtype=P.contact_dtype)
    hit = rec["num_contacts"] > 0
    s = (sf[hit], ss[hit], rec[hit], len(sf), int(hit.sum()))
    v = np.zeros(n_configs, dtype=np.uint8)
    v[np.asarray(e[0], dtype=np.int64) // LINKS] = 1
    v[np.asarray(s[0], dtype=np.int64) // LINKS] = 1
    return v, e, s


def assert_same(got, want, records=True):
    v, e, s = got
    wv, we, ws = want
    assert np.array_equal(v, wv)
    for g, w in ((e, we), (s, ws)):
        assert g[3:5] == w[3:5]
        if records:
            assert by_pair(*g[:3]) == by_pair(*w[:3])


def kinds(want):
    """configurations that are free, collide with the environment only, with themselves only, with both"""
    v, e, s = want
    n = len(v)
    env_hit = np.zeros(n, dtype=bool)
    env_hit[np.asarray(e[0], dtype=np.int64) // LINKS] = True
    self_hit = np.zeros(n, dtype=bool)
    self_hit[np.asarray(s[0], dtype=np.int64) // LINKS] = True
    return (~env_hit & ~self_hit), (env_hit & ~self_hit), (~env_hit & self_hit), (env_hit & self_hit)


def test_configs_match_the_existing_calls():
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = config_scene(eng)
    env = eng.env_create(hb, tfb)
    want = expected(eng, env, ha, tfa)
    free, env_only, self_only, both = kinds(want)
    assert min(free.sum(), env_only.sum(), self_only.sum(), both.sum()) >= 5  # every kind of configuration occurs
    got = eng.env_collide_configs(env, ha, tfa, LINKS, TPL, env_capacity=BIG_CAP, self_capacity=BIG_CAP)
    assert_same(got, want)
    assert got[2][3] > 500 and got[2][4] > 40 and got[1][4] > 100
    # configuration ranges add up to the whole
    n_configs = len(ha) // LINKS
    parts = [{}, {}]
    counts = np.zeros(4, dtype=np.int64)
    verdicts = np.zeros(n_configs, dtype=np.uint8)
    for g0, ng in ((0, 50), (50, 1), (51, 0), (51, n_configs - 51)):
        r = eng.env_collide_configs(env, ha, tfa, LINKS, TPL, env_capacity=BIG_CAP, self_capacity=BIG_CAP, first_config=g0,
                                    num_configs=ng)
        assert_same(r, expected(eng, env, ha, tfa, g0=g0, ng=ng))
        assert not r[0][:g0].any() and not r[0][g0 + ng:].any()
        for k in (1, 2):
            assert all(g0 * LINKS <= a < (g0 + ng) * LINKS for a in r[k][0])
            parts[k - 1].update(by_pair(*r[k][:3]))
        counts += [r[1][3], r[1][4], r[2][3], r[2][4]]
        verdicts |= r[0]
    assert parts == [by_pair(*got[1][:3]), by_pair(*got[2][:3])]
    assert list(counts) == [got[1][3], got[1][4], got[2][3], got[2][4]] and np.array_equal(verdicts, got[0])
    # verdicts only: no records, the same counts
    only = eng.env_collide_configs(env, ha, tfa, LINKS, TPL, env_capacity=0, self_capacity=0)
    assert len(only[1][0]) == len(only[2][0]) == 0
    assert_same(only, want, records=False)
    # capacities below the hit counts: every pair counted, the kept ones as the full set has them
    r = eng.env_collide_configs(env, ha, tfa, LINKS, TPL, env_capacity=30, self_capacity=7)
    assert_same(r, want, records=False) and len(r[1][0]) == 30 and len(r[2][0]) == 7
    for k in (1, 2):
        full = by_pair(*want[k][:3])
        assert all(full[p] == rec for p, rec in by_pair(*r[k][:3]).items())
    # pairs without verdicts
    r = eng.env_collide_configs(env, ha, tfa, LINKS, TPL, env_capacity=BIG_CAP, self_capacity=BIG_CAP, verdicts=False)
    assert r[0] is None and r[1][3:] == want[1][3:] and by_pair(*r[2][:3]) == by_pair(*want[2][:3])
    # an empty template: the env's flags OR-ed per configuration
    empty = np.zeros((0, 2), dtype=np.uint32)
    r = eng.env_collide_configs(env, ha, tfa, LINKS, empty, env_capacity=BIG_CAP, self_capacity=BIG_CAP)
    flags = eng.env_collide(env, ha, tfa, capacity=0, flags=True)[5]
    assert np.array_equal(r[0], flags.reshape(-1, LINKS).max(axis=1)) and r[2][3:] == (0, 0)
    assert_same(r, expected(eng, env, ha, tfa, tpl=empty))
    # security_margin = -inf: candidates counted, no contacts, all verdicts 0
    req = P.CollisionRequestPOD()
    req.security_margin = -np.inf
    r = eng.env_collide_configs(env, ha, tfa, LINKS, TPL, req, BIG_CAP, BIG_CAP)
    assert not r[0].any() and r[1][3:] == (want[1][3], 0) and r[2][3:] == (want[2][3], 0)
    assert len(r[1][0]) == len(r[2][0]) == 0
    # refused: num_max_contacts = 0, malformed templates, a range past the end, n_a not a multiple of the links
    req = P.CollisionRequestPOD()
    req.num_max_contacts = 0
    for call in (lambda: eng.env_collide_configs(env, ha, tfa, LINKS, TPL, req),
                 lambda: eng.env_collide_configs(env, ha, tfa, LINKS, [(0, 2), (2, 0)]),
                 lambda: eng.env_collide_configs(env, ha, tfa, LINKS, [(3, 3)]),
                 lambda: eng.env_collide_configs(env, ha, tfa, LINKS, [(0, LINKS)]),
                 lambda: eng.env_collide_configs(env, ha, tfa, LINKS, TPL, first_config=n_configs - 1, num_configs=2),
                 lambda: eng.env_collide_configs(env, ha[:-1], tfa[:-1], LINKS, TPL),
                 lambda: eng.env_collide_configs(env, ha, tfa, 0, TPL)):
        with pytest.raises(hf.EngineError, match="invalid argument"):
            call()
    assert_same(eng.env_collide_configs(env, ha, tfa, LINKS, TPL, env_capacity=BIG_CAP, self_capacity=BIG_CAP), want)
    eng.env_destroy(env)


def test_env_without_objects_checks_the_self_pairs():
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = config_scene(eng)
    env = eng.env_create(hb[:0], tfb[:0])
    want = expected(eng, env, ha, tfa)
    assert want[1][3:] == (0, 0) and want[2][4] > 20
    got = eng.env_collide_configs(env, ha, tfa, LINKS, TPL, env_capacity=BIG_CAP, self_capacity=BIG_CAP)
    assert_same(got, want)
    assert got[0].sum() == len(np.unique(np.asarray(want[2][0]) // LINKS))
    r = eng.env_collide_configs(env, ha[:0], tfa[:0], LINKS, TPL)
    assert len(r[0]) == 0 and r[1][3:] == r[2][3:] == (0, 0)
    eng.env_destroy(env)


def test_update_flips_a_verdict():
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = config_scene(eng)
    tfb = tfb.copy()
    env = eng.env_create(hb, tfb)
    want = expected(eng, env, ha, tfa)
    free = np.nonzero(kinds(want)[0])[0]
    g = int(free[len(free) // 2])
    # a small object of B moved onto link 8 of a free configuration
    k = next(i for i in range(20, len(hb) - 1) if w["geom_b"][i] >= LINKS and w["geom_b"][i] < LINKS + 64)
    t = tfb[[k]].copy()
    t["T"] = tfa["T"][g * LINKS + 8]
    tfb[k] = t[0]
    eng.env_update(env, [k], t)
    got = eng.env_collide_configs(env, ha, tfa, LINKS, TPL, env_capacity=BIG_CAP, self_capacity=BIG_CAP)
    want2 = expected(eng, env, ha, tfa)
    assert_same(got, want2)
    assert got[0][g] == 1 and (g * LINKS + 8, k) in by_pair(*got[1][:3])
    changed = np.nonzero(got[0] != want[0])[0]
    assert g in changed
    eng.env_destroy(env)


def dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1)).cuda()


class DeviceOut:
    """device buffers of the configurations query and their download"""

    def __init__(self, n_configs, cap):
        import torch
        self.cap = cap
        z = lambda n, dt=torch.int32: torch.zeros(n, dtype=dt, device="cuda")  # noqa: E731
        self.v = torch.full((n_configs,), 7, dtype=torch.uint8, device="cuda")
        self.kinds = [(z(cap), z(cap), z(cap * P.contact_dtype.itemsize, torch.uint8)) for _ in range(2)]
        self.cnt = z(4)  # env colliding, env candidates, self colliding, self candidates

    def out(self, caps):
        c = self.cnt.data_ptr()
        return [(f.data_ptr(), s.data_ptr(), r.data_ptr(), cap, c + 8 * k, c + 8 * k + 4)
                for k, ((f, s, r), cap) in enumerate(zip(self.kinds, caps))]

    def result(self, caps):
        cnt = [int(x) for x in self.cnt.cpu().numpy()]
        res = []
        for k, ((f, s, r), cap) in enumerate(zip(self.kinds, caps)):
            m = min(cnt[2 * k], cap)
            rec = r[:m * P.contact_dtype.itemsize].cpu().numpy().view(P.contact_dtype)
            res.append((f[:m].cpu().numpy().astype(np.uint32), s[:m].cpu().numpy().astype(np.uint32), rec, cnt[2 * k + 1],
                        cnt[2 * k]))
        return self.v.cpu().numpy(), res[0], res[1]


def test_device_form_equals_host_form():
    import torch
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = config_scene(eng)
    env = eng.env_create(hb, tfb)
    n_configs = len(ha) // LINKS
    d = DeviceOut(n_configs, 100_000)
    stream = torch.cuda.Stream()
    rng = np.random.default_rng(2)
    for k, (g0, ng, caps) in enumerate(((0, n_configs, (d.cap, d.cap)), (40, 100, (d.cap, d.cap)), (0, n_configs, (0, 0)),
                                        (0, n_configs, (25, 9)))):
        t = tfa.copy()
        t["T"] += rng.uniform(-0.2, 0.2, (n_configs, 1, 3)).repeat(LINKS, axis=1).reshape(-1, 3) * (k % 2)
        d_h, d_t = dev(ha), dev(t)
        torch.cuda.synchronize()
        eng.env_collide_configs_device(env, len(ha), d_h.data_ptr(), d_t.data_ptr(), LINKS, TPL, d.v.data_ptr(),
                                       *d.out(caps), stream=stream.cuda_stream, first_config=g0, num_configs=ng)
        stream.synchronize()
        got = d.result(caps)
        host = eng.env_collide_configs(env, ha, t, LINKS, TPL, env_capacity=caps[0], self_capacity=caps[1], first_config=g0,
                                       num_configs=ng)
        full = caps[0] >= host[1][4] and caps[1] >= host[2][4]
        assert_same(got, host, records=full)
        assert host[2][4] > 0 and host[1][4] > 0
        if not full:  # a different subset of the colliding pairs may be kept: each as the full set has it
            whole = eng.env_collide_configs(env, ha, t, LINKS, TPL, env_capacity=BIG_CAP, self_capacity=BIG_CAP,
                                            first_config=g0, num_configs=ng)
            for kk in (1, 2):
                assert len(got[kk][0]) == min(caps[kk - 1], host[kk][4])
                ref = by_pair(*whole[kk][:3])
                assert all(ref[p] == r for p, r in by_pair(*got[kk][:3]).items())


def test_device_call_then_host_env_calls_unsynchronised():
    """the device form returns while its narrow phase and compaction still run on the caller's stream; host env calls
    on the same context that follow with no synchronisation in between must wait for it: both results right"""
    import torch
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = config_scene(eng)
    env = eng.env_create(hb, tfb)
    n_configs = len(ha) // LINKS
    t_other = tfa.copy()
    t_other["T"] += 0.15
    want_dev = eng.env_collide_configs(env, ha, tfa, LINKS, TPL, env_capacity=BIG_CAP, self_capacity=BIG_CAP)
    want_cfg = eng.env_collide_configs(env, ha, t_other, LINKS, TPL[::2], env_capacity=BIG_CAP, self_capacity=BIG_CAP)
    want_env = eng.env_collide(env, ha, t_other, capacity=BIG_CAP, flags=True)
    d = DeviceOut(n_configs, 100_000)
    caps = (d.cap, d.cap)
    d_h, d_t = dev(ha), dev(tfa)
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    for host_call, check in ((lambda: eng.env_collide_configs(env, ha, t_other, LINKS, TPL[::2], env_capacity=BIG_CAP,
                                                              self_capacity=BIG_CAP), lambda r: assert_same(r, want_cfg)),
                             (lambda: eng.env_collide(env, ha, t_other, capacity=BIG_CAP, flags=True),
                              lambda r: r[3:5] == want_env[3:5] and by_pair(*r[:3]) == by_pair(*want_env[:3]) and
                              np.array_equal(r[5], want_env[5]))):
        eng.env_collide_configs_device(env, len(ha), d_h.data_ptr(), d_t.data_ptr(), LINKS, TPL, d.v.data_ptr(),
                                       *d.out(caps), stream=side.cuda_stream)
        got = host_call()  # no synchronisation in between
        side.synchronize()
        assert check(got) is not False
        assert_same(d.result(caps), want_dev)


def test_self_records_equal_the_reference():
    """the self pairs of a small scene: the device's candidates are the host finder's, and its records equal the
    reference build's (its recorded outputs where it is not built here)"""
    load_recorded()
    sc = make_scenes(gpu=True, emu=True, ref=True)
    eng = sc.b["gpu"]
    w, ha, tfa, f, s = reference_sample(sc)
    env = eng.env_create(ha[:0], tfa[:0])
    got = eng.env_collide_configs(env, ha, tfa, LINKS, TPL, env_capacity=BIG_CAP, self_capacity=BIG_CAP)
    rr = sc.b["ref"].batch_collide(ha[f], tfa[f], ha[s], tfa[s])
    hit = rr["num_contacts"] > 0
    assert got[2][3] == len(f) and got[2][4] == int(hit.sum()) > 20
    mine = by_pair(*got[2][:3])
    keys = list(zip(f[hit].tolist(), s[hit].tolist()))
    assert set(mine) == set(keys)
    rec = np.frombuffer(b"".join(mine[p] for p in keys), dtype=P.contact_dtype)
    compare_distance(rr[hit], rec, what="self pairs against the reference")
    eng.env_destroy(env)


def test_nonfinite_and_huge_poses():
    """a configuration with a NaN pose and one displaced by 1e100: exactly the oracle's colliding pairs and records
    there (whole records where the poses are finite, the fields the edge suite compares elsewhere)"""
    sc = make_scenes(gpu=True, emu=False)
    eng, orc = sc.b["gpu"], sc.b["oracle"]
    w, ha, tfa, hb, tfb = config_scene(sc, n_configs=64, n_env=600, oracle=True)
    tfa = tfa.copy()
    g_nan, g_far = 5, 9
    tfa["T"][g_nan * LINKS + 6, 1] = np.nan
    tfa["R"][g_nan * LINKS + 11, 4] = np.inf
    tfa["T"][g_far * LINKS:(g_far + 1) * LINKS] += 1e100
    env = eng.env_create(hb, tfb)
    got = eng.env_collide_configs(env, ha, tfa, LINKS, TPL, env_capacity=BIG_CAP, self_capacity=BIG_CAP)
    bb = eng.scene_aabbs(ha, tfa)
    finite = np.isfinite(tfa["T"]).all(axis=1) & np.isfinite(tfa["R"]).all(axis=1)
    for g in (g_nan, g_far):
        cand = brute_config(bb, LINKS, TPL, g, 1)
        i, j = np.array([p[0] for p in cand]), np.array([p[1] for p in cand])
        ro = orc.batch_collide(ha[i], tfa[i], ha[j], tfa[j], nthreads=0)
        want = {cand[r] for r in np.nonzero(ro["num_contacts"] > 0)[0]}
        mine = {p: r for p, r in by_pair(*got[2][:3]).items() if g * LINKS <= p[0] < (g + 1) * LINKS}
        assert set(mine) == want and (g != g_far or len(want) == len(TPL))
        keys = sorted(want)
        if not keys:
            continue
        rows = np.array([cand.index(p) for p in keys])
        rec = np.frombuffer(b"".join(mine[p] for p in keys), dtype=P.contact_dtype)
        ok = finite[i[rows]] & finite[j[rows]]
        compare_distance(ro[rows][ok], rec[ok], what="finite self pairs")
        same_fields(ro[rows][~ok], rec[~ok], NONFINITE_FIELDS, "non-finite self pairs")
    # the other configurations are as the existing calls give them
    want = expected(eng, env, ha, tfa)
    assert np.array_equal(got[0], want[0]) and got[2][3:] == want[2][3:]
    eng.env_destroy(env)


def mirror_scene(rng, n_configs=128, base_z=0.3, n_env=120):
    """a chain robot (boxes and capsules) folded at random and an environment with a floor -> (links, robot poses as
    (R, T) per object, environment (geometry index, R, T) per object)"""
    links = 8
    ang = rng.uniform(-2.8, 2.8, (n_configs, links))
    base = rng.uniform(0, 3, (n_configs, 3)) * [1, 1, 0] + [0, 0, base_z]
    robot = []
    for g in range(n_configs):
        R, p = np.eye(3), base[g].copy()
        for k in range(links):
            R = R @ W._axis_rotations(2 if k % 2 == 0 else 1, np.array(ang[g, k]))
            robot.append((R.copy(), p + 0.11 * R[:, 2]))
            p = p + 0.22 * R[:, 2]
    env = [(3, np.eye(3), np.zeros(3))]
    for _ in range(n_env):
        q = rng.normal(size=4)
        env.append((int(rng.integers(0, 3)), W.quat_to_rot(*(q / np.linalg.norm(q))), rng.uniform(0, 3, 3) * [1, 1, 0.4]))
    return links, robot, env


def mirror_geoms():
    return [hf.Box(0.3, 0.2, 0.25), hf.Sphere(0.15), hf.Capsule(0.1, 0.3), hf.Halfspace(np.array([0.0, 0, 1]), 0.02)]


def python_mirror(rng):
    """the Python mirror's configurations query on mirror_scene(rng), checked against the existing routes (the
    environment's pairs by collide_batch, the template's pairs through hfb_batch_collide_objects) -> (links, robot, env,
    template, verdicts, environment pairs, self pairs)"""
    links, robot, env = mirror_scene(rng)
    tpl = W.chain_self_pairs(links)
    geoms = mirror_geoms()
    link_geom = [hf.Capsule(0.05, 0.14), hf.Box(0.08, 0.08, 0.22)]
    ro = [hf.CollisionObject(link_geom[link_kind(k, links)], hf.Transform3f(R, T)) for k, (R, T) in enumerate(robot)]
    eo = [hf.CollisionObject(geoms[gi], hf.Transform3f(R, T)) for gi, R, T in env]
    mr, me = hf.DynamicAABBTreeCollisionManager(), hf.DynamicAABBTreeCollisionManager()
    mr.registerObjects(ro)
    me.registerObjects(eo)
    mr.setup()
    me.setup()
    with hf.ResidentEnvironment(me) as re:
        v, ep, sp = re.collide_configurations(mr, links, tpl)
        assert np.array_equal(re.configuration_flags(mr, links, tpl), v)
        f, s, rec = mr.collide_batch(other=me)
        hit = rec["num_contacts"] > 0
        assert by_pair(*ep) == by_pair(f[hit], s[hit], rec[hit])
        sf, ss = hf.broadphase_config_pairs(mr._boxes, links, tpl)
        srec = mr.scene.engine.batch_collide_objects(mr._handles, mr._tfs, sf, ss)
        shit = srec["num_contacts"] > 0
        assert by_pair(*sp) == by_pair(sf[shit], ss[shit], srec[shit])
        assert len(sp[0]) > 5 and len(ep[0]) > 5 and 0 < v.sum() < len(v)
        with pytest.raises(hf.EngineError, match="invalid argument"):
            re.collide_configurations(mr, links, [(0, 2), (2, 0)])
    return links, robot, env, tpl, v, ep, sp


def link_kind(k, links):
    """0: capsule, 1: box (every third link)"""
    return int((k % links) % 3 == 2)


def test_python_mirror():
    python_mirror(np.random.default_rng(19))
