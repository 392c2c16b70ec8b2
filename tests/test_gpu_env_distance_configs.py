"""Each configuration's clearance (hfb_env_distance_configs*): its nearest pair over the environment pairs and the
template's self pairs.  The ground truth is the composition of existing calls: hfb_env_distance over the range's links,
hfb_batch_distance_objects over the host finder's self pairs (hfb_broadphase_config_distance_pairs), then the argmin the
header defines -- the smallest eligible distance, compared as doubles; on a tie environment pairs first (by link, then
by B index, as hfb_env_distance already orders them), then self pairs in template order.  kind, first, second and
min_distance must match exactly, the records byte for byte, and all three counts."""
import numpy as np
import pytest

from tests.common import P, hf
from tests.test_gpu_edge_inputs import same_fields
from tests.test_gpu_env_configs import LINKS, TPL, config_scene
from tests.test_gpu_env_distance import dev, fresh
from hppfcl_b200 import workloads as W

pytestmark = pytest.mark.gpu

CUTOFFS = (0.0, 0.05, 0.3, np.inf)
NONE = np.uint32(0xFFFFFFFF)


def compose(eng, env, ha, tfa, maxd, tpl=TPL, links=LINKS, g0=0, ng=None, req=None):
    """-> (kind, first, second, min_distance, records, n_env_candidates, n_self_candidates, n_unsupported) from the
    existing calls"""
    n_configs = len(ha) // links
    ng = n_configs - g0 if ng is None else ng
    near, dist, erec, n_env, unsup = eng.env_distance(env, ha, tfa, req, maxd, first_a=g0 * links, num_a=ng * links)
    tpl = np.asarray(tpl, dtype=np.uint32).reshape(-1, 2)
    sf, ss = hf.broadphase_config_distance_pairs(eng.scene_aabbs(ha, tfa), links, tpl, maxd, g0, ng)
    srec = eng.batch_distance_objects(ha, tfa, sf, ss, req) if len(sf) else np.zeros(0, dtype=P.distance_result_dtype)
    sbad = P.status_path(srec["status"]) == P.PATH_UNSUPPORTED
    entry = {(int(i), int(j)): k for k, (i, j) in enumerate(tpl)}
    kind = np.full(n_configs, -1, dtype=np.int8)
    first, second = np.full(n_configs, NONE), np.full(n_configs, NONE)
    rec = fresh(n_configs)
    best = {}  # configuration -> (distance, ordinal, kind, first, second, record)
    for i in np.flatnonzero(near >= 0):
        c = (dist[i], int(i) % links, 0, int(i), int(near[i]), erec[i])
        g = int(i) // links
        if g not in best or c[:2] < best[g][:2]:
            best[g] = c
    for p in np.flatnonzero(~sbad & (srec["min_distance"] <= maxd)):
        a, b = int(sf[p]), int(ss[p])
        g = a // links
        c = (srec["min_distance"][p], links + entry[(a - g * links, b - g * links)], 1, a, b, srec[p])
        if g not in best or c[:2] < best[g][:2]:
            best[g] = c
    for g, c in best.items():
        kind[g], first[g], second[g], rec[g] = c[2], c[3], c[4], c[5]
    return kind, first, second, rec["min_distance"].copy(), rec, n_env, len(sf), unsup + int(sbad.sum())


def assert_same(got, want):
    for k in range(4):
        assert got[k].tobytes() == want[k].tobytes(), k
    if got[4] is not None:
        assert got[4].tobytes() == want[4].tobytes()
    assert got[5:] == want[5:]


@pytest.mark.parametrize("n_env", [500, 100_000])
def test_robot_workload_equals_the_composition(n_env):
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = config_scene(eng, n_configs=256, n_env=n_env, room=3.0 if n_env == 500 else 6.0)
    env = eng.env_create(hb, tfb)
    n_configs = len(ha) // LINKS
    kinds = set()
    for maxd in CUTOFFS:
        want = compose(eng, env, ha, tfa, maxd)
        got = eng.env_distance_configs(env, ha, tfa, LINKS, TPL, max_distance=maxd)
        assert_same(got, want)
        kinds |= set(want[0].tolist())
        if np.isfinite(maxd):
            assert want[6] < n_configs * len(TPL)  # the box test skips self pairs
        else:
            assert want[6] == n_configs * len(TPL) and (want[0] >= 0).all()
        # clearance: the distances alone
        assert eng.env_distance_configs(env, ha, tfa, LINKS, TPL, max_distance=maxd, records=False)[3].tobytes() == \
            want[3].tobytes()
        # ranges: outside its range a configuration gets the no-winner values
        for g0, ng in ((0, 37), (37, 1), (38, 0), (38, n_configs - 38)):
            r = eng.env_distance_configs(env, ha, tfa, LINKS, TPL, max_distance=maxd, first_config=g0, num_configs=ng)
            assert_same(r, compose(eng, env, ha, tfa, maxd, g0=g0, ng=ng))
    # environment winners and self winners (some of them penetrating) occur, and among the sparse environment also
    # configurations with none
    assert kinds == ({-1, 0, 1} if n_env == 500 else {0, 1}) or kinds == {-1, 0, 1}
    want = compose(eng, env, ha, tfa, np.inf)
    assert ((want[0] == 1) & (want[3] < 0)).any()


def test_empty_env_empty_template_and_no_eligible_pair():
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = config_scene(eng, n_configs=64)
    env = eng.env_create(hb, tfb)
    empty = eng.env_create(hb[:0], tfb[:0])
    for maxd in (0.05, np.inf):
        got = eng.env_distance_configs(empty, ha, tfa, LINKS, TPL, max_distance=maxd)  # the self pairs alone
        assert_same(got, compose(eng, empty, ha, tfa, maxd))
        assert got[5] == 0 and set(got[0].tolist()) <= {-1, 1} and (got[0] == 1).any()
        no_tpl = np.zeros((0, 2), np.uint32)
        got = eng.env_distance_configs(env, ha, tfa, LINKS, no_tpl, max_distance=maxd)  # the environment alone
        assert_same(got, compose(eng, env, ha, tfa, maxd, tpl=no_tpl))
        assert got[6] == 0 and set(got[0].tolist()) <= {-1, 0}
    got = eng.env_distance_configs(empty, ha, tfa, LINKS, np.zeros((0, 2), np.uint32))
    assert (got[0] == -1).all() and (got[1] == NONE).all() and (got[2] == NONE).all()
    assert got[4].tobytes() == fresh(len(got[0])).tobytes() and got[5:] == (0, 0, 0)
    # no A objects at all
    got = eng.env_distance_configs(env, ha[:0], tfa[:0], LINKS, TPL)
    assert len(got[0]) == 0 and got[5:] == (0, 0, 0)
    # refusals: a malformed template or range, a bad cutoff
    for tpl in ([(0, LINKS)], [(2, 2)], [(0, 2), (2, 0)]):
        with pytest.raises(hf.EngineError, match="invalid argument"):
            eng.env_distance_configs(env, ha, tfa, LINKS, tpl)
    with pytest.raises(hf.EngineError, match="invalid argument"):
        eng.env_distance_configs(env, ha[:-1], tfa[:-1], LINKS, TPL)
    with pytest.raises(hf.EngineError, match="invalid argument"):
        eng.env_distance_configs(env, ha, tfa, LINKS, TPL, first_config=60, num_configs=5)


def obb_scene(eng):
    """two configurations of 3 links: a sphere, a plain BVHModel<OBB> (never eligible) and a box; B: one sphere"""
    rng = np.random.default_rng(5)
    sph, box = (int(x) for x in eng.register_shapes(P.make_shapes([P.GEOM_SPHERE, P.GEOM_BOX], [[0.2, 0, 0], [0.1, 0.1, 0.1]])))
    verts, tris = W.sphere_mesh(0.3, 12, 6, noise=0.02, rng=rng)
    nodes = hf.build_bvh_obbrss(verts, tris)
    obb = int(eng.register_shapes(P.make_shapes([P.BV_OBB], [[0, 0, 0]], data=[eng.register_bvh_obb(nodes, verts, tris)]))[0])
    eng.commit()
    ha = np.array([sph, obb, box] * 2, dtype=np.uint32)
    tfa = W.identity_transforms(6, T=[[0, 0, 0], [0.45, 0, 0], [5, 0, 0], [0, 3, 0], [0.2, 3, 0], [0, 3.5, 0]])
    hb = np.array([sph], dtype=np.uint32)
    tfb = W.identity_transforms(1, T=[[0.3, 1.0, 0]])
    return ha, tfa, hb, tfb


def test_plain_obb_link_and_nonfinite_poses():
    eng = hf.Engine(0)
    ha, tfa, hb, tfb = obb_scene(eng)
    env = eng.env_create(hb, tfb)
    tpl = [(0, 1), (1, 2), (0, 2)]
    for maxd in (0.05, 1.0, np.inf):
        got = eng.env_distance_configs(env, ha, tfa, 3, tpl, max_distance=maxd)
        want = compose(eng, env, ha, tfa, maxd, tpl=tpl, links=3)
        assert_same(got, want)
        assert 1 not in got[1] and 4 not in got[1] and 1 not in got[2][got[0] == 1]  # the OBB link never wins
        assert got[7] >= 1  # its pairs came back unsupported
    # NaN, infinite and far poses: each decided as the composition decides it
    bad = tfa.copy()
    bad["T"][0] = np.nan
    bad["R"][3, 0] = np.nan
    bad["T"][5, 1] = np.inf
    for maxd in (0.05, np.inf):
        got = eng.env_distance_configs(env, ha, bad, 3, tpl, max_distance=maxd)
        assert_same(got, compose(eng, env, ha, bad, maxd, tpl=tpl, links=3))
    for shift in (1e6, 1e100):
        ta, tb = tfa.copy(), tfb.copy()
        ta["T"] += shift
        tb["T"] += shift
        e3 = eng.env_create(hb, tb)
        for maxd in (0.05, np.inf):
            assert_same(eng.env_distance_configs(e3, ha, ta, 3, tpl, max_distance=maxd),
                        compose(eng, e3, ha, ta, maxd, tpl=tpl, links=3))
        eng.env_destroy(e3)


def test_ties_between_kinds_and_template_entries():
    """spheres on a line at exact binary distances: an environment pair and a self pair at the same distance (the
    environment wins), two self pairs at the same distance (the earlier template entry wins)"""
    eng = hf.Engine(0)
    sph = int(eng.register_shapes(P.make_shapes([P.GEOM_SPHERE], [[0.25, 0, 0]]))[0])
    eng.commit()
    ha = np.full(3, sph, dtype=np.uint32)
    tfa = W.identity_transforms(3, T=[[0, 0, 0], [1.0, 0, 0], [-1.0, 0, 0]])  # links 1 and 2 both 0.5 from link 0
    hb = np.full(1, sph, dtype=np.uint32)
    env = eng.env_create(hb, W.identity_transforms(1, T=[[0, 1.0, 0]]))  # 0.5 from link 0 too
    far = eng.env_create(hb, W.identity_transforms(1, T=[[0, 10.0, 0]]))
    for tpl, e, want_kind, want_pair in (([(0, 1), (0, 2)], env, 0, (0, 0)), ([(0, 1), (0, 2)], far, 1, (0, 1)),
                                         ([(0, 2), (0, 1)], far, 1, (0, 2)), ([(2, 0), (1, 0)], far, 1, (2, 0))):
        got = eng.env_distance_configs(e, ha, tfa, 3, tpl)
        assert_same(got, compose(eng, e, ha, tfa, np.inf, tpl=tpl, links=3))
        assert got[3][0] == 0.5 and got[0][0] == want_kind and (got[1][0], got[2][0]) == want_pair


def test_after_update():
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = config_scene(eng, n_configs=64, n_env=2000)
    env = eng.env_create(hb, tfb)
    rng = np.random.default_rng(9)
    idx = rng.choice(len(hb), 400, replace=False).astype(np.uint32)
    t2 = tfb.copy()
    t2["T"][idx] += rng.uniform(-0.4, 0.4, (len(idx), 3))
    eng.env_update(env, idx, t2[idx])
    ref = eng.env_create(hb, t2)
    for maxd in (0.05, np.inf):
        got = eng.env_distance_configs(env, ha, tfa, LINKS, TPL, max_distance=maxd)
        assert_same(got, compose(eng, ref, ha, tfa, maxd))


def test_device_form_and_unsynchronised_host_calls():
    """the device form equals the host form; a device call on a side stream followed by host env calls on the same
    context on another stream, with no synchronisation in between: both results as each call alone gives them"""
    import torch
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = config_scene(eng, n_configs=128, n_env=2000)
    env = eng.env_create(hb, tfb)
    n, nc = len(ha), len(ha) // LINKS
    t_other = tfa.copy()
    t_other["T"] += 0.2
    d_h, d_t = dev(ha), dev(tfa)
    d_kind = torch.zeros(nc, dtype=torch.int8, device="cuda")
    d_first = torch.zeros(nc, dtype=torch.int32, device="cuda")
    d_second = torch.zeros(nc, dtype=torch.int32, device="cuda")
    d_min = torch.zeros(nc, dtype=torch.float64, device="cuda")
    d_rec = torch.zeros(nc * P.distance_result_dtype.itemsize, dtype=torch.uint8, device="cuda")
    d_cnt = torch.zeros(3, dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()

    def run(maxd, g0=0, ng=None):
        eng.env_distance_configs_device(env, n, d_h.data_ptr(), d_t.data_ptr(), LINKS, TPL, d_kind.data_ptr(),
                                        d_first.data_ptr(), d_second.data_ptr(), d_min.data_ptr(), d_rec.data_ptr(),
                                        d_cnt.data_ptr(), d_cnt.data_ptr() + 4, d_cnt.data_ptr() + 8, max_distance=maxd,
                                        stream=side.cuda_stream, first_config=g0, num_configs=ng)

    def fetch():
        side.synchronize()
        c = d_cnt.cpu().numpy()
        return (d_kind.cpu().numpy(), d_first.cpu().numpy().view(np.uint32), d_second.cpu().numpy().view(np.uint32),
                d_min.cpu().numpy(), d_rec.cpu().numpy().view(P.distance_result_dtype), int(c[0]), int(c[1]), int(c[2]))

    torch.cuda.synchronize()
    for maxd, g0, ng in ((0.05, 0, None), (np.inf, 0, None), (0.3, 40, 50)):
        want = eng.env_distance_configs(env, ha, tfa, LINKS, TPL, max_distance=maxd, first_config=g0, num_configs=ng)
        run(maxd, g0, ng)
        assert_same(fetch(), want)
    want_dev = eng.env_distance_configs(env, ha, tfa, LINKS, TPL, max_distance=0.3)
    want_cfg = eng.env_distance_configs(env, ha, t_other, LINKS, TPL, max_distance=np.inf)
    want_dist = eng.env_distance(env, ha, t_other, max_distance=np.inf)
    for host_call, want in ((lambda: eng.env_distance_configs(env, ha, t_other, LINKS, TPL, max_distance=np.inf), want_cfg),
                            (lambda: eng.env_distance(env, ha, t_other, max_distance=np.inf), want_dist)):
        run(0.3)
        got = host_call()  # no synchronisation in between
        for a, b in zip(got, want):
            assert (a.tobytes() == b.tobytes()) if isinstance(a, np.ndarray) else a == b
        assert_same(fetch(), want_dev)
    assert eng.stats()["watchdog_trips"] == 0


def test_python_mirror():
    """ResidentEnvironment.distance_configurations / configuration_clearance on managers: the composition over the
    managers' tables; a bad cutoff or template raises ValueError"""
    eng_scene = hf.DynamicAABBTreeCollisionManager()
    rng = np.random.default_rng(23)
    geoms = [hf.Box(0.3, 0.2, 0.4), hf.Sphere(0.15), hf.Capsule(0.1, 0.3)]
    links = 5

    def pose(c):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        return hf.Transform3f.from_quat(*q, T=c + rng.uniform(-0.4, 0.4, 3))

    robot = [hf.CollisionObject(geoms[i % 3], pose(np.array([i // links, 0.0, 0.0]) * 1.5)) for i in range(40)]
    env_objs = [hf.CollisionObject(hf.Halfspace(np.array([0.0, 0, 1]), -0.8))]
    env_objs += [hf.CollisionObject(geoms[i % 3], pose(rng.uniform(-1, 12, 3) * [1, 0.3, 0.3])) for i in range(200)]
    mr = hf.DynamicAABBTreeCollisionManager()
    mr.registerObjects(robot)
    eng_scene.registerObjects(env_objs)
    mr.setup()
    eng_scene.setup()
    tpl = W.chain_self_pairs(links, 2)
    with hf.ResidentEnvironment(eng_scene) as re:
        eng = re.engine
        env = eng.env_create(eng_scene._handles, eng_scene._tfs)
        for maxd in (0.2, np.inf):
            got = re.distance_configurations(mr, links, tpl, max_distance=maxd)
            want = compose(eng, env, mr._handles, mr._tfs, maxd, tpl=tpl, links=links)
            assert_same(tuple(got) + want[5:], want)
            assert re.configuration_clearance(mr, links, tpl, maxd).tobytes() == want[3].tobytes()
        for bad in (np.nan, -0.1):
            with pytest.raises(ValueError):
                re.distance_configurations(mr, links, tpl, max_distance=bad)
        for bad_tpl in ([(0, links)], [(1, 1)], [(0, 2), (2, 0)]):
            with pytest.raises(ValueError):
                re.configuration_clearance(mr, links, bad_tpl)
        eng.env_destroy(env)


def test_winners_equal_the_reference():
    """the sample of tests/test_env_distance_configs_reference.py: the device finds the oracle's winners at every cutoff,
    and their records equal the oracle's, which equal the reference build's (its recorded outputs where it is not built
    here)"""
    from tests.common import make_scenes
    from tests.test_env_distance_configs_reference import load_recorded, reference_sample
    from tests.test_env_distance_reference import assert_fields
    load_recorded()
    sc = make_scenes(gpu=True, emu=False, ref=True)
    eng = sc.b["gpu"]
    scenes, args, orec = reference_sample(sc)
    rr = sc.b["ref"].batch_distance(*args)
    assert_fields(rr, orec, "oracle winners against the reference build")
    for ha, tfa, hb, tfb, links, tpl, win in scenes:
        env = eng.env_create(hb, tfb)
        for maxd, (kind, first, second) in win.items():
            got = eng.env_distance_configs(env, ha, tfa, links, tpl, max_distance=maxd)
            assert got[0].tobytes() == kind.tobytes() and got[1].tobytes() == first.tobytes()
            assert got[2].tobytes() == second.tobytes()
            for c in np.flatnonzero(kind >= 0):
                other = (hb, tfb) if kind[c] == 0 else (ha, tfa)
                one = sc.b["oracle"].batch_distance(ha[first[c]:first[c] + 1], tfa[first[c]:first[c] + 1],
                                                    other[0][second[c]:second[c] + 1], other[1][second[c]:second[c] + 1],
                                                    nthreads=0)
                assert got[4][c:c + 1].tobytes() == one.tobytes()
        eng.env_destroy(env)
    # non-finite and far poses of the robot scene against the oracle's winners
    ha, tfa, hb, tfb, links, tpl, _ = scenes[0]
    env = eng.env_create(hb, tfb)
    bad = tfa.copy()
    bad["T"][3] = np.nan
    bad["R"][21, 0] = np.nan
    bad["T"][40, 1] = np.inf
    bad["T"][64:80] += 1e100
    from tests.test_env_distance_configs_reference import oracle_winners
    for maxd in (0.05, np.inf):
        kind, first, second, rec = oracle_winners(sc.b["oracle"], ha, bad, hb, tfb, links, tpl, maxd)
        got = eng.env_distance_configs(env, ha, bad, links, tpl, max_distance=maxd)
        assert got[0].tobytes() == kind.tobytes() and got[1].tobytes() == first.tobytes()
        assert got[2].tobytes() == second.tobytes()
        # (the records as the oracle's, a NaN equal to a NaN whatever its sign bit, as tests/test_gpu_edge_inputs.py
        # compares non-finite inputs)
        same_fields(got[4][kind >= 0], rec[kind >= 0], P.distance_result_dtype.names, "non-finite and far poses")
    eng.env_destroy(env)
