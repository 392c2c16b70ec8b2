"""hfb_env_validate_motions on the device against its contract (tests/validate_common.py): the hand scene against the
CPU narrow phase; robot_motions' chain at room scales 16 and 32 against validate_reference driven by the library's
existing public calls (bit for bit, round and sample counts included); D = d0 against one sampling and certification;
soundness by dense resampling; the witness against hfb_env_collide_motions; range splits; the device form; an env
update; and refusals that write nothing."""
import numpy as np
import pytest

from tests.common import P, hf, make_scenes
from tests.robot_common import local_boxes
from tests.test_gpu_env_configs import dev
from tests.test_gpu_env_motions import LINKS, motion_scene
from tests.test_gpu_robot import download, empty
from tests.validate_common import cpu_narrow, effective_cap, hand_scene, q_at, run_layout, sweeps_of, validate_reference
from hppfcl_b200 import workloads as W

pytestmark = pytest.mark.gpu

TPL = W.chain_self_pairs(LINKS)
FIELDS = ("status", "t_valid", "t_collide", "n_rounds", "n_samples", "n_env_candidates", "n_self_candidates",
          "n_unsupported")


def create(eng, m):
    return eng.robot_create(m["parent"], m["types"], m["axis"], m["placement"], m["link_joint"], m["link_placement"],
                            m["handles"])


def assert_same(got, want, fields=FIELDS):
    for f in fields:
        g, w = np.asarray(got[f]), np.asarray(want[f])
        assert g.tobytes() == w.tobytes(), "%s differs: %s vs %s" % (f, g, w)


def library_narrow(eng, env, robot, tpl, q_from, q_to, D, req):
    """the narrow phase from the library's existing public calls: host-computed q at the run samples, hfb_robot_poses,
    hfb_robot_sample_motions over 2-sample motions for the sweeps, then hfb_env_certify_motions"""
    J, L = eng.robot_dims(robot)

    def narrow(depth, runs):
        qs, off, qa, qb = run_layout(runs, q_from, q_to, D)
        tfa, ha = eng.robot_poses(robot, qs)
        sweep, fin = sweeps_of(lambda a, b, o: eng.robot_sample_motions(robot, a, b, o)[3], runs, qa, qb, L)
        fi, _, cert, cnt = eng.env_certify_motions(env, ha, tfa, sweep, L, tpl, off, req)
        return fi, [cert[off[r]:off[r + 1] - 1] for r in range(len(runs))], fin, cnt[:3]
    return narrow


def test_hand_scene_matches_the_cpu_reference():
    sc = make_scenes(gpu=True, emu=True)
    model, hb, tfb, q0, q1, names = hand_scene(sc)
    sc.commit()
    eng, orc, emu = sc.b["gpu"], sc.b["oracle"], sc.b["emu"]
    boxes = local_boxes(emu, model["handles"])
    env = eng.env_create(hb, tfb)
    robot = create(eng, model)
    for margin, d0, D, cap in ((0.0, 1, 6, 1 << 20), (0.3, 2, 5, 1 << 20), (0.0, 2, 4, 7), (-np.inf, 1, 6, 1 << 20)):
        req = P.CollisionRequestPOD()
        req.security_margin = margin
        want = validate_reference(cpu_narrow(orc, emu, model, boxes, hb, tfb, [(0, 1)], q0, q1, D, req), len(q0), d0, D,
                                  effective_cap(cap, len(hb), 2))
        got = eng.env_validate_motions(env, robot, q0, q1, [(0, 1)], d0, D, cap, req)
        assert_same(got, want)


def chain_scene(room, n_motions=1024):
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = motion_scene(eng, n_motions, room=room)
    m = W.chain_robot_model(w)
    m["handles"] = ha[:LINKS]
    env = eng.env_create(hb, tfb)
    return eng, env, create(eng, m), m, hb, tfb


@pytest.mark.parametrize("room", [16.0, 32.0])
def test_chain_matches_the_composition_of_existing_calls(room):
    eng, env, robot, m, hb, tfb = chain_scene(room)
    q0, q1 = m["q_from"], m["q_to"]
    req = P.CollisionRequestPOD()
    for d0 in (2, 4):
        D = d0 + 8
        want = validate_reference(library_narrow(eng, env, robot, TPL, q0, q1, D, req), len(q0), d0, D,
                                  effective_cap(1 << 40, len(hb), LINKS))
        got = eng.env_validate_motions(env, robot, q0, q1, TPL, d0, D, 1 << 40, req)
        assert_same(got, want)
        # D = d0: one sampling of 2^d0 + 1 samples and one certification
        n = 1 << d0
        off = np.arange(0, (n + 1) * len(q0) + 1, n + 1, dtype=np.uint32)
        tfa, ha, _, sw = eng.robot_sample_motions(robot, q0, q1, off)
        fi, fu, _, _ = eng.env_certify_motions(env, ha, tfa, sw, LINKS, TPL, off, req)
        one = eng.env_validate_motions(env, robot, q0, q1, TPL, d0, d0, 1 << 40, req)
        assert np.array_equal(one["t_collide"], np.where(fi >= 0, fi / float(n), -1.0))
        assert np.array_equal(one["t_valid"], np.where(fu >= 0, fu / float(n), 1.0))
        # a deeper D never shortens the certified prefix (the cap does not bind)
        deeper = eng.env_validate_motions(env, robot, q0, q1, TPL, d0, D + 2, 1 << 40, req)
        assert (deeper["t_valid"] >= got["t_valid"]).all()
        # the witness is hfb_env_collide_motions' at q(t_collide)
        hit = np.flatnonzero(got["status"] == 1)
        c = [want["c"][k] for k in hit]
        qs = np.array([q_at(q0[k], q1[k], ck, D) for k, ck in zip(hit, c)]).reshape(-1, q0.shape[1])
        tfa, ha = eng.robot_poses(robot, qs)
        fi, kind, first, second, rec, _ = eng.env_collide_motions(env, ha, tfa, LINKS, TPL,
                                                                  np.arange(len(hit) + 1, dtype=np.uint32), req)
        assert (fi == 0).all()
        base = np.arange(len(hit), dtype=np.uint32) * LINKS
        assert np.array_equal(got["kind"][hit], kind)
        assert np.array_equal(got["first"][hit], first - base)
        assert np.array_equal(got["second"][hit], np.where(kind == 0, second, second - base))
        assert got["contacts"][hit].tobytes() == rec.tobytes()
        assert (got["kind"][got["status"] != 1] == -1).all()


def test_soundness_range_split_device_form_and_update():
    eng, env, robot, m, hb, tfb = chain_scene(16.0, 256)
    q0, q1 = m["q_from"], m["q_to"]
    req = P.CollisionRequestPOD()
    d0, D = 2, 9
    got = eng.env_validate_motions(env, robot, q0, q1, TPL, d0, D, 1 << 40, req)
    # soundness: [0, t_valid] resampled densely has no colliding configuration; a configuration collides at t_collide
    qs, owner = [], []
    for k in np.flatnonzero(got["t_valid"] > 0):  # (t_valid = 0: an empty prefix)
        for t in np.linspace(0.0, got["t_valid"][k], 33):
            qs.append(q0[k] + t * (q1[k] - q0[k]))
            owner.append(k)
    tfa, ha = eng.robot_poses(robot, np.array(qs))
    verdicts = eng.env_collide_configs(env, ha, tfa, LINKS, TPL, req, 0, 0)[0]
    assert not verdicts.any(), "a sample inside a certified prefix collides"
    hit = np.flatnonzero(got["status"] == 1)
    qc = np.array([q_at(q0[k], q1[k], int(round(got["t_collide"][k] * (1 << D))), D) for k in hit])
    tfa, ha = eng.robot_poses(robot, qc)
    assert eng.env_collide_configs(env, ha, tfa, LINKS, TPL, req, 0, 0)[0].all()
    # a range split gives the same per-motion results
    a = eng.env_validate_motions(env, robot, q0, q1, TPL, d0, D, 1 << 40, req, first_motion=0, num_motions=100)
    b = eng.env_validate_motions(env, robot, q0, q1, TPL, d0, D, 1 << 40, req, first_motion=100, num_motions=156)
    for f in ("status", "t_valid", "t_collide", "kind", "first", "second"):
        assert np.array_equal(np.concatenate([a[f][:100], b[f][100:]]), got[f])
    assert (a["status"][100:] == -1).all() and (b["status"][:100] == -1).all()
    # the device form equals the host form
    n = len(q0)
    bufs = [empty(n), empty(8 * n), empty(8 * n), empty(n), empty(4 * n), empty(4 * n),
            empty(P.contact_dtype.itemsize * n), empty(4), empty(8), empty(8), empty(8), empty(8)]
    d_q0, d_q1 = dev(q0), dev(q1)
    eng.env_validate_motions_device(env, robot, n, d_q0.data_ptr(), d_q1.data_ptr(), TPL, d0, D, 1 << 40,
                                    *[x.data_ptr() for x in bufs[:7]], d_counts=[x.data_ptr() for x in bufs[7:]],
                                    req=req)
    dt = [np.int8, np.float64, np.float64, np.int8, np.uint32, np.uint32, P.contact_dtype]
    for f, x, t in zip(("status", "t_valid", "t_collide", "kind", "first", "second", "contacts"), bufs, dt):
        assert download(x, t)[:n].tobytes() == np.asarray(got[f]).tobytes(), f
    cn = [int(download(bufs[7], np.uint32)[0])] + [int(download(x, np.uint64)[0]) for x in bufs[8:]]
    assert cn == [got[f] for f in ("n_rounds", "n_samples", "n_env_candidates", "n_self_candidates", "n_unsupported")]
    # after an env update the results follow the composition again
    idx = np.arange(0, len(hb) - 1, 7, dtype=np.uint32)
    tf = tfb[idx].copy()
    tf["T"][:, 2] += 0.3
    eng.env_update(env, idx, tf)
    want = validate_reference(library_narrow(eng, env, robot, TPL, q0, q1, D, req), n, d0, D,
                              effective_cap(1 << 40, len(hb), LINKS))
    assert_same(eng.env_validate_motions(env, robot, q0, q1, TPL, d0, D, 1 << 40, req), want)
    # a refused call writes nothing, in either form
    for bad in ((3, 2, 100), (2, 31, 100), (2, 9, 1)):
        for x in bufs:
            x.fill_(0xAB)
        with pytest.raises(Exception):
            eng.env_validate_motions_device(env, robot, n, d_q0.data_ptr(), d_q1.data_ptr(), TPL, *bad,
                                            *[x.data_ptr() for x in bufs[:7]],
                                            d_counts=[x.data_ptr() for x in bufs[7:]], req=req)
        assert all((download(x, np.uint8) == 0xAB).all() for x in bufs)
    with pytest.raises(Exception):
        eng.env_validate_motions(env, robot, q0, q1, [(0, LINKS)], d0, D, 100, req)


def test_refusals_write_nothing_and_follow_the_robot():
    import ctypes as C
    sc = make_scenes(gpu=True, emu=False)
    model, hb, tfb, q0, q1, names = hand_scene(sc)
    sc.commit()
    eng = sc.b["gpu"]
    env = eng.env_create(hb, tfb)
    robot = create(eng, model)
    n = len(q0)
    qf, qt = np.ascontiguousarray(q0), np.ascontiguousarray(q1)
    req = P.CollisionRequestPOD()

    def call(tpl, p):
        """the host form straight through the ABI, into caller buffers filled with a pattern -> (rc, the buffers)"""
        bufs = [np.full(n, 0x55, np.int8), np.full(n, 7.0), np.full(n, 7.0), np.full(n, 0x55, np.int8),
                np.full(n, 0x5555, np.uint32), np.full(n, 0x5555, np.uint32),
                np.frombuffer(b"\x55" * (P.contact_dtype.itemsize * n), dtype=P.contact_dtype).copy(),
                np.full(1, 0x5555, np.uint32)] + [np.full(1, 0x5555, np.uint64) for _ in range(4)]
        out = P.ValidateOut(*[b.ctypes.data for b in bufs])
        t = np.ascontiguousarray(tpl, dtype=np.uint32).reshape(-1, 2)
        rc = eng.L.hfb_env_validate_motions(eng.h, env, robot, n, qf.ctypes.data, qt.ctypes.data, t.shape[0],
                                            t.ctypes.data, 0, n, C.byref(req), C.byref(P.ValidateParams(*p)),
                                            C.byref(out))
        return rc, bufs

    rc, bufs = call([(0, 1)], (1, 4, 100))
    assert rc == 0 and bufs[0][0] == 0
    pristine = call([(0, 1)], (5, 4, 100))[1]  # refused before the context is read
    for tpl, p in (([(0, 2)], (1, 4, 100)), ([(0, 0)], (1, 4, 100)), ([(0, 1)], (5, 4, 100)), ([(0, 1)], (1, 31, 100)),
                   ([(0, 1)], (1, 4, 1))):
        rc, bufs = call(tpl, p)
        assert rc != 0
        assert all(b.tobytes() == w.tobytes() for b, w in zip(bufs, pristine)), "a refused call wrote its outputs"
    # a link's shape released: the robot is refused after the next commit; after hfb_geom_clear every call is
    eng.release_shapes([model["handles"][1]])
    eng.commit()
    rc, bufs = call([(0, 1)], (1, 4, 100))
    assert rc != 0 and all(b.tobytes() == w.tobytes() for b, w in zip(bufs, pristine))
    eng.clear_geometry()
    rc, bufs = call([(0, 1)], (1, 4, 100))
    assert rc != 0 and all(b.tobytes() == w.tobytes() for b, w in zip(bufs, pristine))


def test_python_mirror_on_real_data():
    """ResidentEnvironment.validate_motions / MotionValidation give what the engine call gives"""
    up = hf.Transform3f(np.eye(3), [0, 0, 0.1])
    joints = [(-1, hf.JOINT_REVOLUTE, [0, 0, 1], hf.Transform3f()),
              (0, hf.JOINT_REVOLUTE, [0, 1, 0], hf.Transform3f(np.eye(3), [0, 0, 0.2]))]
    links = [(0, up, hf.Box(0.05, 0.05, 0.2)), (1, up, hf.Capsule(0.03, 0.1))]
    q0 = np.array([[0.0, 0.0], [1.0, -0.5], [-2.0, 0.3]])
    q1 = np.array([[1.5, 1.0], [-1.0, 0.5], [2.0, 0.3]])
    with hf.RobotModel(joints, links) as robot:
        mgr = hf.DynamicAABBTreeCollisionManager()
        mgr.registerObjects([hf.CollisionObject(hf.Box(0.1, 0.1, 0.1), hf.Transform3f(np.eye(3), [0.2, 0.1, 0.25]))])
        with hf.ResidentEnvironment(mgr) as env:
            v = env.validate_motions(robot, q0, q1, [], initial_depth=1, max_depth=7, max_samples=1 << 20)
            r = env.engine.env_validate_motions(env._env, robot._robot, q0, q1, np.zeros((0, 2), np.uint32), 1, 7,
                                                1 << 20)
    for f in r:
        assert np.asarray(getattr(v, f)).tobytes() == np.asarray(r[f]).tobytes(), f
    assert set(v.status.tolist()) <= {0, 1, 2} and v.n_rounds >= 1
