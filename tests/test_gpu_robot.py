"""The robot model on the device (hfb_robot_*): forward kinematics and motion sampling bit for bit against the host
build of the same arithmetic (tests/emu/kin_emu.cpp), at one configuration and past every grid cap; device sampling
chained into hfb_env_certify_motions_device / hfb_env_collide_motions_device against the host calls fed the host
build's arrays; the geometry lifecycle; and the Python mirror feeding ResidentEnvironment."""
import numpy as np
import pytest

from tests.common import P, hf
from tests.robot_common import emu_poses, emu_sample, link_shapes, local_boxes, random_tree
from tests.test_gpu_env_configs import dev
from tests.test_gpu_env_motions import motion_scene
from hppfcl_b200 import workloads as W

pytestmark = pytest.mark.gpu

LINKS = 16
TPL = W.chain_self_pairs(LINKS)


def create(eng, m):
    return eng.robot_create(m["parent"], m["types"], m["axis"], m["placement"], m["link_joint"], m["link_placement"],
                            m["handles"])


def tree_scene(seed, J, L, world_links=1):
    eng = hf.Engine(0)
    hs = eng.register_shapes(link_shapes())
    eng.commit()
    rng = np.random.default_rng(seed)
    m = random_tree(rng, J, L, hs, world_links)
    return eng, m, local_boxes(eng, m["handles"]), rng


def download(t, dtype):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy().view(dtype)


def empty(nbytes):
    import torch
    return torch.full((max(int(nbytes), 1),), 0xAB, dtype=torch.uint8, device="cuda")


def device_poses(eng, robot, q, L):
    n = q.shape[0]
    d_q = dev(q)
    d_t, d_h = empty(n * L * 96), empty(n * L * 4)
    eng.robot_poses_device(robot, n, d_q.data_ptr(), d_t.data_ptr(), d_h.data_ptr())
    return download(d_t, P.transform_dtype)[:n * L], download(d_h, np.uint32)[:n * L]


def test_fk_parity_one_configuration_and_past_the_grid_caps():
    eng, m, boxes, rng = tree_scene(21, 40, 24, world_links=2)
    r = create(eng, m)
    q = rng.uniform(-3, 3, (1, 40))
    t, h = device_poses(eng, r, q, 24)
    assert t.tobytes() == emu_poses(m, boxes, q).tobytes()
    assert np.array_equal(h, m["handles"])
    th, hh = eng.robot_poses(r, q)  # the host form
    assert th.tobytes() == t.tobytes() and np.array_equal(hh, h)
    # one link on two joints, 2^24 + 5 configurations: more threads than 2^16 blocks of 256
    eng2, m2, boxes2, rng2 = tree_scene(22, 2, 1, world_links=0)
    m2["link_joint"][:] = 1
    r2 = create(eng2, m2)
    n = (1 << 24) + 5
    q2 = rng2.uniform(-4, 4, (n, 2))
    q2[::1000003] = np.nan  # non-finite q propagates
    t2, h2 = device_poses(eng2, r2, q2, 1)
    want = emu_poses(m2, boxes2, q2)
    assert t2.tobytes() == want.tobytes()
    assert (h2 == m2["handles"][0]).all()
    bad = t2[::1000003]
    assert (np.isnan(bad["R"]).any(axis=1) | np.isnan(bad["T"]).any(axis=1)).all()


@pytest.mark.parametrize("seed", range(3))
def test_sampling_parity(seed):
    J, L = [(7, 5), (33, 20), (64, 3)][seed]
    eng, m, boxes, rng = tree_scene(40 + seed, J, L)
    n_samples = rng.integers(0, 40, 300)
    n_samples[:3] = (0, 1, 2)
    off = np.concatenate([[0], np.cumsum(n_samples)]).astype(np.uint32)
    qf = rng.uniform(-3, 3, (300, J))
    qt = qf + rng.uniform(-1, 1, qf.shape)
    r = create(eng, m)
    want = emu_sample(m, boxes, qf, qt, off)
    n = int(off[-1])
    d_qf, d_qt = dev(qf), dev(qt)
    d_t, d_h, d_q, d_s = empty(n * L * 96), empty(n * L * 4), empty(n * J * 8), empty(n * L * 8)
    eng.robot_sample_motions_device(r, off, d_qf.data_ptr(), d_qt.data_ptr(), d_t.data_ptr(), d_h.data_ptr(),
                                    d_q.data_ptr(), d_s.data_ptr())
    got = (download(d_t, P.transform_dtype)[:n * L], download(d_h, np.uint32)[:n * L],
           download(d_q, np.float64)[:n * J].reshape(n, J), download(d_s, np.float64)[:n * L])
    for g, w_ in zip(got, want):
        assert g.tobytes() == w_.tobytes()
    host = eng.robot_sample_motions(r, qf, qt, off, q=True, sweep=True)
    for g, w_ in zip(host, want):
        assert g.tobytes() == w_.tobytes()


@pytest.mark.parametrize("n_motions", [64, 1024])
def test_device_sampling_into_certify_and_collide(n_motions):
    import torch
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = motion_scene(eng, n_motions=n_motions, seed=61)
    m = W.chain_robot_model(w)
    m["handles"] = ha[:LINKS]
    boxes = local_boxes(eng, m["handles"])
    off = w["offsets"]
    r = create(eng, m)
    tfs_e, h_e, _, sw_e = emu_sample(m, boxes, m["q_from"], m["q_to"], off)
    assert np.abs(tfs_e["T"] - tfa["T"]).max() < 1e-9  # the library's samples are robot_motions' up to rounding
    env = eng.env_create(hb, tfb)
    n_cfg = int(off[-1])
    n_a = n_cfg * LINKS
    want_c = eng.env_certify_motions(env, h_e, tfs_e, sw_e, LINKS, TPL, off)
    want_m = eng.env_collide_motions(env, h_e, tfs_e, LINKS, TPL, off)
    d_qf, d_qt = dev(m["q_from"]), dev(m["q_to"])
    d_t, d_h, d_s = empty(n_a * 96), empty(n_a * 4), empty(n_a * 8)
    eng.robot_sample_motions_device(r, off, d_qf.data_ptr(), d_qt.data_ptr(), d_t.data_ptr(), d_h.data_ptr(),
                                    None, d_s.data_ptr())
    n = len(off) - 1
    fi = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    fu = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    cert = torch.full((n_cfg,), 7, dtype=torch.uint8, device="cuda")
    cnt = torch.full((4,), 7, dtype=torch.int32, device="cuda")
    eng.env_certify_motions_device(env, n_a, d_h.data_ptr(), d_t.data_ptr(), d_s.data_ptr(), LINKS, TPL, off,
                                   fi.data_ptr(), fu.data_ptr(), cert.data_ptr(), tuple(cnt[k:].data_ptr() for k in range(4)))
    torch.cuda.synchronize()
    got_c = (fi.cpu().numpy(), fu.cpu().numpy(), cert.cpu().numpy(), tuple(int(c) for c in cnt.cpu().numpy()))
    for k in range(3):
        assert got_c[k].tobytes() == want_c[k].tobytes(), k
    assert got_c[3] == tuple(want_c[3])
    assert (got_c[2] == 1).any()
    mfi = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    kind = torch.full((n,), 7, dtype=torch.int8, device="cuda")
    first = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    second = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    recs = empty(n * P.contact_dtype.itemsize)
    mcnt = torch.full((4,), 7, dtype=torch.int32, device="cuda")
    eng.env_collide_motions_device(env, n_a, d_h.data_ptr(), d_t.data_ptr(), LINKS, TPL, off, mfi.data_ptr(),
                                   kind.data_ptr(), first.data_ptr(), second.data_ptr(), recs.data_ptr(),
                                   tuple(mcnt[k:].data_ptr() for k in range(4)))
    torch.cuda.synchronize()
    assert mfi.cpu().numpy().tobytes() == want_m[0].tobytes()
    assert kind.cpu().numpy().tobytes() == want_m[1].tobytes()
    assert first.cpu().numpy().view(np.uint32).tobytes() == want_m[2].tobytes()
    assert second.cpu().numpy().view(np.uint32).tobytes() == want_m[3].tobytes()
    assert download(recs, P.contact_dtype)[:n].tobytes() == want_m[4].tobytes()
    assert tuple(int(c) for c in mcnt.cpu().numpy()) == tuple(want_m[5])
    eng.env_destroy(env)
    eng.robot_destroy(r)


def test_geometry_lifecycle():
    eng, m, boxes, rng = tree_scene(70, 6, 4)
    r = create(eng, m)
    q = rng.uniform(-1, 1, (3, 6))
    eng.robot_poses(r, q)
    # a geometry changed in place: the sweep bounds follow the committed local boxes
    big = P.make_shapes([P.GEOM_BOX], [[1.0, 1.0, 1.0]])
    eng.update_shapes([m["handles"][0]], big)
    eng.commit()
    off = np.array([0, 3], dtype=np.uint32)
    _, _, _, sw = eng.robot_sample_motions(r, q[:1], q[1:2], off)
    assert sw.tobytes() == emu_sample(m, local_boxes(eng, m["handles"]), q[:1], q[1:2], off)[3].tobytes()
    # a released handle refuses the robot after the next commit
    eng.release_shapes([m["handles"][1]])
    eng.commit()
    with pytest.raises(hf.EngineError):
        eng.robot_poses(r, q)
    with pytest.raises(hf.EngineError):
        create(eng, m)
    eng.robot_destroy(r)
    # after hfb_geom_clear every call on a robot is refused until it is destroyed
    hs = eng.register_shapes(link_shapes())
    eng.commit()
    m["handles"] = hs[:len(m["handles"])]
    r = create(eng, m)
    eng.clear_geometry()
    eng.register_shapes(link_shapes())
    eng.commit()
    with pytest.raises(hf.EngineError):
        eng.robot_poses(r, q)
    with pytest.raises(hf.EngineError):
        eng.robot_sample_motions(r, q[:1], q[1:2], off)
    eng.robot_destroy(r)
    with pytest.raises(hf.EngineError):
        eng.robot_destroy(r)


def test_python_mirror_feeds_the_resident_environment():
    links = [(0, hf.Transform3f(np.eye(3), [0, 0, 0.1]), hf.Box(0.05, 0.05, 0.2)),
             (1, hf.Transform3f(np.eye(3), [0, 0, 0.1]), hf.Capsule(0.03, 0.1)),
             (-1, hf.Transform3f(np.eye(3), [0.5, 0, 0]), hf.Sphere(0.05))]
    joints = [(-1, hf.JOINT_REVOLUTE, [0, 0, 1], hf.Transform3f()),
              (0, hf.JOINT_REVOLUTE, [0, 1, 0], hf.Transform3f(np.eye(3), [0, 0, 0.2]))]
    with hf.RobotModel(joints, links) as robot:
        mgr = hf.DynamicAABBTreeCollisionManager()
        mgr.registerObjects([hf.CollisionObject(hf.Box(0.1, 0.1, 0.1), hf.Transform3f(np.eye(3), [0.2, 0.1, 0.25]))])
        env = hf.ResidentEnvironment(mgr)
        q_from = np.array([[0.0, 0.0], [1.0, -0.5]])
        q_to = np.array([[1.5, 1.0], [-1.0, 0.5]])
        s = robot.sample_motions(q_from, q_to, [0, 20, 45])
        tpl = [(0, 2)]
        got = env.certify_motions(s, 3, tpl, s.offsets, s.sweep)
        want = robot.engine.env_certify_motions(env._env, s.handles, s.tfs, s.sweep, 3, np.array(tpl, dtype=np.uint32),
                                                s.offsets)
        for g, w_ in zip(got, want[:3]):
            assert np.array_equal(g, w_)
        v = env.configuration_flags(robot.poses(s.q), 3, tpl)
        assert np.array_equal(v, env.configuration_flags(s, 3, tpl))
        env.close()
