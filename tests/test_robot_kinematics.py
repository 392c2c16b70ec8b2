"""The robot-model kinematics (csrc/hfb_kin.cuh) in their host build (tests/emu/kin_emu.cpp), without a GPU: hfb_sincos
against numpy, forward kinematics against a numpy restatement of the header's semantics on the chain model and on
seeded random trees, the chain model against workloads.robot_motions, the sampling rule's end points, and the sweep
bounds' soundness (no corner of a link's local box travels farther than its bound over a densely resampled segment)."""
import numpy as np
import pytest

from tests.common import EmuScene, P
from tests.robot_common import (chain_model, depth, emu_poses, emu_sample, link_shapes, local_boxes, np_poses,
                                random_tree, sincos)
from hppfcl_b200 import workloads as W

EPS = np.finfo(np.float64).eps


def ulps(a, b):
    """distance in units in the last place of b"""
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(b), np.finfo(np.float64).tiny))


def test_sincos_within_one_ulp():
    rng = np.random.default_rng(11)
    lim = np.nextafter(2.0 ** 20 * np.pi / 2, 0)
    x = np.concatenate([rng.uniform(-4, 4, 200_000), rng.uniform(-100, 100, 100_000), rng.uniform(-lim, lim, 100_000),
                        np.arange(-64, 65) * (np.pi / 4), np.arange(-64, 65) * (np.pi / 2), [1e-300, -1e-300, 1e-9, 0.3,
                        np.nextafter(np.pi / 4, 0), np.pi / 4, np.nextafter(lim, 0)],
                        rng.uniform(-1e-8, 1e-8, 1000)])
    s, c = sincos(x)
    assert ulps(s, np.sin(x)).max() <= 1.0
    assert ulps(c, np.cos(x)).max() <= 1.0
    s, c = sincos(np.array([0.0, -0.0]))
    assert s[0] == 0 and not np.signbit(s[0]) and s[1] == 0 and np.signbit(s[1]) and (c == 1).all()
    s, c = sincos(np.array([np.nan, np.inf, -np.inf, 1e7, -1.65e6]))
    assert np.isnan(s).all() and np.isnan(c).all()  # non-finite, and past the reduction's range


def emu_tree_scene(rng, n_joints, n_links, world_links=1):
    emu = EmuScene()
    hs = emu.register_shapes(link_shapes())
    m = random_tree(rng, n_joints, n_links, hs, world_links)
    return m, local_boxes(emu, m["handles"])


@pytest.mark.parametrize("seed", range(6))
def test_fk_matches_numpy_on_random_trees(seed):
    rng = np.random.default_rng(100 + seed)
    J = int(rng.integers(1, 65))
    m, boxes = emu_tree_scene(rng, J, int(rng.integers(1, 40)), world_links=int(rng.integers(0, 3)))
    q = rng.uniform(-3, 3, (64, J))
    got = emu_poses(m, boxes, q)
    R, T = np_poses(m, q)
    d = np.maximum(depth(m), 1)
    L = len(m["link_joint"])
    gR = got["R"].reshape(64, L, 3, 3).transpose(0, 1, 3, 2)
    gT = got["T"].reshape(64, L, 3)
    scale = 1.0 + np.abs(T).max()
    assert (np.abs(gR - R).max(axis=(2, 3)) <= 16 * EPS * d).all()
    assert (np.abs(gT - T).max(axis=2) <= 16 * EPS * d * scale).all()


def test_chain_model_reproduces_robot_motions():
    w = W.robot_motions(16, n_env=200, room=3.0, seed=3)
    emu = EmuScene()
    m = chain_model(w, w["register"](emu))
    assert len(m["parent"]) == w["n_links"] + 2
    got = emu_poses(m, local_boxes(emu, m["handles"]), m["q"])
    assert np.abs(got["R"] - w["tf_a"]["R"]).max() <= 1e-12
    assert np.abs(got["T"] - w["tf_a"]["T"]).max() <= 1e-12
    R, T = np_poses(m, m["q"][:50])
    assert np.abs(R.transpose(0, 1, 3, 2).reshape(-1, 9) - got["R"][:50 * w["n_links"]]).max() <= 1e-12


def test_sampling_end_points_are_exact():
    rng = np.random.default_rng(7)
    m, boxes = emu_tree_scene(rng, 9, 5)
    J = 9
    n_samples = np.array([5, 1, 0, 2, 17, 0, 3])
    off = np.concatenate([[0], np.cumsum(n_samples)]).astype(np.uint32)
    qf = rng.uniform(-2, 2, (len(n_samples), J))
    qt = qf + rng.uniform(-0.3, 0.3, qf.shape) * rng.random(qf.shape) ** 3
    tfs, h, q, sw = emu_sample(m, boxes, qf, qt, off)
    for k, n in enumerate(n_samples):
        if n == 0:
            continue
        assert q[off[k]].tobytes() == qf[k].tobytes()
        if n > 1:
            assert q[off[k + 1] - 1].tobytes() == qt[k].tobytes()
            t = np.arange(n) / (n - 1.0)
            assert np.array_equal(q[off[k] + 1:off[k + 1] - 1], (qf[k] + t[1:-1, None] * (qt[k] - qf[k])))
        assert (sw.reshape(-1, 5)[off[k + 1] - 1] == 0).all()  # a motion's last sample
    assert (sw.reshape(-1, 5)[:, np.asarray(m["link_joint"]) < 0] == 0).all()  # links fixed to the world
    assert np.array_equal(tfs.tobytes(), emu_poses(m, boxes, q).tobytes())  # the samples' poses are poses(q)


def corners(boxes):
    b = np.asarray(boxes).reshape(-1, 6)
    idx = np.array([[i, j, k] for i in (0, 3) for j in (1, 4) for k in (2, 5)])
    return b[:, idx]  # (L, 8, 3)


def world_points(tfs, pts):
    R = tfs["R"].reshape(-1, 3, 3).transpose(0, 2, 1)
    return np.einsum("lij,lkj->lki", R, pts) + tfs["T"][:, None, :]


@pytest.mark.parametrize("seed", range(4))
def test_sweep_bounds_are_sound(seed):
    rng = np.random.default_rng(300 + seed)
    J, L = int(rng.integers(2, 20)), int(rng.integers(2, 12))
    m, boxes = emu_tree_scene(rng, J, L)
    n_samples = rng.integers(1, 6, 24)
    off = np.concatenate([[0], np.cumsum(n_samples)]).astype(np.uint32)
    qf = rng.uniform(-2, 2, (24, J))
    qt = qf + rng.uniform(-1, 1, qf.shape)
    _, _, q, sw = emu_sample(m, boxes, qf, qt, off)
    sw = sw.reshape(-1, L)
    c = corners(boxes)
    t = np.arange(0, 66) / 65.0  # the segment's ends and 64 interior points, linear in q
    checked = 0
    for g in range(len(q) - 1):
        if g + 1 in off:
            continue  # a motion's last sample
        qs = q[g] + t[:, None] * (q[g + 1] - q[g])
        p = world_points(emu_poses(m, boxes, qs), np.tile(c, (len(t), 1, 1))).reshape(len(t), L, 8, 3)
        path = np.linalg.norm(np.diff(p, axis=0), axis=3).sum(axis=0).max(axis=1)  # per link, its farthest corner
        assert (path <= sw[g] + 1e-12).all(), (g, path - sw[g])
        checked += 1
    assert checked > 20


def test_chain_sweep_close_to_the_hand_bound():
    w = W.robot_motions(32, n_env=200, room=3.0, seed=5)
    emu = EmuScene()
    m = chain_model(w, w["register"](emu))
    _, _, q, sw = emu_sample(m, local_boxes(emu, m["handles"]), m["q_from"], m["q_to"], w["offsets"])
    hand = W.chain_sweep_bounds(w)
    assert np.isfinite(sw).all()
    moving = hand > 0
    ratio = sw[moving] / hand[moving]
    assert 0.5 < ratio.min() and ratio.max() < 2.0
    assert (sw[~moving] == 0).all()
