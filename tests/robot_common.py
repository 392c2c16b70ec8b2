"""Helpers of the robot-model tests: the host build of the kinematics (tests/emu/kin_emu.cpp, the arithmetic of the
device kernel), a numpy restatement of the model's semantics (include/hppfcl_b200.h, hfb_robot_desc), and seeded
random trees."""
import ctypes as C
import os
import subprocess

import numpy as np

from tests.common import EMU_DIR, ROOT, P, hf
from hppfcl_b200 import workloads as W

_KIN = None


def kin_lib():
    global _KIN
    if _KIN is None:
        so = os.path.join(EMU_DIR, "libkin_emu.so")
        src = os.path.join(EMU_DIR, "kin_emu.cpp")
        csrc = os.path.join(ROOT, "hpp-fcl_b200", "csrc")
        deps = [src, os.path.join(csrc, "hfb_kin.cuh"), os.path.join(csrc, "hfb_math.cuh"),
                os.path.join(ROOT, "include", "hppfcl_b200.h")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-march=x86-64-v2",
                                   "-shared", "-o", so, src])
        L = C.CDLL(so)
        vp, sz = C.c_void_p, C.c_size_t
        L.kin_sincos.argtypes = [sz, vp, vp, vp]
        L.kin_poses.argtypes = [vp, vp, sz, vp, vp]
        L.kin_sample_motions.argtypes = [vp, vp, sz, vp, vp, vp, vp, vp, vp]
        _KIN = L
    return _KIN


def _p(a):
    return None if a is None else a.ctypes.data


def sincos(x):
    x = np.ascontiguousarray(x, dtype=np.float64)
    s, c = np.empty_like(x), np.empty_like(x)
    kin_lib().kin_sincos(x.size, _p(x), _p(s), _p(c))
    return s, c


def desc(m):
    """the hfb_robot_desc of a model dict (parent, types, axis, placement, link_joint, link_placement, handles)"""
    return hf.robot_desc(m["parent"], m["types"], m["axis"], m["placement"], m["link_joint"], m["link_placement"],
                         m["handles"])


def emu_poses(m, boxes, q):
    d, keep = desc(m)
    J, L = d.num_joints, d.num_links
    q = np.ascontiguousarray(q, dtype=np.float64).reshape(-1, J)
    b = np.ascontiguousarray(boxes, dtype=np.float64)
    tfs = np.empty(q.shape[0] * L, dtype=P.transform_dtype)
    assert kin_lib().kin_poses(C.byref(d), _p(b), q.shape[0], _p(q), _p(tfs)) == 0
    return tfs


def emu_sample(m, boxes, q_from, q_to, off):
    """-> (tfs, handles, q, sweep) as hfb_robot_sample_motions writes them"""
    d, keep = desc(m)
    J, L = d.num_joints, d.num_links
    off = np.ascontiguousarray(off, dtype=np.uint32)
    qf = np.ascontiguousarray(q_from, dtype=np.float64)
    qt = np.ascontiguousarray(q_to, dtype=np.float64)
    b = np.ascontiguousarray(boxes, dtype=np.float64)
    n = int(off[-1])
    tfs = np.empty(n * L, dtype=P.transform_dtype)
    q = np.empty((n, J))
    sw = np.empty(n * L)
    assert kin_lib().kin_sample_motions(C.byref(d), _p(b), len(off) - 1, _p(qf), _p(qt), _p(off), _p(tfs), _p(q),
                                        _p(sw)) == 0
    return tfs, np.tile(np.asarray(m["handles"], dtype=np.uint32), n), q, sw


def local_boxes(scene, handles):
    """the links' committed local boxes: scene_aabbs at the identity pose returns them unchanged"""
    h = np.asarray(handles, dtype=np.uint32)
    return scene.scene_aabbs(h, P.make_transforms(np.broadcast_to(np.eye(3), (len(h), 3, 3)), np.zeros((len(h), 3))))


def _mats(tfs):
    tfs = np.asarray(tfs)
    return tfs["R"].reshape(-1, 3, 3).transpose(0, 2, 1), tfs["T"].reshape(-1, 3)  # (column-major storage)


def np_poses(m, q):
    """the header's semantics in numpy (np.sin / np.cos, matrix products) -> (R (n, L, 3, 3), T (n, L, 3))"""
    q = np.asarray(q, dtype=np.float64)
    n = q.shape[0]
    PR, PT = _mats(m["placement"])
    LR, LT = _mats(m["link_placement"])
    ax = np.asarray(m["axis"], dtype=np.float64)
    ax = ax / np.linalg.norm(ax, axis=1, keepdims=True)
    FR, FT = [], []
    for j, (par, typ) in enumerate(zip(m["parent"], m["types"])):
        if par < 0:
            R0, T0 = np.broadcast_to(PR[j], (n, 3, 3)), np.broadcast_to(PT[j], (n, 3))
        else:
            R0 = FR[par] @ PR[j]
            T0 = np.einsum("nij,j->ni", FR[par], PT[j]) + FT[par]
        a = ax[j]
        if typ == P.JOINT_PRISMATIC:
            FR.append(R0)
            FT.append(T0 + np.einsum("nij,nj->ni", R0, q[:, j, None] * a))
        else:
            s, c = np.sin(q[:, j]), np.cos(q[:, j])
            K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
            X = c[:, None, None] * np.eye(3) + s[:, None, None] * K + (1 - c)[:, None, None] * np.outer(a, a)
            FR.append(R0 @ X)
            FT.append(T0)
    R = np.empty((n, len(m["link_joint"]), 3, 3))
    T = np.empty((n, len(m["link_joint"]), 3))
    for i, lj in enumerate(m["link_joint"]):
        if lj < 0:
            R[:, i], T[:, i] = LR[i], LT[i]
        else:
            R[:, i] = FR[lj] @ LR[i]
            T[:, i] = np.einsum("nij,j->ni", FR[lj], LT[i]) + FT[lj]
    return R, T


def depth(m):
    d = []
    for lj in m["link_joint"]:
        k = 0
        while lj >= 0:
            k, lj = k + 1, m["parent"][lj]
        d.append(k)
    return np.array(d)


def random_tree(rng, n_joints, n_links, handles, world_links=1):
    """a seeded tree of revolute and prismatic joints (random parents, axes, placements), n_links links on random
    joints and `world_links` of them fixed to the world; geometry handles drawn from `handles`"""
    J, L = n_joints, n_links
    parent = np.array([-1] + [int(rng.integers(-1, j)) for j in range(1, J)], dtype=np.int32)
    types = np.where(rng.random(J) < 0.3, P.JOINT_PRISMATIC, P.JOINT_REVOLUTE).astype(np.uint32)
    axis = rng.standard_normal((J, 3)) * rng.uniform(0.5, 2.0, (J, 1))
    axis[rng.random(J) < 0.3] = np.eye(3)[rng.integers(0, 3)]  # some axes exactly along x, y or z
    placement = W.random_transforms(rng, J, (-0.3, -0.3, -0.3), (0.3, 0.3, 0.3))
    link_joint = rng.integers(0, J, L).astype(np.int32)
    link_joint[rng.permutation(L)[:world_links]] = -1
    link_placement = W.random_transforms(rng, L, (-0.1, -0.1, -0.1), (0.1, 0.1, 0.1))
    return dict(parent=parent, types=types, axis=axis, placement=placement, link_joint=link_joint,
                link_placement=link_placement, handles=np.asarray(handles, dtype=np.uint32)[rng.integers(0, len(handles), L)])


def chain_model(w, hs):
    """workloads.chain_robot_model(w) with the handles `hs` of w's registered geometry"""
    m = W.chain_robot_model(w)
    m["handles"] = np.asarray(hs, dtype=np.uint32)[m["geom"]]
    return m


def link_shapes():
    """link geometry of the random trees: boxes, capsules and spheres of a few cm"""
    return P.make_shapes([P.GEOM_BOX, P.GEOM_CAPSULE, P.GEOM_SPHERE, P.GEOM_BOX],
                         [[0.05, 0.02, 0.1], [0.03, 0.08, 0], [0.04, 0, 0], [0.2, 0.01, 0.01]])
