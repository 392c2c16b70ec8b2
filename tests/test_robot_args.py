"""hfb_robot_create and the robot calls refuse malformed arguments before they touch the context or the device: each
malformed model (a bad parent, type or link joint, J = 0 or J > 64, no links, L * J >= 2^32, a zero or non-finite axis, a null array),
null pointers, and malformed motion offsets.  The Python mirrors refuse arrays of the wrong length with ValueError."""
import ctypes as C

import numpy as np
import pytest

from tests.common import P, hf
from hppfcl_b200 import workloads as W

INVALID = 1


def model(J=3, L=2):
    return dict(parent=np.arange(-1, J - 1, dtype=np.int32), types=np.zeros(J, dtype=np.uint32),
                axis=np.tile([0.0, 0.0, 1.0], (J, 1)), placement=W.identity_transforms(J),
                link_joint=np.arange(L, dtype=np.int32) % J, link_placement=W.identity_transforms(L),
                handles=np.zeros(L, dtype=np.uint32))


def create(L, m, ctx, **null):
    d, keep = hf.robot_desc(m["parent"], m["types"], m["axis"], m["placement"], m["link_joint"], m["link_placement"],
                            m["handles"])
    for k in null:
        setattr(d, k, None)
    out = C.c_void_p()
    return L.hfb_robot_create(ctx, C.byref(d), C.byref(out))


def test_create_refuses_malformed_models_before_the_context():
    L = hf.load_library()
    ctx = C.create_string_buffer(4096)  # a stand-in: the call must refuse before reading it
    bad = []
    m = model(); m["parent"][1] = 1; bad.append(m)           # not an earlier joint
    m = model(); m["parent"][2] = -2; bad.append(m)          # below -1
    m = model(); m["parent"][0] = 0; bad.append(m)
    m = model(); m["types"][1] = 2; bad.append(m)            # unknown type
    m = model(); m["link_joint"][0] = 3; bad.append(m)       # past the joints
    m = model(); m["link_joint"][1] = -2; bad.append(m)
    m = model(); m["axis"][1] = 0.0; bad.append(m)           # zero axis
    m = model(); m["axis"][2, 0] = np.nan; bad.append(m)     # non-finite axes
    m = model(); m["axis"][0, 1] = np.inf; bad.append(m)
    bad.append(model(J=65))                                  # J > 64
    for m in bad:
        assert create(L, m, ctx) == INVALID
    m = model()
    for field in ("parent", "type", "axis", "placement", "link_joint", "link_placement", "link_handles"):
        assert create(L, m, ctx, **{field: 0}) == INVALID, field
    d, keep = hf.robot_desc(*[m[k] for k in ("parent", "types", "axis", "placement", "link_joint", "link_placement",
                                             "handles")])
    out = C.c_void_p()
    # J = 0, no links, and L * J past 32 bits (refused from the counts, before the link arrays are read)
    for nj, nl in ((0, 2), (3, 0), (64, 1 << 26), (2, 0x80000000)):
        d2 = P.RobotDesc(nj, d.parent, d.type, d.axis, d.placement, nl, d.link_joint, d.link_placement, d.link_handles)
        assert L.hfb_robot_create(ctx, C.byref(d2), C.byref(out)) == INVALID
    assert L.hfb_robot_create(None, C.byref(d), C.byref(out)) == INVALID
    assert L.hfb_robot_create(ctx, None, C.byref(out)) == INVALID
    assert L.hfb_robot_create(ctx, C.byref(d), None) == INVALID


def test_calls_refuse_null_pointers_and_bad_offsets():
    L = hf.load_library()
    ctx = C.create_string_buffer(4096)
    robot = C.create_string_buffer(4096)
    q = np.zeros(12)
    tfs = np.zeros(8, dtype=P.transform_dtype)
    h = np.zeros(8, dtype=np.uint32)
    qp, tp, hp = q.ctypes.data, tfs.ctypes.data, h.ctypes.data
    for fn in (L.hfb_robot_poses, L.hfb_robot_poses_device):
        extra = [None] if fn is L.hfb_robot_poses_device else []
        assert fn(None, robot, 2, qp, tp, hp, *extra) == INVALID
        assert fn(ctx, None, 2, qp, tp, hp, *extra) == INVALID
        assert fn(ctx, robot, 2, None, tp, hp, *extra) == INVALID
        assert fn(ctx, robot, 2, qp, None, hp, *extra) == INVALID
    ok = P.RobotSamplesOut(tp, hp, None, None)
    for fn in (L.hfb_robot_sample_motions, L.hfb_robot_sample_motions_device):
        extra = [None] if fn is L.hfb_robot_sample_motions_device else []

        def call(ctx=ctx, robot=robot, qf=qp, qt=qp, off=(0, 1, 3), out=C.byref(ok)):
            o = None if off is None else np.asarray(off, dtype=np.uint32)
            return fn(ctx, robot, 2 if o is None else len(o) - 1, qf, qt, None if o is None else o.ctypes.data, out,
                      *extra)

        assert call(ctx=None) == INVALID
        assert call(robot=None) == INVALID
        assert call(qf=None) == INVALID
        assert call(qt=None) == INVALID
        assert call(off=None) == INVALID
        assert call(out=None) == INVALID
        assert call(out=C.byref(P.RobotSamplesOut(None, hp, None, None))) == INVALID
        assert call(out=C.byref(P.RobotSamplesOut(tp, None, None, None))) == INVALID
        assert call(off=(1, 2, 3)) == INVALID             # offsets do not start at 0
        assert call(off=(0, 2, 1)) == INVALID             # decreasing
        assert call(off=(0, 0x80000000)) == INVALID       # a motion of more than INT32_MAX samples


def test_python_mirror_lengths():
    m = model()
    with pytest.raises(ValueError):
        hf.robot_desc(m["parent"], m["types"][:2], m["axis"], m["placement"], m["link_joint"], m["link_placement"],
                      m["handles"])
    with pytest.raises(ValueError):
        hf.robot_desc(m["parent"], m["types"], m["axis"], m["placement"], m["link_joint"], m["link_placement"],
                      m["handles"][:1])
    eng = hf.Engine.__new__(hf.Engine)  # (no context: the checks come first)
    eng._robots = {1: (3, 2)}
    with pytest.raises(ValueError):
        eng.robot_poses(C.c_void_p(1), np.zeros(7))
    with pytest.raises(ValueError):
        eng.robot_sample_motions(C.c_void_p(1), np.zeros(3), np.zeros(6), [0, 2])
