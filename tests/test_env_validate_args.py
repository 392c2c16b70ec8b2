"""hfb_env_validate_motions refuses malformed arguments before it touches the context or the device: the depths, the
cap, null context, env, robot, request, params, output struct or required outputs, a null template or null end points
with work to do, and a range past the end; a refused call writes nothing.  The Python mirror raises ValueError for
wrong shapes and the same refusals before the engine is called (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest

from tests.common import P, hf
from hppfcl_b200 import api

INVALID = 1


def test_validate_abi_argument_checks():
    L = hf.load_library()
    # stand-ins: the calls must refuse before reading them
    ctx, env, robot = (C.create_string_buffer(4096) for _ in range(3))
    q = np.zeros((2, 3), dtype=np.float64)
    qp = q.ctypes.data
    tpl = np.array([[0, 1]], dtype=np.uint32)
    req = P.CollisionRequestPOD()
    st = np.full(2, 0x55, dtype=np.int8)
    tv = np.full(2, 7.0)
    tc = np.full(2, 7.0)
    ok = P.ValidateOut(st.ctypes.data, tv.ctypes.data, tc.ctypes.data, *[None] * 9)
    good = P.ValidateParams(1, 4, 100)
    for fn in (L.hfb_env_validate_motions, L.hfb_env_validate_motions_device):
        extra = [None] if fn is L.hfb_env_validate_motions_device else []

        def call(ctx=ctx, env=env, robot=robot, n=2, qf=qp, qt=qp, n_tpl=1, tp_=tpl.ctypes.data, m0=0, nm=2,
                 req=C.byref(req), p=C.byref(good), out=C.byref(ok)):
            return fn(ctx, env, robot, n, qf, qt, n_tpl, tp_, m0, nm, req, p, out, *extra)

        assert call(ctx=None) == INVALID
        assert call(env=None) == INVALID
        assert call(robot=None) == INVALID
        assert call(req=None) == INVALID
        assert call(p=None) == INVALID
        assert call(out=None) == INVALID
        for k in range(3):  # status, t_valid and t_collide are required
            fields = [st.ctypes.data, tv.ctypes.data, tc.ctypes.data]
            fields[k] = None
            assert call(out=C.byref(P.ValidateOut(*fields, *[None] * 9))) == INVALID
        assert call(tp_=None) == INVALID
        assert call(qf=None) == INVALID
        assert call(qt=None) == INVALID
        assert call(m0=1, nm=2) == INVALID and call(m0=3, nm=0) == INVALID
        for bad in ((5, 4, 100), (1, 31, 100), (0, 4, 1), (0, 4, 0)):  # d0 > D, D > 30, max_samples < 2
            assert call(p=C.byref(P.ValidateParams(*bad))) == INVALID
        assert (st == 0x55).all() and (tv == 7.0).all() and (tc == 7.0).all()  # nothing written


class _Model:
    nq, num_links = 3, 2


def test_python_mirror_refusals():
    env = api.ResidentEnvironment.__new__(api.ResidentEnvironment)  # (each refusal comes before the environment is used)
    f = api.ResidentEnvironment.validate_motions
    q = np.zeros((4, 3))
    kw = dict(initial_depth=1, max_depth=4, max_samples=100)
    for a, b in ((np.zeros((4, 2)), np.zeros((4, 2))), (q, np.zeros((3, 3))), (q.reshape(-1), q.reshape(-1))):
        with pytest.raises(ValueError):
            f(env, _Model(), a, b, [(0, 1)], **kw)
    for bad in (dict(initial_depth=5, max_depth=4, max_samples=100), dict(initial_depth=0, max_depth=31, max_samples=100),
                dict(initial_depth=0, max_depth=4, max_samples=1)):
        with pytest.raises(ValueError):
            f(env, _Model(), q, q, [(0, 1)], **bad)
    with pytest.raises(ValueError):
        f(env, _Model(), q, q, [(0, 2)], **kw)  # a link index out of range
    with pytest.raises(ValueError):
        f(env, _Model(), q, q, [(0, 1)], first_motion=3, num_motions=2, **kw)
