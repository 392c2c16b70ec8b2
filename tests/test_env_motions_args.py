"""hfb_env_collide_motions refuses malformed arguments before it touches the context or the device: null context, env,
request, output, offsets or buffers, and outputs without any of first_invalid, kind and contacts.  The Python mirror
refuses malformed motion offsets and a motion range past the end with ValueError before the engine is called (no GPU
needed)."""
import ctypes as C

import numpy as np
import pytest

from tests.common import P, hf

INVALID = 1


def test_motions_abi_argument_checks():
    L = hf.load_library()
    # stand-ins: the calls must refuse before reading them
    ctx = C.create_string_buffer(4096)
    env = C.create_string_buffer(4096)
    h = np.zeros(4, dtype=np.uint32)
    t = np.zeros(4, dtype=P.transform_dtype)
    hp, tp = h.ctypes.data, t.ctypes.data
    tpl = np.array([[0, 1]], dtype=np.uint32)
    off = np.array([0, 2], dtype=np.uint32)
    op = off.ctypes.data
    req = P.CollisionRequestPOD()
    fi = np.zeros(1, dtype=np.int32)
    kind = np.zeros(1, dtype=np.int8)
    rec = np.zeros(1, dtype=P.contact_dtype)
    cnt = np.zeros(4, dtype=np.uint32)
    ok = P.MotionsOut(fi.ctypes.data, kind.ctypes.data, None, None, rec.ctypes.data, *[cnt[k:].ctypes.data for k in range(4)])
    none = P.MotionsOut(None, None, None, None, None, *[cnt[k:].ctypes.data for k in range(4)])
    witness_only = P.MotionsOut(None, None, cnt.ctypes.data, cnt[1:].ctypes.data, None, None, None, None, None)
    for fn in (L.hfb_env_collide_motions, L.hfb_env_collide_motions_device):
        extra = [None] if fn is L.hfb_env_collide_motions_device else []

        def call(ctx=ctx, env=env, a_h=hp, a_t=tp, n_tpl=1, tp_=tpl.ctypes.data, offs=op, req=C.byref(req), out=C.byref(ok)):
            return fn(ctx, env, 4, a_h, a_t, 2, n_tpl, tp_, 1, offs, 0, 1, req, out, *extra)

        assert call(ctx=None) == INVALID
        assert call(env=None) == INVALID
        assert call(a_h=None) == INVALID
        assert call(a_t=None) == INVALID
        assert call(tp_=None) == INVALID
        assert call(offs=None) == INVALID
        assert call(req=None) == INVALID
        assert call(out=None) == INVALID
        assert call(out=C.byref(none)) == INVALID  # all three main outputs null
        assert call(out=C.byref(witness_only)) == INVALID  # first and second alone are not enough


def _args(n_objects=12, links=3, off=(0, 2, 4), first=0, num=None):
    return hf.ResidentEnvironment._motion_args(n_objects, links, np.asarray(off), first, num)


def test_python_mirror_accepts_well_formed_offsets():
    off, first, num = _args()
    assert off.dtype == np.uint32 and off.tolist() == [0, 2, 4] and (first, num) == (0, 2)
    assert _args(off=(0, 0, 4, 4), first=1, num=2)[1:] == (1, 2)  # empty motions are allowed
    assert _args(n_objects=0, off=(0,))[1:] == (0, 0)  # no motions at all
    assert _args(first=2, num=0)[1:] == (2, 0)  # an empty range at the end


@pytest.mark.parametrize("off, first, num", [
    ((1, 2, 4), 0, None),          # first offset not 0
    ((0, 3, 2, 4), 0, None),       # decreasing
    ((0, 2, 3), 0, None),          # last offset not n_configs
    ((0, 2, 5), 0, None),
    ((), 0, None),                 # no offsets at all
    ((0, 2, 4), 3, None),          # range past the end
    ((0, 2, 4), 1, 2),
    ((0, 2, 4), 0, 3),
])
def test_python_mirror_refuses_malformed_offsets(off, first, num):
    with pytest.raises(ValueError):
        _args(off=off, first=first, num=num)


def test_python_mirror_refuses_a_size_that_is_not_whole_configurations():
    with pytest.raises(ValueError):
        _args(n_objects=13)


@pytest.mark.parametrize("off", [[0, -1, 4], [0, 2 ** 32], [0.0, 2.0], []])
def test_engine_refuses_offsets_that_are_not_uint32(off):
    from hppfcl_b200 import engine
    with pytest.raises(ValueError):
        engine._offsets(np.array(off))


def test_engine_takes_offsets_of_any_integer_type():
    from hppfcl_b200 import engine
    for dt in (np.int64, np.uint32, np.int32, np.uint64):
        off = engine._offsets(np.array([0, 3, 3, 7], dtype=dt))
        assert off.dtype == np.uint32 and off.flags.c_contiguous and off.tolist() == [0, 3, 3, 7]
