"""The resident environment's C ABI refuses malformed arguments before it touches the context or the device: null
context, env, request, output or buffers, and a capacity without pair buffers (no GPU needed)."""
import ctypes as C

import numpy as np

from tests.common import P, hf

INVALID = 1


def test_env_abi_argument_checks():
    L = hf.load_library()
    # stand-ins: the calls must refuse before reading them
    ctx = C.create_string_buffer(4096)
    env = C.create_string_buffer(4096)
    h = np.zeros(4, dtype=np.uint32)
    t = np.zeros(4, dtype=P.transform_dtype)
    hp, tp = h.ctypes.data, t.ctypes.data
    req = P.CollisionRequestPOD()
    f, s = np.zeros(8, dtype=np.uint32), np.zeros(8, dtype=np.uint32)
    rec = np.zeros(8, dtype=P.contact_dtype)
    cnt = np.zeros(2, dtype=np.uint32)
    ok = P.EnvOut(f.ctypes.data, s.ctypes.data, rec.ctypes.data, 8, cnt.ctypes.data, cnt[1:].ctypes.data, None)
    out = C.c_void_p()
    assert L.hfb_env_create(None, 4, hp, tp, C.byref(out)) == INVALID
    assert L.hfb_env_create(ctx, 4, hp, tp, None) == INVALID
    assert L.hfb_env_create(ctx, 4, None, tp, C.byref(out)) == INVALID
    assert L.hfb_env_create(ctx, 4, hp, None, C.byref(out)) == INVALID
    assert L.hfb_env_update(None, env, 1, hp, tp) == INVALID
    assert L.hfb_env_update(ctx, None, 1, hp, tp) == INVALID
    assert L.hfb_env_update(ctx, env, 1, None, tp) == INVALID
    assert L.hfb_env_update(ctx, env, 1, hp, None) == INVALID
    for fn, a_h, a_t in ((L.hfb_env_collide, hp, tp), (L.hfb_env_collide_device, hp, tp)):
        extra = [None] if fn is L.hfb_env_collide_device else []
        assert fn(None, env, 4, a_h, a_t, 0, 4, C.byref(req), C.byref(ok), *extra) == INVALID
        assert fn(ctx, None, 4, a_h, a_t, 0, 4, C.byref(req), C.byref(ok), *extra) == INVALID
        assert fn(ctx, env, 4, None, a_t, 0, 4, C.byref(req), C.byref(ok), *extra) == INVALID
        assert fn(ctx, env, 4, a_h, None, 0, 4, C.byref(req), C.byref(ok), *extra) == INVALID
        assert fn(ctx, env, 4, a_h, a_t, 0, 4, None, C.byref(ok), *extra) == INVALID
        assert fn(ctx, env, 4, a_h, a_t, 0, 4, C.byref(req), None, *extra) == INVALID
        for k in range(3):  # a capacity without one of the three pair buffers
            bad = P.EnvOut(*[None if j == k else getattr(ok, n) for j, (n, _) in enumerate(P.EnvOut._fields_)])
            assert fn(ctx, env, 4, a_h, a_t, 0, 4, C.byref(req), C.byref(bad), *extra) == INVALID
    assert L.hfb_env_destroy(None, env) == INVALID
    assert L.hfb_env_destroy(ctx, None) == INVALID
