"""The resident environment's distance query (hfb_env_distance*) refuses malformed arguments before it touches the
context or the device: null context, env, request or output, an output with all three per-object buffers null, and a
max_distance that is NaN or negative (no GPU needed)."""
import ctypes as C

import numpy as np

from tests.common import P, hf

INVALID = 1


def test_env_distance_abi_argument_checks():
    L = hf.load_library()
    # stand-ins: the calls must refuse before reading them
    ctx = C.create_string_buffer(4096)
    env = C.create_string_buffer(4096)
    h = np.zeros(4, dtype=np.uint32)
    t = np.zeros(4, dtype=P.transform_dtype)
    hp, tp = h.ctypes.data, t.ctypes.data
    req = P.DistanceRequestPOD()
    nearest = np.zeros(4, dtype=np.int32)
    dist = np.zeros(4, dtype=np.float64)
    rec = np.zeros(4, dtype=P.distance_result_dtype)
    cnt = np.zeros(2, dtype=np.uint32)
    ok = P.EnvDistanceOut(nearest.ctypes.data, dist.ctypes.data, rec.ctypes.data, cnt.ctypes.data, cnt[1:].ctypes.data)
    none = P.EnvDistanceOut(None, None, None, cnt.ctypes.data, cnt[1:].ctypes.data)
    for fn in (L.hfb_env_distance, L.hfb_env_distance_device):
        extra = [None] if fn is L.hfb_env_distance_device else []
        assert fn(None, env, 4, hp, tp, 0, 4, C.byref(req), np.inf, C.byref(ok), *extra) == INVALID
        assert fn(ctx, None, 4, hp, tp, 0, 4, C.byref(req), np.inf, C.byref(ok), *extra) == INVALID
        assert fn(ctx, env, 4, None, tp, 0, 4, C.byref(req), np.inf, C.byref(ok), *extra) == INVALID
        assert fn(ctx, env, 4, hp, None, 0, 4, C.byref(req), np.inf, C.byref(ok), *extra) == INVALID
        assert fn(ctx, env, 4, hp, tp, 0, 4, None, np.inf, C.byref(ok), *extra) == INVALID
        assert fn(ctx, env, 4, hp, tp, 0, 4, C.byref(req), np.inf, None, *extra) == INVALID
        assert fn(ctx, env, 4, hp, tp, 0, 4, C.byref(req), np.inf, C.byref(none), *extra) == INVALID
        for bad in (np.nan, -1.0, -np.inf, -1e-300, -5e-324):
            assert fn(ctx, env, 4, hp, tp, 0, 4, C.byref(req), bad, C.byref(ok), *extra) == INVALID
    assert list(cnt) == [0, 0] and not nearest.any() and not dist.any()

