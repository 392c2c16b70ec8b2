"""hfb_env_certify_motions refuses malformed arguments before it touches the context or the device: null context, env,
request, sweep, output, offsets or buffers, and outputs without any of first_invalid, first_uncertified and certified.
hfb_broadphase_sweep_pairs refuses what the query refuses.  The Python mirrors refuse a sweep of the wrong length
with ValueError before the engine is called (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest

from tests.common import P, hf

INVALID = 1


def test_certify_abi_argument_checks():
    L = hf.load_library()
    # stand-ins: the calls must refuse before reading them
    ctx = C.create_string_buffer(4096)
    env = C.create_string_buffer(4096)
    h = np.zeros(4, dtype=np.uint32)
    t = np.zeros(4, dtype=P.transform_dtype)
    sw = np.zeros(4, dtype=np.float64)
    hp, tp, swp = h.ctypes.data, t.ctypes.data, sw.ctypes.data
    tpl = np.array([[0, 1]], dtype=np.uint32)
    off = np.array([0, 2], dtype=np.uint32)
    op = off.ctypes.data
    req = P.CollisionRequestPOD()
    fi = np.zeros(1, dtype=np.int32)
    fu = np.zeros(1, dtype=np.int32)
    cert = np.zeros(2, dtype=np.uint8)
    cnt = np.zeros(4, dtype=np.uint32)
    counts = [cnt[k:].ctypes.data for k in range(4)]
    ok = P.CertifyOut(fi.ctypes.data, fu.ctypes.data, cert.ctypes.data, *counts)
    none = P.CertifyOut(None, None, None, *counts)
    for fn in (L.hfb_env_certify_motions, L.hfb_env_certify_motions_device):
        extra = [None] if fn is L.hfb_env_certify_motions_device else []

        def call(ctx=ctx, env=env, a_h=hp, a_t=tp, s=swp, tp_=tpl.ctypes.data, offs=op, req=C.byref(req), out=C.byref(ok)):
            return fn(ctx, env, 4, a_h, a_t, s, 2, 1, tp_, 1, offs, 0, 1, req, out, *extra)

        assert call(ctx=None) == INVALID
        assert call(env=None) == INVALID
        assert call(a_h=None) == INVALID
        assert call(a_t=None) == INVALID
        assert call(s=None) == INVALID
        assert call(tp_=None) == INVALID
        assert call(offs=None) == INVALID
        assert call(req=None) == INVALID
        assert call(out=None) == INVALID
        assert call(out=C.byref(none)) == INVALID  # all three per-item outputs null
        # each per-item output alone is enough: refused here only for the stand-in context
        for alone in (P.CertifyOut(fi.ctypes.data, None, None, None, None, None, None),
                      P.CertifyOut(None, fu.ctypes.data, None, None, None, None, None),
                      P.CertifyOut(None, None, cert.ctypes.data, None, None, None, None)):
            assert call(ctx=None, out=C.byref(alone)) == INVALID


def test_sweep_pairs_abi_argument_checks():
    L = hf.load_library()
    bb = np.zeros((4, 6), dtype=np.float64)
    sw = np.zeros(4, dtype=np.float64)
    tpl = np.array([[0, 1]], dtype=np.uint32)
    first = np.zeros(8, dtype=np.uint32)
    second = np.zeros(8, dtype=np.uint32)
    n = C.c_size_t(0)

    def call(n_a=4, b=bb.ctypes.data, s=sw.ctypes.data, links=2, tp_=tpl.ctypes.data, n_tpl=1, off=(0, 1, 2), m0=0,
             nm=None, cap=8, out=C.byref(n), f=first.ctypes.data, sec=second.ctypes.data):
        o = np.asarray(off, dtype=np.uint32)
        nm = len(o) - 1 - m0 if nm is None else nm
        return L.hfb_broadphase_sweep_pairs(n_a, b, s, links, n_tpl, tp_, len(o) - 1, o.ctypes.data, m0, nm, f, sec,
                                            cap, out)

    assert call() == 0
    assert call(b=None) == INVALID
    assert call(s=None) == INVALID
    assert call(out=None) == INVALID
    assert call(f=None) == INVALID and call(f=None, cap=0) == 0
    assert call(tp_=None) == INVALID
    assert call(links=3) == INVALID                      # n_a not a multiple of links
    assert call(off=(1, 2)) == INVALID                   # offsets do not start at 0
    assert call(off=(0, 2, 1, 2)) == INVALID             # decreasing
    assert call(off=(0, 1)) == INVALID                   # do not end at n_configs
    assert call(m0=1, nm=2) == INVALID                   # range past the end
    bad = np.array([[0, 0]], dtype=np.uint32)
    assert call(tp_=bad.ctypes.data) == INVALID          # a link paired with itself


def test_python_mirror_sweep_length():
    bb = np.zeros((4, 6))
    with pytest.raises(ValueError):
        hf.broadphase_sweep_pairs(bb, np.zeros(3), 2, [(0, 1)], [0, 1, 2])
    eng = hf.Engine.__new__(hf.Engine)  # (no context: the check comes first)
    with pytest.raises(ValueError):
        eng.env_certify_motions(None, np.zeros(4, np.uint32), np.zeros(4, P.transform_dtype), np.zeros(3), 2,
                                [(0, 1)], [0, 1, 2])
