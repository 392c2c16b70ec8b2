"""The self pairs whose distance() the configurations distance query runs (hfb_broadphase_config_distance_pairs) and the
argument checks of that query (hfb_env_distance_configs*): no GPU needed.  The definition the finder must meet: for
every configuration g of the range and every template pair (i, j), the pair (g * L + i, g * L + j) runs unless both
boxes exist and are finite and j's box does not overlap i's box widened by max_distance -- each lower bound rounded
down, each upper bound rounded up (the device's __dsub_rd / __dadd_ru) -- configuration by configuration in the
template's order.  The rounding here is computed exactly with fractions, independently of the library's."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

from tests.common import P, hf
from tests.test_config_pairs import BIG, INVALID, NONE, chain_boxes
from hppfcl_b200 import workloads as W


MAXF = Fraction(BIG)


def round_down(q):
    """the largest double <= the rational q"""
    if q < -MAXF:
        return -np.inf
    if q > MAXF:
        return BIG
    d = float(q)
    return np.nextafter(d, -np.inf) if Fraction(d) > q else d


def round_up(q):
    return -round_down(-q)


def widen(lo, hi, r):
    """[lo - r rounded down, hi + r rounded up] from the exact rational values (lo, hi finite, r >= 0 or inf)"""
    if np.isinf(r):
        return -np.inf, np.inf
    return round_down(Fraction(lo) - Fraction(r)), round_up(Fraction(hi) + Fraction(r))


def runs(x, y, r):
    if (x[0] == BIG and x[3] == -BIG) or (y[0] == BIG and y[3] == -BIG):
        return True
    if not (np.isfinite(x).all() and np.isfinite(y).all()):
        return True
    for k in range(3):
        lo, hi = widen(x[k], x[3 + k], r)
        if lo > y[3 + k] or hi < y[k]:
            return False
    return True


def brute(bb, links, tpl, r, g0=0, ng=None):
    tpl = np.asarray(tpl, dtype=np.int64).reshape(-1, 2)
    ng = len(bb) // links - g0 if ng is None else ng
    return [(g * links + i, g * links + j) for g in range(g0, g0 + ng) for i, j in tpl
            if runs(bb[g * links + i], bb[g * links + j], r)]


def found(bb, links, tpl, r, g0=0, ng=None):
    f, s = hf.broadphase_config_distance_pairs(bb, links, tpl, r, first_config=g0, num_configs=ng)
    return list(zip(f.tolist(), s.tolist()))


def test_random_boxes_match_the_definition():
    rng = np.random.default_rng(11)
    for links, skip in ((16, 2), (6, 1)):
        bb = chain_boxes(rng, 40, links)
        tpl = W.chain_self_pairs(links, skip)
        counts = []
        for r in (0.0, 0.05, 0.3, np.inf):
            want = brute(bb, links, tpl, r)
            assert found(bb, links, tpl, r) == want
            counts.append(len(want))
        # the cutoff widens the set, and at inf every template pair runs
        assert counts == sorted(counts) and counts[0] < counts[2] < counts[3] == 40 * len(tpl)
        # at 0 the set is the collide finder's (closed intervals, nothing widened)
        f, s = hf.broadphase_config_pairs(bb, links, tpl)
        assert found(bb, links, tpl, 0.0) == list(zip(f.tolist(), s.tolist()))


def test_exact_gap_and_outward_rounding():
    one_up, one_down = np.nextafter(1.0, 2.0), np.nextafter(1.0, 0.0)
    tiny = 1e-17  # below half an ulp of 1: 1 + tiny rounds to 1 to nearest, to the next double upward
    links = 2
    cases = [  # (box of link 0, box of link 1, max_distance, runs)
        ([0, 0, 0, 1, 1, 1], [1.25, 0, 0, 2, 1, 1], 0.25, True),  # the gap is exactly the cutoff
        ([0, 0, 0, 1, 1, 1], [1.25, 0, 0, 2, 1, 1], np.nextafter(0.25, 0), True),  # rounded up to 1.25 again
        ([0, 0, 0, 1, 1, 1], [1.25, 0, 0, 2, 1, 1], 0.25 - 2.0 ** -52, False),  # 1.25 - 2^-52 exactly
        ([0, 0, 0, 1, 1, 1], [one_up, 0, 0, 2, 1, 1], tiny, True),  # to nearest the widened box would end at 1
        ([0, 0, 0, 1, 1, 1], [one_up, 0, 0, 2, 1, 1], 0.0, False),
        ([1, 0, 0, 2, 1, 1], [0, 0, 0, one_down, 1, 1], tiny, True),  # the lower side, rounded down
        ([1, 0, 0, 2, 1, 1], [0, 0, 0, one_down, 1, 1], 0.0, False),
        ([0, 0, 0, 1, 1, 1], [0, 0, 1 + 0.1, 1, 1, 2], 0.1, True),  # 1 + 0.1 is inexact: rounded up it reaches
        ([0, 0, 0, 0.1, 1, 1], [0.3, 0, 0, 1, 1, 1], 0.2, True),  # 0.1 + 0.2 > 0.3 to nearest, and upward
        ([0, 0, 0, 1e300, 1, 1], [1.5e300, 0, 0, 1.6e300, 1, 1], 4e299, False),
        ([0, 0, 0, 1e300, 1, 1], [1.5e300, 0, 0, 1.6e300, 1, 1], 5e299, True),
    ]
    for x, y, r, want in cases:
        bb = np.array([x, y], dtype=np.float64)
        assert runs(bb[0], bb[1], r) == want, (x, y, r)
        assert (found(bb, links, [(0, 1)], r) == [(0, 1)]) == want, (x, y, r)
    # the template's order: link i is the one widened
    bb = np.array([[0, 0, 0, 1, 1, 1], [one_up, 0, 0, 2, 1, 1]], dtype=np.float64)
    assert found(bb, 2, [(1, 0)], tiny) == brute(bb, 2, [(1, 0)], tiny)


def test_boxless_nonfinite_and_unbounded_links():
    rng = np.random.default_rng(12)
    links = 6
    bb = chain_boxes(rng, 30, links, spread=0.6)
    floor = [-BIG, -BIG, -BIG, BIG, BIG, -5.0]  # a halfspace link, far below the others
    tilted = [-np.inf, -np.inf, -np.inf, np.inf, np.inf, np.inf]
    bb[[2, 9, 20]] = [floor, tilted, floor]
    bb[[3, 31]] = NONE
    bb[13, 1] = np.nan
    bb[15, 0] = np.inf
    bb[16, 5] = -np.inf
    bb[17] = np.nan
    tpl = W.chain_self_pairs(links, 1)
    for r in (0.0, 0.05, 1.0, np.inf):
        want = brute(bb, links, tpl, r)
        assert found(bb, links, tpl, r) == want
        got = set(want)
        # a boxless or non-finite link always runs; the far floor is skipped within a small cutoff only
        assert all(p in got for p in [(0, 3), (1, 3), (12, 13), (12, 15), (12, 17), (6, 9)])
    assert (0, 2) not in set(found(bb, links, tpl, 0.05)) and (0, 2) in set(found(bb, links, tpl, np.inf))


def test_partial_ranges_capacity_and_empty_template():
    rng = np.random.default_rng(13)
    links = 16
    bb = chain_boxes(rng, 60, links)
    tpl = W.chain_self_pairs(links)
    whole = found(bb, links, tpl, 0.05)
    parts = []
    for g0, ng in ((0, 1), (1, 20), (21, 0), (21, 39)):
        part = found(bb, links, tpl, 0.05, g0, ng)
        assert part == brute(bb, links, tpl, 0.05, g0, ng)
        parts += part
    assert parts == whole
    L = hf.load_library()
    tp = np.ascontiguousarray(tpl)
    f, s = np.zeros(5, np.uint32), np.zeros(5, np.uint32)
    cnt = C.c_size_t(0)
    fn = L.hfb_broadphase_config_distance_pairs
    assert fn(len(bb), bb.ctypes.data, links, len(tp), tp.ctypes.data, 0, 60, 0.05, f.ctypes.data, s.ctypes.data, 5,
              C.byref(cnt)) == 0
    assert cnt.value == len(whole) and list(zip(f.tolist(), s.tolist())) == whole[:5]
    assert fn(len(bb), bb.ctypes.data, links, len(tp), tp.ctypes.data, 0, 60, 0.05, None, None, 0, C.byref(cnt)) == 0
    assert cnt.value == len(whole)
    assert found(bb, links, np.zeros((0, 2), np.uint32), np.inf) == []
    assert found(bb[:0], links, tpl, np.inf) == []


def test_host_finder_refusals():
    L = hf.load_library()
    bb = chain_boxes(np.random.default_rng(14), 3, 4)
    tp = np.ascontiguousarray(np.array([(0, 2), (1, 3)], dtype=np.uint32))
    f, s = np.zeros(8, np.uint32), np.zeros(8, np.uint32)
    cnt = C.c_size_t(12345)
    fn = L.hfb_broadphase_config_distance_pairs
    B, T, F, S = bb.ctypes.data, tp.ctypes.data, f.ctypes.data, s.ctypes.data

    def call(n=12, links=4, g0=0, ng=3, aabbs=B, n_tpl=2, tpl=T, r=0.1, first=F, second=S, cap=8, out=C.byref(cnt)):
        return fn(n, aabbs, links, n_tpl, tpl, g0, ng, r, first, second, cap, out)

    for bad in (dict(links=0), dict(n=11), dict(links=5), dict(g0=4, ng=0), dict(g0=1, ng=3), dict(ng=4),
                dict(aabbs=None), dict(tpl=None), dict(first=None), dict(second=None), dict(out=None),
                dict(r=np.nan), dict(r=-1.0), dict(r=-np.inf), dict(r=-5e-324)):
        assert call(**bad) == INVALID, bad
    for tpl in ([(0, 4)], [(1, 1)], [(0, 2), (2, 0)]):
        t2 = np.ascontiguousarray(np.array(tpl, dtype=np.uint32))
        assert call(n_tpl=len(t2), tpl=t2.ctypes.data) == INVALID, tpl
    assert cnt.value == 12345  # nothing written
    for bad in (np.nan, -0.5):
        with pytest.raises(hf.EngineError):
            hf.broadphase_config_distance_pairs(bb, 4, tp, bad)
    assert call(r=0.0) == 0 and call(r=np.inf) == 0 and cnt.value == 6


def test_configs_distance_abi_argument_checks():
    """the configurations distance query refuses null and malformed arguments before it touches the context or the
    env: null context, env, handles, poses, template, request or output, an output with kind, min_distance and results
    all null, and a max_distance that is NaN or negative"""
    L = hf.load_library()
    ctx = C.create_string_buffer(4096)  # stand-ins: the calls must refuse before reading them
    env = C.create_string_buffer(4096)
    h = np.zeros(8, dtype=np.uint32)
    t = np.zeros(8, dtype=P.transform_dtype)
    tp = np.ascontiguousarray(np.array([(0, 2), (1, 3)], dtype=np.uint32))
    req = P.DistanceRequestPOD()
    kind = np.zeros(2, dtype=np.int8)
    first, second = np.zeros(2, dtype=np.uint32), np.zeros(2, dtype=np.uint32)
    dist = np.zeros(2, dtype=np.float64)
    rec = np.zeros(2, dtype=P.distance_result_dtype)
    cnt = np.zeros(3, dtype=np.uint32)
    ok = P.ConfigsDistanceOut(kind.ctypes.data, first.ctypes.data, second.ctypes.data, dist.ctypes.data, rec.ctypes.data,
                              cnt.ctypes.data, cnt[1:].ctypes.data, cnt[2:].ctypes.data)
    none = P.ConfigsDistanceOut(None, first.ctypes.data, second.ctypes.data, None, None, cnt.ctypes.data,
                                cnt[1:].ctypes.data, cnt[2:].ctypes.data)
    for fn in (L.hfb_env_distance_configs, L.hfb_env_distance_configs_device):
        extra = [None] if fn is L.hfb_env_distance_configs_device else []

        def call(c=ctx, e=env, a_h=h.ctypes.data, a_t=t.ctypes.data, tpl=tp.ctypes.data, r=C.byref(req), maxd=np.inf,
                 o=C.byref(ok)):
            return fn(c, e, 8, a_h, a_t, 4, 2, tpl, 0, 2, r, maxd, o, *extra)

        for bad in (dict(c=None), dict(e=None), dict(a_h=None), dict(a_t=None), dict(tpl=None), dict(r=None),
                    dict(o=None), dict(o=C.byref(none))):
            assert call(**bad) == INVALID, bad
        for maxd in (np.nan, -1.0, -np.inf, -1e-300, -5e-324):
            assert call(maxd=maxd) == INVALID, maxd
    assert not cnt.any() and not kind.any() and not dist.any() and not first.any()
