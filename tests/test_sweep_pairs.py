"""hfb_broadphase_sweep_pairs, the self candidates of the motion certification, against its definition computed
exactly with fractions.Fraction (include/hppfcl_b200.h, hfb_env_certify_motions): a side is a sweep bound that is
finite and >= 0 where the segment exists; a self pair's thresholds are the sums of its links' sides rounded up; its
reach w is half the larger valid threshold rounded up; the pair is a candidate when both links have a box and, unless
both boxes are finite, j's box overlaps i's box widened by w, rounded outward.  The device kernel shares the predicate
(sweep_pair of hfb_broadphase.cuh), so this pins its rounding.  No GPU needed."""
import math
from fractions import Fraction

import numpy as np

from tests.common import hf

DMAX = np.finfo(np.float64).max
EMPTY = [DMAX, DMAX, DMAX, -DMAX, -DMAX, -DMAX]
TINY = 5e-324


def ru(x):
    """the smallest double >= x (x a Fraction)"""
    if x > Fraction(DMAX):
        return math.inf
    if x < -Fraction(DMAX):
        return -DMAX
    d = float(x)
    return d if Fraction(d) >= x else math.nextafter(d, math.inf)


def rd(x):
    return -ru(-x)


def side(s):
    return s if math.isfinite(s) and s >= 0 else None


def reference(bb, sweep, links, tpl, off, m0, nm):
    """the candidates, configuration by configuration in template order, by exact arithmetic"""
    sides = {}
    for m in range(m0, m0 + nm):
        for g in range(int(off[m]), int(off[m + 1])):
            for i in range(links):
                o = g * links + i
                r = side(sweep[o]) if g + 1 < off[m + 1] else None
                left = side(sweep[o - links]) if g > off[m] else None
                sides[o] = (r, left)
    out = []
    for g in range(int(off[m0]), int(off[m0 + nm])):
        for i, j in tpl:
            a, b = g * links + int(i), g * links + int(j)
            x, y = bb[a], bb[b]
            if list(x) == EMPTY[:6] or list(y) == EMPTY[:6] or (x[0] == DMAX and x[3] == -DMAX) or \
                    (y[0] == DMAX and y[3] == -DMAX):
                continue
            if not (np.isfinite(x).all() and np.isfinite(y).all()):
                out.append((a, b))
                continue
            th = []
            for k in range(2):
                sa, sb = sides[a][k], sides[b][k]
                if sa is not None and sb is not None:
                    th.append(ru(Fraction(sa) + Fraction(sb)))
            if th and max(th) == math.inf:  # (a sum past DBL_MAX: the reach is infinite, the box everything)
                out.append((a, b))
                continue
            w = ru(Fraction(max(th)) / 2) if th else 0.0
            lo = [rd(Fraction(x[c]) - Fraction(w)) for c in range(3)]
            hi = [ru(Fraction(x[3 + c]) + Fraction(w)) for c in range(3)]
            if all(lo[c] <= y[3 + c] and hi[c] >= y[c] for c in range(3)):
                out.append((a, b))
    return out


def library(bb, sweep, links, tpl, off, m0=0, nm=None, capacity=None):
    f, s = hf.broadphase_sweep_pairs(bb, sweep, links, tpl, off, m0, nm, capacity)
    return list(zip(f.tolist(), s.tolist()))


def two_links(gap_x, size=1.0, lo0=0.0):
    """link 0's box [lo0, lo0 + size] on x, link 1's box starting gap_x after it; y and z overlap"""
    return [lo0, 0, 0, lo0 + size, 1, 1], [lo0 + size + gap_x, 0, 0, lo0 + size + gap_x + 1, 1, 1]


def build(configs):
    """configs: [(box0, box1, sweep0, sweep1)] -> (bb, sweep)"""
    bb = np.array([b for c in configs for b in c[:2]], dtype=np.float64)
    sw = np.array([s for c in configs for s in c[2:]], dtype=np.float64)
    return bb, sw


def check(configs, off, tpl=((0, 1),), m0=0, nm=None):
    bb, sw = build(configs)
    off = np.asarray(off, dtype=np.uint32)
    nm = len(off) - 1 - m0 if nm is None else nm
    want = reference(bb, sw, 2, tpl, off, m0, nm)
    got = library(bb, sw, 2, tpl, off, m0, nm)
    assert got == want
    return got


def test_gap_at_the_reach_and_one_ulp_either_side():
    # one motion of two samples: at sample 0 only the right side, at sample 1 only the left; threshold 0.25 + 0.25,
    # reach 0.25: a gap of exactly 0.25 is a candidate (closed intervals), one ulp more is not
    for lo1, want in ((1.25, True), (math.nextafter(1.25, 0), True), (math.nextafter(1.25, 2), False)):
        boxes = ([0, 0, 0, 1, 1, 1], [lo1, 0, 0, lo1 + 1, 1, 1])  # link 0's box ends at 1: the gap is lo1 - 1
        got = check([(*boxes, 0.25, 0.25), (*boxes, 7.0, 7.0)], [0, 2])
        assert ((0, 1) in got) == want
        assert ((2, 3) in got) == want  # the left side of sample 1 is sample 0's bound


def test_rounding_upward_where_nearest_differs():
    # 1 + 2^-60 rounds to 1 at nearest, to 1 + 2^-52 upward: the reach is (1 + 2^-52) / 2
    s1, s2 = 1.0, 2.0 ** -60
    w = (1.0 + 2.0 ** -52) / 2
    for gap in (w, math.nextafter(w, 0), math.nextafter(w, 1), 0.5):
        check([(*two_links(gap, lo0=0.3), s1, s2), (*two_links(gap), 0.0, 0.0)], [0, 2])
    got = check([(*two_links(math.nextafter(0.5, 1), lo0=0.3), s1, s2), (*two_links(9.0), 0.0, 0.0)], [0, 2])
    assert got == [(0, 1)]  # a nearest sum would have missed it
    # widening a coordinate that is not a multiple of w's ulp: the outward rounding decides
    for lo0 in (0.1, 1e-3, 12345.678, -0.7):
        for gap in (0.1, math.nextafter(0.1, 1), 0.3):
            check([(*two_links(gap, size=0.3, lo0=lo0), 0.05, 0.05), (*two_links(gap, lo0=lo0), 0.1, 0.0)], [0, 2])


def test_subnormal_sweeps():
    for s in (TINY, 3 * TINY, 2.0 ** -1060, 2.0 ** -1022):
        for gap in (0.0, TINY, 2 * TINY, s, math.nextafter(s, 1)):
            check([(*two_links(gap), s, 0.0), (*two_links(gap), s, s)], [0, 2])
    got = check([(*two_links(TINY), TINY, 0.0), (*two_links(1.0), 0.0, 0.0)], [0, 2])
    assert got == [(0, 1)]  # half of the smallest subnormal, rounded up, is itself


def test_invalid_sweeps_widen_nothing():
    for bad in (math.nan, -1.0, -TINY, math.inf, -math.inf):
        got = check([(*two_links(0.1), bad, 10.0), (*two_links(0.1), 10.0, 10.0)], [0, 2])
        assert got == []  # neither sample is widened: the right side of 0 and the left of 1 are one bound
    got = check([(*two_links(0.0), math.nan, 1.0), (*two_links(0.1), 1.0, 1.0)], [0, 2])
    assert got == [(0, 1)]  # overlapping boxes stay candidates
    assert check([(*two_links(0.1), -0.0, 0.4), (*two_links(0.1), 0.0, 0.0)], [0, 2]) == [(0, 1), (2, 3)]  # -0 is valid


def test_first_middle_and_last_samples():
    # a three-sample motion: the middle one takes the larger of its two sides, the last one's own bound is not read
    cfg = [(*two_links(0.3), 0.2, 0.2), (*two_links(0.3), 0.35, 0.35), (*two_links(0.3), 100.0, 100.0)]
    assert check(cfg, [0, 3]) == [(2, 3), (4, 5)]
    # ... and split into one-sample motions nothing is widened
    assert check(cfg, [0, 1, 2, 3]) == []
    assert check(cfg, [0, 0, 3, 3]) == [(2, 3), (4, 5)]  # empty motions around it


def test_empty_and_non_finite_boxes():
    far = [50, 0, 0, 51, 1, 1]
    for box in (EMPTY, [math.inf, 0, 0, math.inf, 1, 1], [math.nan] * 6, [0, 0, 0, math.inf, 1, 1]):
        got = check([(list(box), far, 1.0, 1.0), (far, list(box), 1.0, 1.0)], [0, 2])
        assert got == ([] if box is EMPTY else [(0, 1), (2, 3)])


def test_random_layouts_ranges_and_capacity():
    rng = np.random.default_rng(11)
    pool = [0.0, TINY, 2.0 ** -1060, 0.1, 0.25, 1.0, 2.0 ** -60, math.nan, -1.0, math.inf, 1e308, DMAX]
    for trial in range(40):
        sizes = rng.integers(0, 5, rng.integers(1, 6))
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
        n = int(off[-1])
        links = 3
        lo = rng.uniform(-1, 1, (n * links, 3))
        ext = rng.choice([0.0, 0.1, 0.5], (n * links, 3))
        bb = np.concatenate([lo, lo + ext], axis=1)
        bb[rng.random(n * links) < 0.05] = EMPTY
        sw = np.where(rng.random(n * links) < 0.5, rng.choice(pool, n * links), rng.uniform(0, 1.5, n * links))
        tpl = [(0, 2), (1, 0), (2, 1)]
        nmot = len(off) - 1
        m0 = int(rng.integers(0, nmot + 1))
        nm = int(rng.integers(0, nmot - m0 + 1))
        want = reference(bb, sw, links, tpl, off, m0, nm)
        assert library(bb, sw, links, tpl, off, m0, nm) == want
        if want:
            cap = len(want) // 2
            f, s = hf.broadphase_sweep_pairs(bb, sw, links, tpl, off, m0, nm, capacity=cap)
            assert list(zip(f.tolist(), s.tolist())) == want[:cap]
