"""Pairs whose GJK ends in a later primitive-pair pass are finished by that pass and give the oracle's bits.

With HFB_GJK_PASSES="1" the first pass runs one iteration, so nearly every GJK-routed pair ends in the last pass,
which writes its result record (witness points from the simplex's support points in shared memory) or its EPA queue
item.  Covered: distance with signed distance (EPA for the penetrating pairs), the warm-start outputs and a second
call that reads them back as cached guesses, collide with contacts (EPA) and without (`Collision` rows that keep the
cached guess they came with).
"""
import numpy as np
import pytest

from tests.common import P, compare_distance, make_scenes
from hppfcl_b200 import workloads as W

pytestmark = pytest.mark.gpu

ALL_PRIMS = (P.GEOM_SPHERE, P.GEOM_CAPSULE, P.GEOM_BOX, P.GEOM_CYLINDER, P.GEOM_CONE, P.GEOM_ELLIPSOID)


def _same_guesses(want, have, what):
    (rg, rh), (gg, gh) = want, have
    assert np.array_equal(rg.view(np.uint64), gg.view(np.uint64)), "%s: cached guesses differ" % what
    assert np.array_equal(rh, gh), "%s: support hints differ" % what


def test_pairs_finished_by_the_last_pass(monkeypatch):
    monkeypatch.setenv("HFB_GJK_PASSES", "1")
    sc = make_scenes(gpu=True, emu=False)
    w = W.config2_mixed_primitives(100_000, pool=4096, types=ALL_PRIMS, seed=11)
    sc.register_shapes(w["shapes"])
    sc.commit()
    rows = (w["h1"], w["tf1"], w["h2"], w["tf2"])

    ref, rg, rh = sc.b["oracle"].batch_distance(*rows, want_guess=True, nthreads=0)
    got, gg, gh = sc.b["gpu"].batch_distance(*rows, want_guess=True)
    compare_distance(ref, got, what="distance")
    _same_guesses((rg, rh), (gg, gh), "distance")
    gjk = ((ref["status"] >> 16) & 0xff) == 0
    assert ((ref["iterations"] & 0xffff)[gjk] > 1).mean() > 0.9  # ended after the first pass
    assert (ref["min_distance"] < 0).sum() > 1000  # pairs reach EPA

    req = P.DistanceRequestPOD(gjk_initial_guess=P.CachedGuess)
    req.q.cached_gjk_guess = rg.ctypes.data
    req.q.cached_support_func_guess = rh.ctypes.data
    ref2, rg2, rh2 = sc.b["oracle"].batch_distance(*rows, req, want_guess=True, nthreads=0)
    got2, gg2, gh2 = sc.b["gpu"].batch_distance(*rows, req, want_guess=True)
    compare_distance(ref2, got2, what="distance from cached guesses")
    _same_guesses((rg2, rh2), (gg2, gh2), "distance from cached guesses")

    for contact in (1, 0):
        req = P.CollisionRequestPOD(security_margin=0.05, enable_contact=contact, gjk_initial_guess=P.CachedGuess)
        req.q.cached_gjk_guess = rg.ctypes.data
        req.q.cached_support_func_guess = rh.ctypes.data
        ref3, rg3, rh3 = sc.b["oracle"].batch_collide(*rows, req, want_guess=True, nthreads=0)
        got3, gg3, gh3 = sc.b["gpu"].batch_collide(*rows, req, want_guess=True)
        what = "collide, enable_contact=%d" % contact
        compare_distance(ref3, got3, what=what)
        _same_guesses((rg3, rh3), (gg3, gh3), what)
        assert (ref3["num_contacts"] > 0).sum() > 1000
