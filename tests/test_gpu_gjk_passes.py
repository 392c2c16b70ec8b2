"""The primitive-pair GJK passes under their optional settings give the oracle's bits.

HFB_GJK_PASSES="3,3,4" runs four passes (3, 3 and 4 iterations, then to convergence), so the loop state of the
running pairs goes through both ping-ponged buffers and back into the first; HFB_EPA_OVERLAP=1 extracts the pairs the
first pass finished at once (the `done` flags) and starts their EPA next to the remaining passes.  The Polyak and
Nesterov variants carry their momentum terms across passes; signed distance sends the penetrating pairs to EPA
through the finished-pair state.
"""
import pytest

from tests.common import P, compare_distance, make_scenes
from hppfcl_b200 import workloads as W

pytestmark = pytest.mark.gpu

ALL_PRIMS = (P.GEOM_SPHERE, P.GEOM_CAPSULE, P.GEOM_BOX, P.GEOM_CYLINDER, P.GEOM_CONE, P.GEOM_ELLIPSOID)

SETTINGS = {
    "four_passes": {"HFB_GJK_PASSES": "3,3,4"},
    "epa_overlap": {"HFB_EPA_OVERLAP": "1"},
    "four_passes_epa_overlap": {"HFB_GJK_PASSES": "3,3,4", "HFB_EPA_OVERLAP": "1"},
}


@pytest.mark.parametrize("setting", sorted(SETTINGS))
def test_gjk_pass_settings(setting, monkeypatch):
    for k, v in SETTINGS[setting].items():
        monkeypatch.setenv(k, v)
    sc = make_scenes(gpu=True, emu=False)
    w = W.config2_mixed_primitives(100_000, pool=4096, types=ALL_PRIMS)
    sc.register_shapes(w["shapes"])
    sc.commit()
    rows = (w["h1"], w["tf1"], w["h2"], w["tf2"])
    for variant in (P.DefaultGJK, P.PolyakAcceleration, P.NesterovAcceleration):
        req = P.DistanceRequestPOD(gjk_variant=variant)
        ref = sc.b["oracle"].batch_distance(*rows, req, nthreads=0)
        got = sc.b["gpu"].batch_distance(*rows, req)
        compare_distance(ref, got, what="%s variant %d" % (setting, variant))
        assert (ref["min_distance"] < 0).sum() > 1000  # pairs reach EPA
        assert ((ref["iterations"] & 0xffff) > 10).sum() > 1000  # pairs reach the fourth pass of "3,3,4"
    req = P.CollisionRequestPOD(security_margin=0.05)
    ref = sc.b["oracle"].batch_collide(*rows, req, nthreads=0)
    got = sc.b["gpu"].batch_collide(*rows, req)
    compare_distance(ref, got, what="%s collide" % setting)
