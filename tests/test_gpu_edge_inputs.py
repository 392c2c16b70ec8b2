"""The kernels at the edges.

A. The edge-input suites of tests/test_fuzz_reference.py (zero sizes, extreme request fields, translations up to 1e100,
   hulls at the linear-scan threshold, NaN and +-Inf poses), run as they are with the kernels in the place of the host
   build of the device code: the same inputs, calls and exclusions, against the oracle (which those CPU tests pin to
   the reference build on exactly these inputs).  Their distance calls run once more with signed distance and each GJK
   variant (the passes are compiled once per variant).
B. Iteration caps and budgets at the launch boundaries: GJK caps that end in, at and after a pass of the primitive-pair
   GJK passes under the default schedule, HFB_GJK_PASSES=3,3,4, =1 and =0 (the single kernel); EPA caps around tier
   0's 24 iterations, with no, one and fewer continuation records than outgrown pairs (HFB_EPA_RESUME); GJK caps around
   the 6 iterations of a leaf item of the mesh-shape task system (HFB_BVH_GJK_CHUNK).  The batch and the requests are
   those of tests/test_launch_boundaries.py, which pins oracle == reference build on them.
C. Poses displaced by 1e6 ... 1e100 and poses with a NaN or an infinity through the device broadphase: scene boxes,
   the self and cross pair finders, hfb_scene_collide_sets and the resident environment.

After every call, no kernel of the context may have given up on a spin wait (stats()["watchdog_trips"]).
"""
import numpy as np
import pytest

import hppfcl_b200 as hf
from oracle import oracle_lib
from tests import common
from tests import test_fuzz_reference as F
from tests import test_launch_boundaries as B
from tests.common import MultiScene, P, compare_distance, make_scenes
from tests.test_broadphase import brute_pairs
from tests.test_broadphase_sets import brute_cross
from hppfcl_b200 import workloads as W

pytestmark = pytest.mark.gpu


def no_watchdog(sc):
    assert sc.b["gpu"].stats()["watchdog_trips"] == 0


# ------------------------------------------------------------------------------------------------------------- A
class KernelsForTheHostBuild:
    """the engine in the place of the host build of the device code in a CPU suite of tests/test_fuzz_reference.py:
    the suite's own calls and comparisons run on the kernels.  Every distance call runs again with signed distance and
    each GJK variant against the oracle (non-finite poses: on the fields that suite compares); no watchdog trip after
    any call.  Registrations and commit go to the engine."""

    def __init__(self, eng, orc, non_finite):
        self.eng, self.orc, self.non_finite = eng, orc, non_finite

    def __getattr__(self, name):
        return getattr(self.eng, name)

    def _run(self, fn, args):
        got = getattr(self.eng, fn)(*args)
        assert self.eng.stats()["watchdog_trips"] == 0
        return got

    def batch_collide(self, *args):
        return self._run("batch_collide", args)

    def batch_distance(self, *args):
        got = self._run("batch_distance", args)
        for r in variant_requests(args[4]):
            what = "signed distance, variant %d" % r.q.gjk_variant
            ro = self.orc.batch_distance(*args[:4], r, nthreads=0)
            g = self._run("batch_distance", args[:4] + (r,))
            if not self.non_finite:
                compare_distance(ro, g, exact=True, what=what)
                continue
            walk = ((ro["status"] >> 16) & 0xff) == P.PATH_BVH
            same_fields(ro[~walk], g[~walk], ("status", "iterations", "min_distance"), what)
            same_fields(ro[walk], g[walk], ("min_distance", "b1", "b2"), what + ", mesh walks")
        return got


def variant_requests(req):
    """`req` with signed distance and each of the three GJK variants (those that differ from `req`)"""
    out = []
    for v in B.VARIANTS:
        r = P.DistanceRequestPOD.from_buffer_copy(bytes(req))
        r.enable_signed_distance = 1
        r.q.gjk_variant = v
        if bytes(r) != bytes(req):
            out.append(r)
    return out


def same_fields(a, b, fields, what=""):
    """the fields equal row by row, a NaN equal to a NaN"""
    for fld in fields:
        x, y = a[fld], b[fld]
        ok = (x == y) | (np.isnan(x) & np.isnan(y)) if x.dtype.kind == "f" else x == y
        assert np.all(ok), "%s: field %s differs at rows %s" % (what, fld, np.unique(np.nonzero(~ok)[0])[:8])


SUITES = ("test_degenerate_sizes", "test_extreme_request_fields", "test_huge_translations",
          "test_hulls_at_the_linear_scan_threshold", "test_non_finite_poses_terminate")


@pytest.mark.parametrize("suite", SUITES)
def test_edge_input_suite_on_the_gpu(suite, monkeypatch):
    """the suite exactly as it runs on the CPU -- its inputs, its calls, its exclusions -- with the kernels where the
    host build of the device code was; the reference build takes no part (the CPU suite pins oracle == reference
    build on these inputs)"""
    def scenes(gpu=False, emu=True, ref=False):
        orc = oracle_lib.OracleScene(P)
        return MultiScene({"oracle": orc, "emu": KernelsForTheHostBuild(hf.Engine(0), orc, suite == SUITES[-1])})
    monkeypatch.setattr(common, "make_scenes", scenes)
    getattr(F, suite)()


# ------------------------------------------------------------------------------------------------------------- B
_ORACLE = {}  # the oracle's records of the boundary batch by call and request (the batch is the same in every test)


def boundary_scene(monkeypatch, knobs):
    """the boundary batch registered in the oracle and in an engine created under `knobs` -> (sc, h1, t1, h2, t2, ns)"""
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)
    sc = make_scenes(gpu=True, emu=False)
    return (sc,) + B.boundary_batch(sc)


def oracle_rows(sc, fn, args):
    key = (fn, len(args[0]), bytes(args[4]))
    if key not in _ORACLE:
        _ORACLE[key] = getattr(sc.b["oracle"], fn)(*args, nthreads=0)
    return _ORACLE[key]


def compare_on_gpu(sc, fn, args, what):
    ro = oracle_rows(sc, fn, args)
    compare_distance(ro, getattr(sc.b["gpu"], fn)(*args), exact=True, what=what)
    no_watchdog(sc)
    return ro


SCHEDULES = {"default": (None, B.GJK_CAPS), "3,3,4": ("3,3,4", B.GJK_CAPS_3_3_4), "1": ("1", B.GJK_CAPS),
             "0": ("0", B.GJK_CAPS)}


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
def test_gjk_caps_at_the_pass_boundaries(schedule, monkeypatch):
    passes, caps = SCHEDULES[schedule]
    monkeypatch.delenv("HFB_GJK_PASSES", raising=False)
    sc, h1, t1, h2, t2, ns = boundary_scene(monkeypatch, {} if passes is None else {"HFB_GJK_PASSES": passes})
    for fn in ("batch_distance", "batch_collide"):
        for cap in caps:
            hit = 0
            for v in B.VARIANTS:
                ro = compare_on_gpu(sc, fn, (h1, t1, h2, t2, B.gjk_cap_request(fn, cap, v)),
                                    "passes %s, %s, cap %d, variant %d" % (schedule, fn, cap, v))
                hit += B.failed_at(ro[:ns], cap)
            assert hit > 0, "%s: no pair reaches the cap of %d" % (fn, cap)


def outgrown_pairs(sc, args):
    """pairs whose EPA reached iteration 24 under the cap of 64: each of them outgrew tier 0's workspace (more may
    have, out of face slots earlier)"""
    ro = oracle_rows(sc, "batch_distance", args)
    return int(((ro["iterations"] >> 16) >= B.EPA_SMALL_IT).sum())


@pytest.mark.parametrize("resume", ["default", "0", "1", "fewer_than_outgrown"])
def test_epa_caps_around_tier_0_and_the_continuation_budget(resume, monkeypatch):
    monkeypatch.delenv("HFB_EPA_RESUME", raising=False)
    knobs = {}
    if resume == "fewer_than_outgrown":
        sc0 = make_scenes(emu=False)
        h1, t1, h2, t2, ns = B.boundary_batch(sc0)
        n_out = outgrown_pairs(sc0, (h1[:ns], t1[:ns], h2[:ns], t2[:ns], B.epa_cap_request("batch_distance", 64)))
        k = n_out - max(2, n_out // 10)
        assert 0 < k < n_out  # a batch of resumed and restarted pairs
        knobs["HFB_EPA_RESUME"] = str(k)
    elif resume != "default":
        knobs["HFB_EPA_RESUME"] = resume
    sc, h1, t1, h2, t2, ns = boundary_scene(monkeypatch, knobs)
    for fn in ("batch_distance", "batch_collide"):
        for cap in B.EPA_CAPS:
            ro = compare_on_gpu(sc, fn, (h1, t1, h2, t2, B.epa_cap_request(fn, cap)),
                                "resume %s, %s, EPA cap %d" % (resume, fn, cap))
            if cap > B.EPA_SMALL_IT:
                assert ((ro["iterations"][:ns] >> 16) >= B.EPA_SMALL_IT).sum() > 10


@pytest.mark.parametrize("chunk", ["default", "1"])
def test_gjk_caps_around_the_leaf_item_chunk(chunk, monkeypatch):
    monkeypatch.delenv("HFB_BVH_GJK_CHUNK", raising=False)
    sc, h1, t1, h2, t2, ns = boundary_scene(monkeypatch, {} if chunk == "default" else {"HFB_BVH_GJK_CHUNK": chunk})
    mesh = (h1[ns:], t1[ns:], h2[ns:], t2[ns:])
    for fn in ("batch_distance", "batch_collide"):
        for cap in B.BVH_CAPS:
            for v in B.VARIANTS:
                compare_on_gpu(sc, fn, mesh + (B.gjk_cap_request(fn, cap, v),),
                               "chunk %s, %s mesh pairs, cap %d, variant %d" % (chunk, fn, cap, v))


# ------------------------------------------------------------------------------------------------------------- C
NONFINITE_FIELDS = ("status", "iterations", "num_contacts", "distance_lower_bound")  # part A's collide fields


def overlap_pairs(ba, bb):
    """AABB::overlap over every (i, j): a box is apart only where a comparison says so -- a NaN coordinate never
    does (brute_pairs / brute_cross, which ask the opposite question, part ways with it on such boxes only)"""
    apart = np.any((ba[:, None, :3] > bb[None, :, 3:]) | (ba[:, None, 3:] < bb[None, :, :3]), axis=2)
    i, j = np.nonzero(~apart)
    return set(zip(i.tolist(), j.tolist()))


def edge_scene(sc, rng, n=3000):
    """n objects: primitives and a 32-vertex hull at ordinary poses in a 12 m cube, 5 % of them displaced by 1e6, 1e15
    or 1e100, 2 % with a NaN or an infinity in a translation or rotation entry; a Halfspace floor as object 0"""
    prims = W.random_primitive_shapes(rng, 48, B.ALL_PRIMS)
    hp = sc.register_shapes(prims)
    pts, tris = W.ellipsoid_hull(rng, 32, radii=(0.3, 0.4, 0.5))
    cid = sc.register_convex(pts, tris)
    hc = sc.register_shapes(P.make_shapes([P.GEOM_CONVEX], [[0, 0, 0]], data=[cid]))
    floor = sc.register_halfspaces(P.GEOM_HALFSPACE, [[0, 0, 1, -2.0]])
    sc.commit()
    pool = np.concatenate([hp, hc])
    oh = pool[rng.integers(0, len(pool), n)].astype(np.uint32)
    tf = W.random_transforms(rng, n, (-6, -6, -6), (6, 6, 6))
    oh[0] = floor[0]
    tf[0] = W.identity_transforms(1)[0]
    far = 1 + rng.choice(n - 1, n // 20, replace=False)
    tf["T"][far] += rng.choice([1e6, 1e15, 1e100], (len(far), 1)) * rng.normal(size=(len(far), 3))
    tf["T"][far[:10]] = tf["T"][far[10]]  # a few of them together out there
    bad = 1 + rng.choice(np.setdiff1d(np.arange(n - 1), far - 1), n // 50, replace=False)
    vals = rng.choice([np.nan, np.inf, -np.inf], len(bad))
    which = rng.integers(0, 12, len(bad))
    for i, v, k in zip(bad, vals, which):
        if k < 3:
            tf["T"][i, k] = v
        else:
            tf["R"][i, k - 3] = v
    return oh, tf, far, bad


def same_boxes(a, b):
    """bit for bit; a NaN equal to a NaN"""
    both_nan = np.isnan(a) & np.isnan(b)
    return np.array_equal(a.view(np.uint64)[~both_nan], b.view(np.uint64)[~both_nan]) and \
        np.array_equal(np.isnan(a), np.isnan(b))


def records_match(orc, pairs, rec, ha, tfa, hb, tfb, finite):
    """the records of (i in A, j in B) pairs against the oracle's batch_collide rows: whole records where both poses
    are finite, part A's fields of a non-finite pose's rows elsewhere"""
    if len(pairs) == 0:
        return
    i, j = np.array([p[0] for p in pairs]), np.array([p[1] for p in pairs])
    ro = orc.batch_collide(ha[i], tfa[i], hb[j], tfb[j], nthreads=0)
    ok = finite[0][i] & finite[1][j]
    compare_distance(ro[ok], rec[ok], exact=True, what="records of finite pairs")
    same_fields(ro[~ok], rec[~ok], NONFINITE_FIELDS, "records of non-finite pairs")


def test_edge_poses_through_the_device_broadphase():
    import torch
    rng = np.random.default_rng(23)
    sc = make_scenes(gpu=True, emu=False)
    eng, orc = sc.b["gpu"], sc.b["oracle"]
    oh, tf, far, bad = edge_scene(sc, rng)
    n = len(oh)
    finite = np.isfinite(tf["T"]).all(axis=1) & np.isfinite(tf["R"]).all(axis=1)
    assert (~finite).sum() == len(bad)

    # scene boxes: device == the library's host function (hfb_scene_aabbs: the same computeAABB, compiled for the
    # host) -- equal to the reference build's on ordinary poses (tests/test_broadphase.py)
    bb = eng.scene_aabbs(oh, tf)

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()

    stream = torch.cuda.current_stream().cuda_stream
    d_h, d_tf = dev(oh), dev(tf)
    d_bb = torch.empty(n * 6, dtype=torch.float64, device="cuda")
    eng.scene_aabbs_device(n, d_h.data_ptr(), d_tf.data_ptr(), d_bb.data_ptr(), stream)
    torch.cuda.synchronize()
    assert same_boxes(d_bb.cpu().numpy().reshape(n, 6), bb)
    assert np.isnan(bb).any(axis=1).sum() > 0 and (np.abs(bb[far]) > 1e90).any()
    no_watchdog(sc)

    # the self pair finder: every i < j whose boxes overlap (AABB::overlap)
    nanbox = np.isnan(bb).any(axis=1)
    want = {p for p in overlap_pairs(bb, bb) if p[0] < p[1]}
    clean = ~nanbox
    idx = np.nonzero(clean)[0]
    assert {(idx[a], idx[b]) for a, b in brute_pairs(bb[clean])} == {p for p in want if clean[p[0]] and clean[p[1]]}
    cap = len(want) + 1000
    d_f = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_s = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int32, device="cuda")
    eng.broadphase_pairs_device(n, d_bb.data_ptr(), d_f.data_ptr(), d_s.data_ptr(), cap, d_n.data_ptr(), stream)
    torch.cuda.synchronize()
    k = int(d_n.item())
    got = set(zip(d_f[:k].cpu().numpy().tolist(), d_s[:k].cpu().numpy().tolist()))
    assert k == len(want) and got == want
    assert any(p[0] == 0 for p in want) and any(nanbox[p[1]] for p in want)
    no_watchdog(sc)

    # the cross pair finder: A = objects 1 .. 799 (a robot's links), B = the floor and the rest
    a_idx = np.arange(1, 800)
    b_idx = np.concatenate([[0], np.arange(800, n)])
    ba, bbb = bb[a_idx], bb[b_idx]
    want_x = overlap_pairs(ba, bbb)
    ca, cb = ~nanbox[a_idx], ~nanbox[b_idx]
    ia, ib = np.nonzero(ca)[0], np.nonzero(cb)[0]
    assert {(ia[a], ib[b]) for a, b in brute_cross(ba[ca], bbb[cb])} == {p for p in want_x if ca[p[0]] and cb[p[1]]}
    d_a, d_b = dev(ba), dev(bbb)
    cap = len(want_x) + 1000
    d_f = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_s = torch.empty(cap, dtype=torch.int32, device="cuda")
    eng.broadphase_cross_pairs_device(len(ba), d_a.data_ptr(), len(bbb), d_b.data_ptr(), d_f.data_ptr(), d_s.data_ptr(),
                                      cap, d_n.data_ptr(), stream)
    torch.cuda.synchronize()
    k = int(d_n.item())
    got = set(zip(d_f[:k].cpu().numpy().tolist(), d_s[:k].cpu().numpy().tolist()))
    assert k == len(want_x) and got == want_x
    no_watchdog(sc)

    # A against B in one call, and the resident environment: the candidates are the pairs above, the records of the
    # colliding ones those of the oracle
    ha, tfa, hb, tfb = oh[a_idx], tf[a_idx], oh[b_idx], tf[b_idx].copy()
    fin = (finite[a_idx], finite[b_idx])

    def expect(tfb_now):
        bx = eng.scene_aabbs(hb, tfb_now)
        cand = sorted(overlap_pairs(ba, bx))
        i, j = np.array([p[0] for p in cand], dtype=np.int64), np.array([p[1] for p in cand], dtype=np.int64)
        ro = orc.batch_collide(ha[i], tfa[i], hb[j], tfb_now[j], nthreads=0)
        return len(cand), {cand[r] for r in np.nonzero(ro["num_contacts"] > 0)[0]}

    def check(res, tfb_now, fin_b):
        f, s, rec, ncand, nhit = res
        want_c, want_hit = expect(tfb_now)
        got_pairs = list(zip(f.tolist(), s.tolist()))
        assert ncand == want_c and nhit == len(want_hit) == len(got_pairs) and set(got_pairs) == want_hit
        records_match(orc, got_pairs, rec, ha, tfa, hb, tfb_now, (fin[0], fin_b))
        no_watchdog(sc)
        return nhit

    big = 1 << 20
    assert check(eng.scene_collide_sets(ha, tfa, hb, tfb, capacity=big), tfb, fin[1]) > 50
    env = eng.env_create(hb, tfb)
    check(eng.env_collide(env, ha, tfa, capacity=big), tfb, fin[1])
    # objects of B moved out to 1e100 and to NaN / infinite poses, then back next to the robot
    moved = rng.choice(np.arange(1, len(hb)), 60, replace=False)
    t = tfb[moved].copy()
    t["T"][:20] = 1e100
    t["T"][20:40, 1] = np.nan
    t["R"][40:50, 4] = np.inf
    t["T"][50:, 2] = -np.inf
    fin_b = fin[1].copy()
    fin_b[moved[20:]] = False
    tfb[moved] = t
    eng.env_update(env, moved, t)
    check(eng.env_collide(env, ha, tfa, capacity=big), tfb, fin_b)
    back = tfa[rng.choice(len(tfa), 60)].copy()
    tfb[moved] = back
    fin_b[moved] = np.isfinite(back["T"]).all(axis=1) & np.isfinite(back["R"]).all(axis=1)
    eng.env_update(env, moved, back)
    assert check(eng.env_collide(env, ha, tfa, capacity=big), tfb, fin_b) > 50
    eng.env_destroy(env)
