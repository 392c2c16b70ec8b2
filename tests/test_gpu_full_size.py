"""The device-pointer batch calls at the sizes bench.py runs them, with every pair class past the grid cap of its
kernel, so that the second and later trips of each grid-stride loop are compared with something.

Every batch kernel caps its grid and strides over the rest; the host entry points cut a batch into chunks that (at
the default lane widths) never reach a cap, so only the *_device forms launch a whole batch at once.  The caps follow
from the SM count and the launch constants below; each test asserts that its batch holds at least twice the cap of
every class it is about, counted from the path byte of the records, and prints the counts.

References: the oracle on every row (bit for bit, tests.common.compare_distance), the host form of the same call
(the bytes of the whole output), and, where oracle/_ref was built, the reference build on a seeded sample."""
import time
import types

import numpy as np
import pytest

from tests.common import P, compare_distance, hf, ref_agrees
from tests.test_convex_support_ref import edge_hulls, pad_hulls, support_ref
from hppfcl_b200 import workloads as W
from oracle import oracle_lib

pytestmark = pytest.mark.gpu

# launch constants of the capped grids
PASS_THREADS = 128          # hfb_gjkpass.cu:36 (PASS_THREADS)
PASS_BLOCKS_FIRST = 4       # hfb_gjkpass.cu:36-37: k_gjk_first, default variant (4 blocks per SM)
PASS_BLOCKS_MOMENTUM = 3    # hfb_gjkpass.cu:36-37: Polyak / Nesterov (PASS_BLOCKS_PER_SM)
PASS_WAVES = 16             # hfb_gjkpass.cu:388-393: at most 16 waves of resident blocks
PAIRS_THREADS = 128         # hfb_kernels.cu:970-977: k_pairs, 128 threads, G lanes per pair
PAIRS_BLOCKS_PER_SM = 32    # hfb_kernels.cu:976


def grid_caps(gc=2):
    """pairs per trip of each capped grid-stride loop on device 0 (gc: lanes per hull / triangle pair, HFB_GC)"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return {"gjk_default": sms * PASS_BLOCKS_FIRST * PASS_WAVES * PASS_THREADS,
            "gjk_momentum": sms * PASS_BLOCKS_MOMENTUM * PASS_WAVES * PASS_THREADS,
            "closed": sms * PAIRS_BLOCKS_PER_SM * PAIRS_THREADS,
            "hull": sms * PAIRS_BLOCKS_PER_SM * (PAIRS_THREADS // gc)}


def assert_past_cap(what, count, cap):
    print("%s: %d pairs, %.2f x its grid cap of %d" % (what, count, count / cap, cap))
    assert count >= 2 * cap, "%s: %d pairs do not reach twice the grid cap (%d)" % (what, count, cap)


def path_counts(status):
    path = P.status_path(status)
    return {"gjk": int((path == P.PATH_GJK).sum()), "closed": int((path == P.PATH_CLOSED_FORM).sum()),
            "bvh": int((path == P.PATH_BVH).sum()), "unsupported": int((path == P.PATH_UNSUPPORTED).sum())}


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()


class Rows:
    """a batch of pair rows on the host and on the device"""

    def __init__(self, h1, tf1, h2, tf2):
        self.h = (np.ascontiguousarray(h1, dtype=np.uint32), np.ascontiguousarray(tf1, dtype=P.transform_dtype),
                  np.ascontiguousarray(h2, dtype=np.uint32), np.ascontiguousarray(tf2, dtype=P.transform_dtype))
        self.d = [dev(a) for a in self.h]
        self.n = len(self.h[0])

    def device(self, eng, kind, req, out=None, stream=None, guess=None, n=None):
        """the *_device call into `out` (a new buffer if None) on `stream` (the current one if None); no sync"""
        import torch
        dt = P.distance_result_dtype if kind == "distance" else P.contact_dtype
        n = self.n if n is None else n
        if out is None:
            out = torch.empty(max(n, 1) * dt.itemsize, dtype=torch.uint8, device="cuda")
        s = (stream or torch.cuda.current_stream()).cuda_stream
        fn = eng.batch_distance_device if kind == "distance" else eng.batch_collide_device
        fn(n, self.d[0].data_ptr(), self.d[1].data_ptr(), self.d[2].data_ptr(), self.d[3].data_ptr(), out.data_ptr(), req,
           stream=s, d_guess=guess)
        return out

    def host(self, sc, kind, req, **kw):
        return getattr(sc, "batch_" + kind)(*self.h, req, **kw)


def records(t, kind, n=None):
    import torch
    torch.cuda.synchronize()
    dt = P.distance_result_dtype if kind == "distance" else P.contact_dtype
    r = t.cpu().numpy().view(dt)
    return r if n is None else r[:n]


def no_watchdog_trip(eng):
    assert eng.stats()["watchdog_trips"] == 0


def reference_scene():
    """the reference build where oracle/_ref exists, else None (its recorded outputs cover the CPU tests only)"""
    return oracle_lib.RefScene(P) if oracle_lib.ref_available() else None


def ref_sample(ref, fn, ro, rows, args, what, fields=None):
    if ref is not None:
        ref_agrees(types.SimpleNamespace(b={"ref": ref}), fn, ro[rows], tuple(a[rows] for a in args[:4]) + args[4:],
                   what, fields=fields)


def sample_rows(n, k, seed):
    return np.sort(np.random.default_rng(seed).choice(n, min(k, n), replace=False))


# ---------------------------------------------------------------------------------------------------------------------
# config 2: every primitive type, past the GJK-pass and closed-form caps.  Spheres and capsules are drawn twice as
# often as the other four types, so that closed-form pairs (sphere-{sphere,capsule,box,cylinder}, capsule-capsule:
# 3/8 of the pairs) and GJK-routed ones (5/8) both reach twice their caps in one batch of 3.6 M rows.
C2_ROWS = 3_600_000
C2_TYPES = (P.GEOM_SPHERE, P.GEOM_SPHERE, P.GEOM_CAPSULE, P.GEOM_CAPSULE, P.GEOM_BOX, P.GEOM_CYLINDER, P.GEOM_CONE,
            P.GEOM_ELLIPSOID)


@pytest.fixture(scope="module")
def c2():
    t0 = time.perf_counter()
    w = W.config2_mixed_primitives(C2_ROWS, seed=0xFC1 + 20, types=C2_TYPES)
    eng = hf.Engine(0)
    orc = oracle_lib.OracleScene(P)
    ref = reference_scene()
    hs = eng.register_shapes(w["shapes"])
    assert np.array_equal(hs, orc.register_shapes(w["shapes"]))
    if ref is not None:
        ref.register_shapes(w["shapes"])
    eng.commit()
    rows = Rows(hs[w["h1"]], w["tf1"], hs[w["h2"]], w["tf2"])
    ro = rows.host(orc, "distance", P.DistanceRequestPOD(), nthreads=0)
    counts = path_counts(ro["status"])
    print("config 2 (%d rows): %s; set up in %.1f s" % (rows.n, counts, time.perf_counter() - t0))
    return types.SimpleNamespace(w=w, eng=eng, orc=orc, ref=ref, hs=hs, rows=rows, ro_default=ro, counts=counts,
                                 shapes=w["shapes"])


@pytest.mark.parametrize("variant", [P.DefaultGJK, P.NesterovAcceleration, P.PolyakAcceleration])
def test_config2_distance_past_the_pass_and_closed_form_caps(c2, variant):
    t0 = time.perf_counter()
    caps = grid_caps()
    assert c2.rows.n == C2_ROWS and c2.counts["unsupported"] == 0 and c2.counts["bvh"] == 0
    assert_past_cap("config 2, GJK-routed, variant %d" % variant, c2.counts["gjk"],
                    caps["gjk_default" if variant == P.DefaultGJK else "gjk_momentum"])
    assert_past_cap("config 2, closed form", c2.counts["closed"], caps["closed"])
    req = P.DistanceRequestPOD(gjk_variant=variant)
    got = records(c2.rows.device(c2.eng, "distance", req), "distance")
    no_watchdog_trip(c2.eng)
    ro = c2.ro_default if variant == P.DefaultGJK else c2.rows.host(c2.orc, "distance", req, nthreads=0)
    compare_distance(ro, got, what="config 2 device distance, variant %d" % variant)
    assert (ro["min_distance"] < 0).sum() > 100_000  # EPA runs on many rows
    host = c2.rows.host(c2.eng, "distance", req)
    assert host.tobytes() == got.tobytes(), "device form and host form differ"
    no_watchdog_trip(c2.eng)
    ref_sample(c2.ref, "batch_distance", ro, sample_rows(c2.rows.n, 100_000, variant), c2.rows.h + (req,),
               "config 2 distance variant %d" % variant)
    print("variant %d: %d rows against the oracle (all), the host form (all); %.1f s"
          % (variant, c2.rows.n, time.perf_counter() - t0))


@pytest.mark.parametrize("margin", [0.0, 0.05, -np.inf])
def test_config2_collide_past_the_caps(c2, margin):
    import torch
    t0 = time.perf_counter()
    req = P.CollisionRequestPOD(security_margin=margin)
    side = torch.cuda.Stream()  # (security_margin = -inf: k_clear_contacts runs on the stream the call names)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        out = torch.full((c2.rows.n * P.contact_dtype.itemsize,), 0xAB, dtype=torch.uint8, device="cuda")
        c2.rows.device(c2.eng, "collide", req, out=out, stream=side)
    side.synchronize()
    got = records(out, "collide")
    no_watchdog_trip(c2.eng)
    ro = c2.rows.host(c2.orc, "collide", req, nthreads=0)
    compare_distance(ro, got, what="config 2 device collide, margin %g" % margin)
    if margin == -np.inf:
        assert got["num_contacts"].sum() == 0 and np.all(np.isnan(got["p1"]))
    else:
        assert got["num_contacts"].sum() > 100_000
    host = c2.rows.host(c2.eng, "collide", req)
    assert host.tobytes() == got.tobytes(), "device form and host form differ"
    no_watchdog_trip(c2.eng)
    ref_sample(c2.ref, "batch_collide", ro, sample_rows(c2.rows.n, 100_000, 7), c2.rows.h + (req,),
               "config 2 collide margin %g" % margin)
    print("margin %g: %d rows against the oracle (all), the host form (all); %.1f s"
          % (margin, c2.rows.n, time.perf_counter() - t0))


def test_config2_bench_rows():
    """bench.py's config 2 rows (make_workload): 1 M object pairs of a 100 k-object scene"""
    t0 = time.perf_counter()
    s = W.config2_scene(100_000, 1_000_000, seed=0xFC1 + 2)
    h1, h2 = s["obj_h"][s["first"]], s["obj_h"][s["second"]]
    tf1, tf2 = np.ascontiguousarray(s["obj_tf"][s["first"]]), np.ascontiguousarray(s["obj_tf"][s["second"]])
    eng = hf.Engine(0)
    orc = oracle_lib.OracleScene(P)
    hs = eng.register_shapes(s["shapes"])
    assert np.array_equal(hs, orc.register_shapes(s["shapes"]))
    eng.commit()
    rows = Rows(hs[h1 % len(hs)], tf1, hs[h2 % len(hs)], tf2)
    req = P.DistanceRequestPOD()
    got = records(rows.device(eng, "distance", req), "distance")
    no_watchdog_trip(eng)
    ro = rows.host(orc, "distance", req, nthreads=0)
    compare_distance(ro, got, what="bench config 2 rows")
    assert rows.host(eng, "distance", req).tobytes() == got.tobytes()
    ref = reference_scene()
    if ref is not None:
        ref.register_shapes(s["shapes"])
        ref_sample(ref, "batch_distance", ro, sample_rows(rows.n, 100_000, 3), rows.h + (req,), "bench config 2 rows")
    print("bench config 2: %d rows %s against the oracle (all), the host form (all); %.1f s"
          % (rows.n, path_counts(ro["status"]), time.perf_counter() - t0))


# ---------------------------------------------------------------------------------------------------------------------
# config 3: 1 M Convex64 pairs, all in the hull / triangle class.  The oracle registers the hulls without faces, so it
# runs the linear-scan support the kernels implement and is bit-identical (DESIGN.md section 4).
C3_REQUESTS = (("distance", P.DistanceRequestPOD(gjk_variant=P.DefaultGJK)),
               ("distance", P.DistanceRequestPOD(gjk_variant=P.NesterovAcceleration)),
               ("collide", P.CollisionRequestPOD(security_margin=0.01)))


@pytest.fixture(scope="module")
def c3():
    t0 = time.perf_counter()
    w = W.config3_convex_pairs(1_000_000)
    orc = oracle_lib.OracleScene(P)
    cids = [orc.register_convex(pts, None) for pts, _ in w["hulls"]]
    hc = orc.register_shapes(P.make_shapes([P.GEOM_CONVEX] * len(cids), np.zeros((len(cids), 3)), data=cids))
    h1, h2 = hc[w["h1"]], hc[w["h2"]]
    ro = []
    for kind, req in C3_REQUESTS:
        t1 = time.perf_counter()
        ro.append(getattr(orc, "batch_" + kind)(h1, w["tf1"], h2, w["tf2"], req, nthreads=0))
        print("config 3 oracle, %s: %.1f s for %d rows" % (kind, time.perf_counter() - t1, len(h1)))
    print("config 3 set up in %.1f s" % (time.perf_counter() - t0))
    return types.SimpleNamespace(w=w, cids=cids, hc=hc, ro=ro)


@pytest.mark.parametrize("gc", [None, "8"])
def test_config3_hull_class_past_its_cap(c3, gc, monkeypatch):
    """default lane width (2 lanes per pair) and HFB_GC=8 (16 pairs per block: the cap is 4x smaller, and the host form's
    chunks cross it too)"""
    t0 = time.perf_counter()
    if gc is not None:
        monkeypatch.setenv("HFB_GC", gc)
    eng = hf.Engine(0)
    cids = [eng.register_convex(pts) for pts, _ in c3.w["hulls"]]
    assert cids == c3.cids
    hc = eng.register_shapes(P.make_shapes([P.GEOM_CONVEX] * len(cids), np.zeros((len(cids), 3)), data=cids))
    assert np.array_equal(hc, c3.hc)
    eng.commit()
    rows = Rows(hc[c3.w["h1"]], c3.w["tf1"], hc[c3.w["h2"]], c3.w["tf2"])
    counts = path_counts(c3.ro[0]["status"])
    assert counts["gjk"] == rows.n
    assert_past_cap("config 3, hull class, HFB_GC=%s" % (gc or "2 (default)"), counts["gjk"],
                    grid_caps(int(gc or 2))["hull"])
    for (kind, req), ro in zip(C3_REQUESTS, c3.ro):
        got = records(rows.device(eng, kind, req), kind)
        no_watchdog_trip(eng)
        compare_distance(ro, got, what="config 3 device %s, HFB_GC=%s" % (kind, gc))
        assert rows.host(eng, kind, req).tobytes() == got.tobytes(), "device form and host form differ"
        no_watchdog_trip(eng)
    assert (P.status_epa(c3.ro[0]["status"]) != P.EPA_DidNotRun).sum() > 200_000
    print("config 3, HFB_GC=%s: %d rows x %d requests against the oracle (all), the host form (all); %.1f s"
          % (gc, rows.n, len(C3_REQUESTS), time.perf_counter() - t0))


# ---------------------------------------------------------------------------------------------------------------------
def test_config4_bvh_walk_at_full_size():
    """bench.py's config 4: 100 k capsule queries against the 10 k-triangle OBBRSS mesh, through k_bvhq's task walk"""
    from tests.common import MultiScene
    t0 = time.perf_counter()
    c = W.config4_mesh_vs_capsules(100_000)
    eng = hf.Engine(0)
    backends = {"oracle": oracle_lib.OracleScene(P), "gpu": eng}
    ref = reference_scene()
    if ref is not None:
        backends["ref"] = ref
    sc = MultiScene(backends)
    bid, _ = sc.register_bvh(c["verts"], c["tris"])
    hm = sc.register_shapes(P.make_shapes([P.BV_OBBRSS], [[0, 0, 0]], data=[bid]))
    hcap = sc.register_shapes(c["capsules"])
    sc.commit()
    rows = Rows(np.full(len(c["hc"]), hm[0], dtype=np.uint32), c["tf_mesh"], hcap[c["hc"]], c["tf_caps"])
    req = P.DistanceRequestPOD()
    got = records(rows.device(eng, "distance", req), "distance")
    no_watchdog_trip(eng)
    ro = rows.host(backends["oracle"], "distance", req, nthreads=0)
    assert path_counts(ro["status"])["bvh"] == rows.n
    compare_distance(ro, got, what="config 4 device distance")
    assert (ro["min_distance"] < 0).sum() > 1000 and (ro["min_distance"] > 0).sum() > 1000
    ref_sample(ref, "batch_distance", ro, sample_rows(rows.n, 20_000, 4), rows.h + (req,), "config 4",
               fields=("min_distance", "p1", "p2", "normal", "b1", "b2"))
    print("config 4: %d mesh-capsule rows against the oracle (all); %.1f s" % (rows.n, time.perf_counter() - t0))


# ---------------------------------------------------------------------------------------------------------------------
def test_config5_broadphase_and_narrow_phase_at_full_size():
    """bench.py's config 5 step: device boxes -> device pair finder -> batch_collide_objects_device, on 100 k boxes, and
    the pair finder cut into two halves of the objects as bench shards it"""
    import torch
    t0 = time.perf_counter()
    n = 100_000
    w = W.config5_moving_boxes(n, seed=0xFC1 + 5)
    eng = hf.Engine(0)
    orc = oracle_lib.OracleScene(P)
    hb = eng.register_shapes(w["shapes"])
    assert np.array_equal(hb, orc.register_shapes(w["shapes"]))
    eng.commit()
    oh = hb[w["obj_h"]].astype(np.uint32)
    tf = w["step"](0)
    stream = torch.cuda.current_stream().cuda_stream
    d_h, d_tf = dev(oh), dev(tf)
    d_bb = torch.empty(n * 6, dtype=torch.float64, device="cuda")
    cap = int(2.0 * 1_000_000 * (n / 100_000.0)) + 65536  # bench.py's capacity at one GPU
    d_f = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_s = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int32, device="cuda")
    eng.scene_aabbs_device(n, d_h.data_ptr(), d_tf.data_ptr(), d_bb.data_ptr(), stream)
    torch.cuda.synchronize()
    bb = eng.scene_aabbs(oh, tf)
    assert d_bb.cpu().numpy().tobytes() == bb.tobytes(), "device boxes differ from the host ones"

    def device_pairs(lo, cnt):
        eng.broadphase_pairs_device(n, d_bb.data_ptr(), d_f.data_ptr(), d_s.data_ptr(), cap, d_n.data_ptr(), stream,
                                    first_object=lo, num_first_objects=cnt)
        torch.cuda.synchronize()
        k = int(d_n.item())
        assert k <= cap
        return k, d_f[:k].cpu().numpy().view(np.uint32), d_s[:k].cpu().numpy().view(np.uint32)

    def key(f, s):
        return np.sort(f.astype(np.int64) * n + s.astype(np.int64))

    k, f, s = device_pairs(0, n)
    hf_, hs_ = hf.broadphase_pairs(bb)
    assert np.array_equal(key(f, s), key(hf_, hs_)), "device pair set differs from the host pair finder's"
    d_out = torch.empty(max(k, 1) * P.contact_dtype.itemsize, dtype=torch.uint8, device="cuda")
    req = P.CollisionRequestPOD()
    eng.batch_collide_objects_device(n, d_h.data_ptr(), d_tf.data_ptr(), k, d_f.data_ptr(), d_s.data_ptr(),
                                     d_out.data_ptr(), req, stream=stream)
    got = records(d_out, "collide", k)
    no_watchdog_trip(eng)
    ro = orc.batch_collide(oh[f], tf[f], oh[s], tf[s], req, nthreads=0)
    compare_distance(ro, got, what="config 5 narrow phase")
    hits = int((ro["num_contacts"] > 0).sum())
    assert hits > 10_000
    ref = reference_scene()
    if ref is not None:
        ref.register_shapes(w["shapes"])
        ref_sample(ref, "batch_collide", ro, sample_rows(k, 100_000, 5), (oh[f], tf[f], oh[s], tf[s], req),
                   "config 5 narrow phase")
    # bench's sharding: two ranges of first objects; disjoint pair sets whose union is the whole
    half = n // 2
    ka, fa, sa = device_pairs(0, half)
    kb, fb, sb = device_pairs(half, n - half)
    assert np.all(fa < half) and np.all(fb >= half) and ka + kb == k
    both = np.concatenate([key(fa, sa), key(fb, sb)])
    assert len(np.unique(both)) == k and np.array_equal(np.sort(both), key(f, s))
    print("config 5: %d boxes, %d candidate pairs %s (%d colliding) against the oracle (all); halves %d + %d; %.1f s"
          % (n, k, path_counts(ro["status"]), hits, ka, kb, time.perf_counter() - t0))


# ---------------------------------------------------------------------------------------------------------------------
# the device form's own contract, on config 2's batch (past every primitive cap)
def test_device_form_repeated_calls_and_a_fresh_context(c2):
    import torch
    req = P.DistanceRequestPOD()
    out = c2.rows.device(c2.eng, "distance", req)
    first = records(out, "distance").tobytes()
    for _ in range(2):
        c2.rows.device(c2.eng, "distance", req, out=out)
        assert records(out, "distance").tobytes() == first, "a repeated call into the same output differs"
    no_watchdog_trip(c2.eng)
    small = c2.rows.n // 10
    c2.rows.device(c2.eng, "distance", req, out=out, n=small)
    assert records(out, "distance", small).tobytes() == c2.ro_default[:small].tobytes()
    c2.rows.device(c2.eng, "distance", req, out=out)
    again = records(out, "distance").tobytes()
    fresh = hf.Engine(0)
    assert np.array_equal(fresh.register_shapes(c2.shapes), c2.hs)
    fresh.commit()
    assert again == records(c2.rows.device(fresh, "distance", req), "distance").tobytes()
    assert again == c2.ro_default.tobytes()
    no_watchdog_trip(c2.eng)
    no_watchdog_trip(fresh)
    del fresh
    torch.cuda.synchronize()


def test_device_form_on_alternating_streams_and_a_host_call_after_it(c2):
    """different inputs on two streams, alternating, no host sync in between: each result is its call's alone"""
    import torch
    req = P.DistanceRequestPOD()
    perm = np.random.default_rng(17).permutation(c2.rows.n)
    b = Rows(c2.rows.h[0][perm], c2.rows.h[1][perm], c2.rows.h[2][perm[::-1]], c2.rows.h[3][perm[::-1]])
    want_a = c2.ro_default.tobytes()
    want_b = records(b.device(c2.eng, "distance", req), "distance").tobytes()
    assert want_b != want_a
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = [torch.empty(c2.rows.n * P.distance_result_dtype.itemsize, dtype=torch.uint8, device="cuda") for _ in range(4)]
    torch.cuda.synchronize()
    c2.rows.device(c2.eng, "distance", req, out=outs[0], stream=s1)
    b.device(c2.eng, "distance", req, out=outs[1], stream=s2)
    c2.rows.device(c2.eng, "distance", req, out=outs[2], stream=s1)
    b.device(c2.eng, "distance", req, out=outs[3], stream=s2)
    torch.cuda.synchronize()
    for k, o in enumerate(outs):
        assert records(o, "distance").tobytes() == (want_a if k % 2 == 0 else want_b), "call %d on alternating streams" % k
    # a host-form call right after a device call, without a sync
    out = torch.empty_like(outs[0])
    c2.rows.device(c2.eng, "distance", req, out=out, stream=s1)
    host = b.host(c2.eng, "distance", req)
    assert host.tobytes() == want_b
    assert records(out, "distance").tobytes() == want_a
    no_watchdog_trip(c2.eng)


def test_device_form_warm_starts_in_device_memory(c2):
    import torch
    n = c2.rows.n
    req = P.DistanceRequestPOD()
    d_g = torch.full((n * 3,), np.nan, dtype=torch.float64, device="cuda")
    d_hint = torch.full((n * 2,), -7, dtype=torch.int32, device="cuda")
    got = records(c2.rows.device(c2.eng, "distance", req, guess=P.GuessOut(d_g.data_ptr(), d_hint.data_ptr())), "distance")
    host, gg, gh = c2.rows.host(c2.eng, "distance", req, want_guess=True)
    assert got.tobytes() == host.tobytes()
    assert d_g.cpu().numpy().tobytes() == gg.tobytes() and d_hint.cpu().numpy().tobytes() == gh.tobytes()
    no_watchdog_trip(c2.eng)
    # cached guesses read from device memory: a guess moved off the converged one, and the hints
    gg2 = gg.reshape(-1, 3) * 0.5 + np.array([0.25, -0.125, 0.5])
    wreq = P.DistanceRequestPOD(gjk_initial_guess=P.CachedGuess)
    d_g2, d_h2 = dev(gg2).view(torch.float64), dev(gh).view(torch.int32)
    wreq.q.cached_gjk_guess, wreq.q.cached_support_func_guess = d_g2.data_ptr(), d_h2.data_ptr()
    got2 = records(c2.rows.device(c2.eng, "distance", wreq), "distance")
    hreq = P.DistanceRequestPOD(gjk_initial_guess=P.CachedGuess)
    hreq.q.cached_gjk_guess, hreq.q.cached_support_func_guess = gg2.ctypes.data, gh.ctypes.data
    assert c2.rows.host(c2.eng, "distance", hreq).tobytes() == got2.tobytes()
    ro2 = c2.rows.host(c2.orc, "distance", hreq, nthreads=0)
    compare_distance(ro2, got2, what="device warm start")
    assert not np.array_equal(ro2["iterations"], c2.ro_default["iterations"])  # the guesses were used
    no_watchdog_trip(c2.eng)


def test_device_form_profiling_refusals_and_empty_batches(c2):
    import torch
    req = P.DistanceRequestPOD()
    c2.eng.set_profiling(True)
    try:
        c2.eng.kernel_times(reset=True)
        got = records(c2.rows.device(c2.eng, "distance", req), "distance")
        kt = c2.eng.kernel_times(reset=True)
    finally:
        c2.eng.set_profiling(False)
    assert got.tobytes() == c2.ro_default.tobytes()
    times = [v for k, v in kt.items() if k.endswith("_ms")]
    assert all(np.isfinite(t) and t >= 0 for t in times) and kt["pairs_launches"] > 0 and kt["closed_launches"] > 0
    r = c2.rows
    for fn, rq in ((c2.eng.batch_distance_device, req), (c2.eng.batch_collide_device, P.CollisionRequestPOD())):
        with pytest.raises(hf.EngineError):
            fn(r.n, r.d[0].data_ptr(), r.d[1].data_ptr(), r.d[2].data_ptr(), r.d[3].data_ptr(), 0, rq)
        out = torch.full((4096,), 0x5A, dtype=torch.uint8, device="cuda")
        fn(0, r.d[0].data_ptr(), r.d[1].data_ptr(), r.d[2].data_ptr(), r.d[3].data_ptr(), out.data_ptr(), rq)
        torch.cuda.synchronize()
        assert bool((out == 0x5A).all()), "an empty batch wrote to its output"
    no_watchdog_trip(c2.eng)


# ---------------------------------------------------------------------------------------------------------------------
def test_convex_support_at_the_roofline_size():
    """bench.py's support roofline: 786 432 hulls of 64 vertices registered in one batch (after a few registered one by
    one, so its first id is not 0), 2 M queries through batch_convex_support_device; then the edge hulls of
    tests/test_convex_support_ref.py through the same call"""
    import torch
    t0 = time.perf_counter()
    eng = hf.Engine(0)
    rng = np.random.default_rng(5)
    lead = [W.ellipsoid_hull(rng, nv)[0] for nv in (7, 32, 40)]
    assert [eng.register_convex(p) for p in lead] == [0, 1, 2]
    n_hulls, nv, n_q = 786432, 64, 1 << 21
    r99 = np.random.default_rng(99)  # bench.py support_kernel_roofline's hulls and queries
    v = r99.normal(size=(n_hulls, nv, 3))
    v /= np.linalg.norm(v, axis=2, keepdims=True)
    v *= 0.05 + 0.95 * r99.random((n_hulls, 1, 3))
    ids = r99.permutation(n_q).astype(np.uint32) % n_hulls
    dirs = r99.normal(size=(n_q, 3))
    dirs[:4096] = np.eye(3)[rng.integers(0, 3, 4096)] * rng.choice([-1.0, 1.0], (4096, 1))  # axis-aligned
    first = eng.register_convex_batch(v)
    assert first == len(lead)
    hulls, e_ids, e_dirs, _ = edge_hulls()
    e_first = first + n_hulls
    assert [eng.register_convex(h) for h in hulls] == list(range(e_first, e_first + len(hulls)))
    eng.commit()

    def run(q_ids, q_dirs):
        n = len(q_ids)
        d_ids, d_dirs = dev(q_ids).view(torch.int32), dev(q_dirs).view(torch.float64)
        d_idx = torch.full((n,), -3, dtype=torch.int32, device="cuda")
        d_sup = torch.empty((n, 3), dtype=torch.float64, device="cuda")
        eng.batch_convex_support_device(n, d_ids.data_ptr(), d_dirs.data_ptr(), d_idx.data_ptr(), d_sup.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return d_idx.cpu().numpy(), d_sup.cpu().numpy()

    gi, gs = run(ids + first, dirs)
    chunk = 1 << 16
    for lo in range(0, n_q, chunk):
        s = slice(lo, lo + chunk)
        wi, ws = support_ref(v, np.full(n_hulls, nv), ids[s], dirs[s])
        bad = np.nonzero(gi[s] != wi)[0]
        assert not len(bad), "support index differs at queries %s" % (lo + bad[:10])
        assert gs[s].tobytes() == ws.tobytes(), "support points differ in chunk at %d" % lo
    # the edge hulls, and queries on the leading hulls mixed in
    l_ids = np.arange(len(e_ids)) % len(lead)
    gi, gs = run(np.concatenate([e_ids + e_first, l_ids]).astype(np.uint32), np.concatenate([e_dirs, e_dirs]))
    m = len(e_ids)
    for (wi, ws), part in ((support_ref(*pad_hulls(hulls), e_ids, e_dirs), slice(0, m)),
                           (support_ref(*pad_hulls(lead), l_ids, e_dirs), slice(m, 2 * m))):
        bad = np.nonzero(gi[part] != wi)[0]
        assert not len(bad), "edge queries: support index differs at %s" % bad[:10]
        assert gs[part].tobytes() == ws.tobytes()
    no_watchdog_trip(eng)
    print("convex support: %d queries on %d hulls (first id %d) and %d edge queries against support_ref (all); %.1f s"
          % (n_q, n_hulls, first, 2 * len(e_ids), time.perf_counter() - t0))
