"""Iteration caps and budgets at the launch boundaries of the device code, on the host: the requests that
tests/test_gpu_edge_inputs.py sends to the kernels, here through the oracle, the host build of the device code and the
reference build, bit for bit (so that on the GPU the oracle stands for the reference on exactly these inputs).

The primitive-pair GJK passes end after 10 iterations (k_gjk_first) and run the rest to convergence (k_gjk_more), or
after 3, 3 and 4 with HFB_GJK_PASSES=3,3,4; EPA's tier 0 holds 24 iterations (HFB_EPA_SMALL_IT), the full-size tier 64;
a leaf item of the mesh-shape task system runs 6 GJK iterations before it parks its state (HFB_BVH_GJK_CHUNK).  A cap
that ends exactly at one of these boundaries must give the record of the reference: status Failed from the kernel that
ran the last iteration, the iteration count carried across the launches.
"""
import gzip
import json
import os

import numpy as np

from oracle import oracle_lib
from tests import common
from tests.common import P, compare_distance, make_scenes, ref_agrees
from tests.tools import fuzz_ref
from hppfcl_b200 import workloads as W

ALL_PRIMS = (P.GEOM_SPHERE, P.GEOM_CAPSULE, P.GEOM_BOX, P.GEOM_CYLINDER, P.GEOM_CONE, P.GEOM_ELLIPSOID)
GJK_CAPS = (0, 1, 9, 10, 11, 20, 128)         # around the first pass of the default schedule
GJK_CAPS_3_3_4 = (2, 3, 4, 6, 7, 10, 11)      # around the passes of HFB_GJK_PASSES=3,3,4
GJK_TOL = 1e-12  # (more pairs reach the later passes, and Nesterov's runs reach 128 iterations)
EPA_CAPS = (0, 1, 23, 24, 25, 64)             # around tier 0's 24 iterations
EPA_TOL = 1e-12
EPA_SMALL_IT = 24
BVH_CAPS = (5, 6, 7, 12, 13)                  # around the leaf item's 6 iterations
VARIANTS = (P.DefaultGJK, P.PolyakAcceleration, P.NesterovAcceleration)

# the reference's recorded outputs for this module's calls (HFB_RECORD_REFERENCE=<this file> records them), looked up
# with those of tests/golden/reference_outputs.json.gz where oracle/_ref is not built
REF_OUTPUTS = os.path.join(common.ROOT, "tests", "golden", "reference_outputs_boundaries.json.gz")


def boundary_batch(sc):
    """BASELINE config 2's mixed primitive pairs (every primitive type, many of them penetrating), 1 000 pairs of a
    32-vertex hull against primitives and 1 000 (mesh, primitive) pairs -> (h1, t1, h2, t2, n_shape_pairs); the mesh
    pairs come last"""
    w = W.config2_mixed_primitives(20000, pool=4096, types=ALL_PRIMS)
    hp = sc.register_shapes(w["shapes"])
    rng = np.random.default_rng(31)
    pts, tris = W.ellipsoid_hull(rng, 32, radii=(0.5, 0.7, 0.9))
    cid = sc.register_convex(pts, tris)
    hc = sc.register_shapes(P.make_shapes([P.GEOM_CONVEX], [[0, 0, 0]], data=[cid]))
    v, f = W.sphere_mesh(1.0, 12, 6, noise=0.05, rng=rng)
    bid, _ = sc.register_bvh(v, f)
    hm = sc.register_shapes(P.make_shapes([P.BV_OBBRSS], [[0, 0, 0]], data=[bid]))
    sc.commit()
    k = 1000
    h1 = np.concatenate([hp[w["h1"]], np.full(k, hc[0]), np.full(k, hm[0])]).astype(np.uint32)
    h2 = np.concatenate([hp[w["h2"]], hp[rng.integers(0, len(hp), 2 * k)]]).astype(np.uint32)
    t1 = np.concatenate([w["tf1"], W.random_transforms(rng, 2 * k, (-1, -1, -1), (1, 1, 1))])
    t2 = np.concatenate([w["tf2"], W.random_transforms(rng, 2 * k, (-1, -1, -1), (1, 1, 1))])
    return h1, t1, h2, t2, len(w["h1"]) + k


def gjk_cap_request(fn, cap, variant):
    R = P.DistanceRequestPOD if fn == "batch_distance" else P.CollisionRequestPOD
    return R(gjk_max_iterations=cap, gjk_variant=variant, gjk_tolerance=GJK_TOL)


def epa_cap_request(fn, cap):
    R = P.DistanceRequestPOD if fn == "batch_distance" else P.CollisionRequestPOD
    return R(epa_max_iterations=cap, epa_tolerance=EPA_TOL)


def failed_at(rec, cap):
    """pairs that stopped with status Failed after exactly `cap` iterations (cap 0 runs one: the test comes after it)"""
    return int((((rec["status"] & 0xff) == P.GJK_Failed) & ((rec["iterations"] & 0xffff) == max(cap, 1))).sum())


def test_iteration_caps_at_the_launch_boundaries():
    """oracle, host build of the device code and reference build agree on every record (mesh pairs: on the fields the
    reference defines); every GJK cap is reached by some pair, and EPA runs outgrow tier 0 under the caps above it"""
    oracle_lib.build_ref()
    if os.path.exists(REF_OUTPUTS):
        common._load_recorded().update(json.load(gzip.open(REF_OUTPUTS, "rt")))
    sc = make_scenes(ref=True)
    h1, t1, h2, t2, ns = boundary_batch(sc)
    shape = (h1[:ns], t1[:ns], h2[:ns], t2[:ns])
    mesh = (h1[ns:], t1[ns:], h2[ns:], t2[ns:])
    for fn in ("batch_distance", "batch_collide"):
        for cap in sorted(set(GJK_CAPS + GJK_CAPS_3_3_4)):
            hit = 0
            for v in VARIANTS:
                req = gjk_cap_request(fn, cap, v)
                what = "%s cap %d variant %d" % (fn, cap, v)
                ro = getattr(sc.b["oracle"], fn)(h1, t1, h2, t2, req, nthreads=0)
                compare_distance(ro, getattr(sc.b["emu"], fn)(h1, t1, h2, t2, req), what=what)
                ref_agrees(sc, fn, ro[:ns], shape + (req,), what)
                hit += failed_at(ro[:ns], cap)
            assert hit > 0, "%s: no pair reaches the cap of %d" % (fn, cap)
        for cap in EPA_CAPS:
            req = epa_cap_request(fn, cap)
            what = "%s EPA cap %d" % (fn, cap)
            ro = getattr(sc.b["oracle"], fn)(h1, t1, h2, t2, req, nthreads=0)
            compare_distance(ro, getattr(sc.b["emu"], fn)(h1, t1, h2, t2, req), what=what)
            ref_agrees(sc, fn, ro[:ns], shape + (req,), what)
            if cap > EPA_SMALL_IT:  # runs that reached iteration 24 had outgrown tier 0's workspace
                assert ((ro["iterations"][:ns] >> 16) >= EPA_SMALL_IT).sum() > 10
        for cap in BVH_CAPS:
            req = gjk_cap_request(fn, cap, P.DefaultGJK)
            what = "%s mesh pairs, cap %d" % (fn, cap)
            ro = getattr(sc.b["oracle"], fn)(*mesh, req, nthreads=0)
            compare_distance(ro, getattr(sc.b["emu"], fn)(*mesh, req), what=what)
            ref_agrees(sc, fn, ro, mesh + (req,), what, fields=fuzz_ref.D_MESH if fn == "batch_distance" else fuzz_ref.C_MESH)
