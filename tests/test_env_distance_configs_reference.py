"""The configurations distance query's winners against the reference build (no GPU needed).  Each configuration's winner
-- over its environment pairs and its template's self pairs -- is found by brute force with the oracle under the
contract of hfb_env_distance_configs (include/hppfcl_b200.h), on the robot workload with joints bending far enough that
some configurations penetrate themselves, and on a scene of exact ties between kinds and between template entries.  The
reference build's distance() on every winning pair must give the oracle's record bit for bit;
tests/test_gpu_env_distance_configs.py then checks that the device finds the same winners with the same records."""
import gzip
import json
import os

import numpy as np

from tests import common
from tests.common import P, compare_distance, make_scenes
from tests.test_env_distance_reference import assert_fields
from oracle import oracle_lib
from hppfcl_b200 import workloads as W

# the reference's recorded outputs for the sample's call (HFB_RECORD_REFERENCE=<this file> records them), looked up
# with those of tests/golden/reference_outputs.json.gz where oracle/_ref is not built
REF_OUTPUTS = os.path.join(common.ROOT, "tests", "golden", "reference_outputs_distance_configs.json.gz")
CUTOFFS = (0.0, 0.05, np.inf)
LINKS = 16


def load_recorded():
    if os.path.exists(REF_OUTPUTS):
        common._load_recorded().update(json.load(gzip.open(REF_OUTPUTS, "rt")))


def oracle_winners(orc, ha, tfa, hb, tfb, links, tpl, maxd):
    """-> (kind, first, second, records) per configuration: the oracle's distance() on every environment pair and every
    template pair, then the header's argmin (smallest distance, then environment pairs by link and B index, then self
    pairs in template order)"""
    na, nb = len(ha), len(hb)
    tpl = np.asarray(tpl, dtype=np.int64).reshape(-1, 2)
    n_configs = na // links
    i, j = np.repeat(np.arange(na), nb), np.tile(np.arange(nb), na)
    erec = orc.batch_distance(ha[i], tfa[i], hb[j], tfb[j], nthreads=0).reshape(na, nb) if nb else None
    g = np.repeat(np.arange(n_configs), len(tpl))
    sa, sb = g * links + np.tile(tpl[:, 0], n_configs), g * links + np.tile(tpl[:, 1], n_configs)
    srec = orc.batch_distance(ha[sa], tfa[sa], ha[sb], tfa[sb], nthreads=0) if len(sa) else None
    kind = np.full(n_configs, -1, dtype=np.int8)
    first = np.full(n_configs, 0xFFFFFFFF, dtype=np.uint32)
    second = first.copy()
    recs = np.zeros(n_configs, dtype=P.distance_result_dtype)
    elig = lambda r: (r["min_distance"] <= maxd) & (P.status_path(r["status"]) != P.PATH_UNSUPPORTED)  # noqa: E731
    for c in range(n_configs):
        best = None  # (distance, ordinal, B index or 0, kind, first, second, record)
        for li in range(links):
            a = c * links + li
            if erec is None:
                break
            for b in np.flatnonzero(elig(erec[a])):
                cand = (erec[a, b]["min_distance"], li, int(b), 0, a, int(b), erec[a, b])
                if best is None or cand[:3] < best[:3]:
                    best = cand
        if srec is not None:
            for k in range(len(tpl)):
                p = c * len(tpl) + k
                if elig(srec[p:p + 1])[0]:
                    cand = (srec[p]["min_distance"], links + k, 0, 1, int(sa[p]), int(sb[p]), srec[p])
                    if best is None or cand[:3] < best[:3]:
                        best = cand
        if best is not None:
            kind[c], first[c], second[c], recs[c] = best[3:]
    return kind, first, second, recs


def tie_geometry(sc):
    """one configuration of three spheres, links 1 and 2 both 0.5 from link 0, and an environment sphere 0.5 from link 0
    (B near) or far from every link (B far)"""
    sph = int(sc.register_shapes(P.make_shapes([P.GEOM_SPHERE], [[0.25, 0, 0]]))[0])
    ha = np.full(3, sph, dtype=np.uint32)
    tfa = W.identity_transforms(3, T=[[0, 0, 0], [1.0, 0, 0], [-1.0, 0, 0]])
    hb = np.full(1, sph, dtype=np.uint32)
    return ha, tfa, hb, W.identity_transforms(1, T=[[0, 1.0, 0]]), W.identity_transforms(1, T=[[0, 10.0, 0]])


def reference_sample(sc):
    """registers the scenes in every backend of sc (which holds the oracle) -> (scenes: [(ha, tfa, hb, tfb, links, tpl,
    {cutoff: (kind, first, second)})], the winning pairs as (h1, tf1, h2, tf2), the oracle's records of them).  The same
    wherever this runs: the oracle is the reference's restatement on the CPU."""
    w = W.robot_vs_environment(n_configs=8, n_env=300, room=3.0, seed=53, joint_range=2.8)
    hs = w["register"](sc, oracle=True)
    # B without the floor (object 0), which every configuration's base touches
    robot = (hs[w["geom_a"]].astype(np.uint32), w["tf_a"], hs[w["geom_b"][1:]].astype(np.uint32), w["tf_b"][1:], LINKS,
             W.chain_self_pairs(LINKS))
    ha, tfa, hb, near, far = tie_geometry(sc)
    sc.commit()
    ties = [(ha, tfa, hb, near, 3, [(0, 1), (0, 2)]), (ha, tfa, hb, far, 3, [(0, 1), (0, 2)]),
            (ha, tfa, hb, far, 3, [(2, 0), (1, 0)])]
    orc = sc.b["oracle"]
    scenes, seen, recs = [], set(), []
    for s, (ha, tfa, hb, tfb, links, tpl) in enumerate([robot] + ties):
        win = {}
        for maxd in CUTOFFS:
            kind, first, second, rec = oracle_winners(orc, ha, tfa, hb, tfb, links, tpl, maxd)
            win[maxd] = (kind, first, second)
            for c in np.flatnonzero(kind >= 0):
                key = (s, int(kind[c]), int(first[c]), int(second[c]))
                if key not in seen:
                    seen.add(key)
                    other = (hb, tfb) if kind[c] == 0 else (ha, tfa)
                    recs.append((ha[first[c]], tfa[first[c]], other[0][second[c]], other[1][second[c]], rec[c]))
        scenes.append((ha, tfa, hb, tfb, links, tpl, win))
    h1 = np.array([r[0] for r in recs], dtype=np.uint32)
    tf1 = np.array([r[1] for r in recs], dtype=P.transform_dtype)
    h2 = np.array([r[2] for r in recs], dtype=np.uint32)
    tf2 = np.array([r[3] for r in recs], dtype=P.transform_dtype)
    return scenes, (h1, tf1, h2, tf2), np.array([r[4] for r in recs], dtype=P.distance_result_dtype)


def test_winners_reference_sample():
    """the reference build's distance() on every winning pair gives the oracle's record; the sample holds environment
    and self winners, penetrating self winners, configurations without a winner, and the tie rules"""
    oracle_lib.build_ref()
    load_recorded()
    sc = make_scenes(ref=True, emu=False)
    scenes, args, orec = reference_sample(sc)
    rr = sc.b["ref"].batch_distance(*args)
    assert_fields(rr, orec, "winning pairs against the reference build")
    rows = P.status_path(orec["status"]) != P.PATH_BVH
    compare_distance(rr[rows], orec[rows], what="winning shape pairs against the reference build")
    robot = scenes[0][6]
    assert (robot[np.inf][0] >= 0).all() and (robot[0.0][0] == -1).any()
    assert (robot[0.0][0] == 1).any()  # a configuration that penetrates itself: a self pair wins at distance <= 0
    assert (robot[0.05][0] == 0).any() and len(orec) > 8
    # ties at 0.5: the environment pair beats the self pair; between two self pairs the earlier template entry wins
    assert [tuple(int(x[0]) for x in t[6][np.inf]) for t in scenes[1:]] == [(0, 0, 0), (1, 0, 1), (1, 2, 0)]
