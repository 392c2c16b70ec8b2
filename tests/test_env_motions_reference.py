"""The motions query's answers against the reference build (no GPU needed).  Each motion's first colliding sample and
its witness are found by brute force under the contract of hfb_env_collide_motions (include/hppfcl_b200.h): boxes from
the host build of the device code, the environment and self candidates from the library's host pair finders, the
oracle's collide() on every candidate, then the first colliding sample and its first colliding pair in the contract's
order (environment pairs by link, then by B index; then self pairs in template order).  The sample holds the robot
workload's motions and a scene of spheres built so that every tie rule decides a witness.  The reference build's
collide() on every witness gives the oracle's record bit for bit; tests/test_gpu_env_motions.py then checks that the
device gives the same answers with the same records."""
import gzip
import json
import os

import numpy as np

from tests import common
from tests.common import P, compare_distance, hf, make_scenes
from oracle import oracle_lib
from hppfcl_b200 import workloads as W

# the reference's recorded outputs for the sample's call (HFB_RECORD_REFERENCE=<this file> records them), looked up
# with those of tests/golden/reference_outputs.json.gz where oracle/_ref is not built
REF_OUTPUTS = os.path.join(common.ROOT, "tests", "golden", "reference_outputs_motions.json.gz")
NONE = 0xFFFFFFFF
MESH_FIELDS = ("distance", "p1", "p2", "normal", "pos", "distance_lower_bound", "b1", "b2", "status", "num_contacts")


def load_recorded():
    if os.path.exists(REF_OUTPUTS):
        common._load_recorded().update(json.load(gzip.open(REF_OUTPUTS, "rt")))


def cleared_contact():
    """CollisionResult::clear()'s record (collision_data.h:483-489), as a motion without a witness gets it"""
    r = np.zeros(1, dtype=P.contact_dtype)
    for f in ("distance", "p1", "p2", "normal", "pos"):
        r[f] = np.nan
    r["distance_lower_bound"] = np.finfo(np.float64).max
    r["b1"] = r["b2"] = -1
    return r[0]


def contract(orc, emu, ha, tfa, hb, tfb, links, tpl, off):
    """the motions query by brute force -> (first_invalid, kind, first, second, records, counts = (env candidates, env
    colliding, self candidates, self colliding))"""
    tpl = np.asarray(tpl, dtype=np.uint32).reshape(-1, 2)
    n, n_b = len(off) - 1, len(hb)
    bb_a = emu.scene_aabbs(ha, tfa)
    ef, es = hf.broadphase_cross_pairs(bb_a, emu.scene_aabbs(hb, tfb)) if n_b else (np.zeros(0, np.uint32),) * 2
    sf, ss = hf.broadphase_config_pairs(bb_a, links, tpl)
    erec = orc.batch_collide(ha[ef], tfa[ef], hb[es], tfb[es], nthreads=0)
    srec = orc.batch_collide(ha[sf], tfa[sf], ha[ss], tfa[ss], nthreads=0)
    entry = {(int(i), int(j)): k for k, (i, j) in enumerate(tpl)}
    best = {}  # configuration -> (ordinal, kind, first, second, record)
    for kind, (f, s, rec) in enumerate(((ef, es, erec), (sf, ss, srec))):
        for p in np.flatnonzero(rec["num_contacts"] > 0):
            a, b = int(f[p]), int(s[p])
            o = (a % links) * n_b + b if kind == 0 else links * n_b + entry[(a % links, b % links)]
            g = a // links
            if g not in best or o < best[g][0]:
                best[g] = (o, kind, a, b, rec[p])
    fi = np.full(n, -1, dtype=np.int32)
    kd = np.full(n, -1, dtype=np.int8)
    first = np.full(n, NONE, dtype=np.uint32)
    second = np.full(n, NONE, dtype=np.uint32)
    recs = np.full(n, cleared_contact(), dtype=P.contact_dtype)
    for m in range(n):
        for g in range(int(off[m]), int(off[m + 1])):
            if g in best:
                _, kd[m], first[m], second[m], recs[m] = best[g]
                fi[m] = g - int(off[m])
                break
    counts = (len(ef), int((erec["num_contacts"] > 0).sum()), len(sf), int((srec["num_contacts"] > 0).sum()))
    return fi, kd, first, second, recs, counts


def tie_scene(sc):
    """configurations of three spheres (radius 0.25; links 1 and 2 one unit apart from link 0 along x unless placed
    otherwise), each at its own place, and environment spheres placed so that each tie rule decides a witness.  The
    template lists (0, 2) before (0, 1).  -> (ha, tfa, hb, tfb, links, tpl, offsets, what each motion shows)"""
    sph = int(sc.register_shapes(P.make_shapes([P.GEOM_SPHERE], [[0.25, 0, 0]]))[0])
    free = [(0, 0, 0), (1, 0, 0), (2, 0, 0)]
    folded = [(0, 0, 0), (0.1, 0, 0), (0.05, 0.05, 0)]  # every link on top of the others
    # (configuration links, environment spheres near them as (position, B index))
    kinds = {
        "F": (free, []),
        "S": (folded, []),
        "E1": (free, [((0, 0.3, 0), 2), ((0, -0.3, 0), 1)]),         # link 0 against B 2 and B 1: B 1 wins
        "E2": (free, [((1, 0.3, 0), 3), ((2, 0.3, 0), 0)]),          # link 1 (B 3) before link 2 (B 0)
        "ES": ([(0, 0, 0), (1, 0, 0), (0.1, 0, 0)], [((0, 0.3, 0), 4)]),  # env (link 0, B 4) before self (0, 2)
    }
    motions = [("valid", ["F", "F", "F"]), ("empty", []), ("at 0, one link, two B objects", ["E1", "F"]),
               ("in the middle, two links", ["F", "E2", "S", "F"]), ("at the last sample, env before self", ["F", "F", "ES"]),
               ("folded at the last sample", ["F", "S"]), ("empty", [])]
    T, bpos = [], {}
    g = 0
    for _, samples in motions:
        for k in samples:
            links, env = kinds[k]
            x0 = 10.0 * g
            T += [(x0 + x, y, z) for x, y, z in links]
            for (x, y, z), j in env:
                bpos[j] = (x0 + x, y, z)
            g += 1
    sizes = [len(s) for _, s in motions]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    ha = np.full(len(T), sph, dtype=np.uint32)
    hb = np.full(len(bpos), sph, dtype=np.uint32)
    tfb = W.identity_transforms(len(bpos), T=[bpos[j] for j in range(len(bpos))])
    return ha, W.identity_transforms(len(T), T=T), hb, tfb, 3, [(0, 2), (0, 1)], off, [m for m, _ in motions]


def reference_sample(sc):
    """registers the scenes in every backend of sc (which holds the oracle and the host build of the device code) ->
    (scenes: [(ha, tfa, hb, tfb, links, tpl, offsets, answer)], the witness pairs as (h1, tf1, h2, tf2), the oracle's
    records of them).  The same wherever this runs."""
    w = W.robot_motions(12, n_env=300, room=3.0, seed=67, joint_range=2.8)
    hs = w["register"](sc, oracle=True)
    # B without the floor (object 0), which every sample's base touches
    robot = (hs[w["geom_a"]].astype(np.uint32), w["tf_a"], hs[w["geom_b"][1:]].astype(np.uint32), w["tf_b"][1:], 16,
             W.chain_self_pairs(16), w["offsets"])
    ties = tie_scene(sc)[:7]
    sc.commit()
    orc, emu = sc.b["oracle"], sc.b["emu"]
    scenes, recs = [], []
    for ha, tfa, hb, tfb, links, tpl, off in (robot, ties):
        ans = contract(orc, emu, ha, tfa, hb, tfb, links, tpl, off)
        fi, kind, first, second, rec, _ = ans
        for m in np.flatnonzero(kind >= 0):
            other = (hb, tfb) if kind[m] == 0 else (ha, tfa)
            recs.append((ha[first[m]], tfa[first[m]], other[0][second[m]], other[1][second[m]], rec[m]))
        scenes.append((ha, tfa, hb, tfb, links, tpl, off, ans))
    h1 = np.array([r[0] for r in recs], dtype=np.uint32)
    tf1 = np.array([r[1] for r in recs], dtype=P.transform_dtype)
    h2 = np.array([r[2] for r in recs], dtype=np.uint32)
    tf2 = np.array([r[3] for r in recs], dtype=P.transform_dtype)
    return scenes, (h1, tf1, h2, tf2), np.array([r[4] for r in recs], dtype=P.contact_dtype)


def test_motions_reference_sample():
    """the reference build's collide() on every witness gives the oracle's record; the sample holds valid and empty
    motions, motions invalid at the first sample, in the middle and at the last, witnesses of both kinds and every tie
    rule"""
    oracle_lib.build_ref()
    load_recorded()
    sc = make_scenes(ref=True, emu=True)
    scenes, args, orec = reference_sample(sc)
    rr = sc.b["ref"].batch_collide(*args)
    assert np.array_equal(rr["num_contacts"], orec["num_contacts"]) and (orec["num_contacts"] > 0).all()
    mesh = P.status_path(orec["status"]) == P.PATH_BVH
    compare_distance(rr[~mesh], orec[~mesh], what="witness shape pairs against the reference build")
    # mesh witnesses: every field but `iterations`, which holds the oracle's own BV and leaf test counters there
    for f in MESH_FIELDS:
        x, y = rr[mesh][f], orec[mesh][f]
        assert np.all((x == y) | (np.isnan(x) & np.isnan(y)) if x.dtype.kind == "f" else x == y), f
    assert mesh.any() and (~mesh).sum() >= 6
    # the robot's motions: valid ones, invalid ones at the first sample, in the middle and at the last, both kinds
    fi, kind = scenes[0][7][:2]
    samples = np.diff(scenes[0][6]).astype(np.int64)
    assert (fi < 0).any() and (fi == 0).any() and ((fi > 0) & (fi < samples - 1)).any()
    assert (kind == 0).any() and (kind == 1).any()
    # the tie scene, motion by motion: (first_invalid, kind, first, second)
    fi, kind, first, second, rec, counts = scenes[1][7]
    off = scenes[1][6]
    g = lambda m, k: int(off[m]) + k  # noqa: E731  (configuration of sample k of motion m)
    want = [(-1, -1, NONE, NONE), (-1, -1, NONE, NONE),
            (0, 0, 3 * g(2, 0), 1),                       # link 0 against B 2 and B 1: the lower B index
            (1, 0, 3 * g(3, 1) + 1, 3),                   # link 1 (B 3) before link 2 (B 0)
            (2, 0, 3 * g(4, 2), 4),                       # the environment pair before the self pair (0, 2)
            (1, 1, 3 * g(5, 1), 3 * g(5, 1) + 2),         # self pairs (0, 2) and (0, 1): the earlier template entry
            (-1, -1, NONE, NONE)]
    assert list(zip(fi.tolist(), kind.tolist(), first.tolist(), second.tolist())) == want
    assert rec[[0, 1, 6]].tobytes() == np.full(3, cleared_contact()).tobytes()
    assert counts[1] == 6 and counts[3] == 2 + 2 + 1  # (the folded samples: both template pairs each; ES: one)
