"""The motion certification's answers by brute force (no GPU needed), under the contract of hfb_env_certify_motions
(include/hppfcl_b200.h): boxes from the host build of the device code, the sides of every sample, the environment
candidates from the library's host cross finder on the boxes widened on the host, the self candidates from
hfb_broadphase_sweep_pairs, the oracle's collide() on every candidate, then the per-sample flags and the outputs.  A
hand-made sample of spheres makes each rule decide something; the reference build agrees on every record, and so on
every lower bound used, and its outputs are recorded in tests/golden/reference_outputs_certify.json.gz
(HFB_RECORD_REFERENCE=<that file> records them where oracle/_ref is built).  tests/test_gpu_env_certify.py checks the
device against the same contract and the recorded sample.  Soundness on the CPU: every certified segment of a few robot motions,
resampled by forward kinematics, has no colliding interior sample."""
import gzip
import json
import os

import numpy as np

from tests import common
from tests.common import P, hf, make_scenes
from oracle import oracle_lib
from hppfcl_b200 import workloads as W

# the reference's recorded outputs for the sample's calls, looked up with those of tests/golden/reference_outputs.json.gz
# where oracle/_ref is not built
REF_OUTPUTS = os.path.join(common.ROOT, "tests", "golden", "reference_outputs_certify.json.gz")
DMAX = np.finfo(np.float64).max


def load_recorded():
    if os.path.exists(REF_OUTPUTS):
        common._load_recorded().update(json.load(gzip.open(REF_OUTPUTS, "rt")))


def add_ru(a, r):
    """a + r rounded up (the nearest sum stepped outward when its TwoSum error lies outward), as the host build does"""
    with np.errstate(all="ignore"):
        s = a + r
        z = s - a
        e = (a - (s - z)) + (r - z)
        return np.where(e > 0, np.nextafter(s, np.inf), s)


def sub_rd(a, r):
    with np.errstate(all="ignore"):
        s = a - r
        z = s - a
        e = (a - (s - z)) - (r + z)
        return np.where(e < 0, np.nextafter(s, -np.inf), s)


def half_ru(s):
    h = s * 0.5
    return np.where(h + h < s, np.nextafter(h, np.inf), h)


def reach(r, left):
    with np.errstate(invalid="ignore"):
        s = np.maximum(np.where(r > 0, r, 0.0), np.where(left > 0, left, 0.0))
    return half_ru(s)


def sides(sweep, links, off, m0, nm):
    """(right, left) per object: the sweep bound of the segment to the next / from the previous sample, NaN when the
    segment does not exist, the motion is outside the range or the bound is not finite and >= 0"""
    n = len(sweep)
    valid = np.where(np.isfinite(sweep) & (sweep >= 0), sweep, np.nan)
    r, left = np.full(n, np.nan), np.full(n, np.nan)
    for m in range(m0, m0 + nm):
        a, b = int(off[m]) * links, int(off[m + 1]) * links
        if b - a > links:
            r[a:b - links] = valid[a:b - links]
            left[a + links:b] = valid[a:b - links]
    return r, left


def contract(orc, emu, ha, tfa, hb, tfb, links, tpl, off, sweep, req=None, m0=0, nm=None):
    """the certification by brute force -> (first_invalid, first_uncertified, certified, counts = (env candidates, self
    candidates, unsupported, uncertified), the candidates' (h1, tf1, h2, tf2) and the oracle's records of them)"""
    req = req or P.CollisionRequestPOD()
    tpl = np.asarray(tpl, dtype=np.uint32).reshape(-1, 2)
    n_m = len(off) - 1
    nm = n_m - m0 if nm is None else nm
    n_cfg = len(ha) // links
    g0, g1 = int(off[m0]), int(off[m0 + nm])
    bb_a = emu.scene_aabbs(ha, tfa)
    bb_b = emu.scene_aabbs(hb, tfb) if len(hb) else np.zeros((0, 6))
    r, left = sides(np.asarray(sweep, dtype=np.float64), links, off, m0, nm)
    w = reach(r, left)
    empty = (bb_a[:, 0] == DMAX) & (bb_a[:, 3] == -DMAX)
    wbb = bb_a.copy()
    wbb[:, :3] = np.where(empty[:, None], bb_a[:, :3], sub_rd(bb_a[:, :3], w[:, None]))
    wbb[:, 3:] = np.where(empty[:, None], bb_a[:, 3:], add_ru(bb_a[:, 3:], w[:, None]))
    if len(hb):
        ef, es = hf.broadphase_cross_pairs(wbb, bb_b)
        keep = (ef >= g0 * links) & (ef < g1 * links)
        ef, es = ef[keep], es[keep]
    else:
        ef = es = np.zeros(0, np.uint32)
    sf, ss = hf.broadphase_sweep_pairs(bb_a, sweep, links, tpl, off, m0, nm)
    f = np.concatenate([ef, sf]).astype(np.int64)
    h2 = np.concatenate([hb[es], ha[ss]]).astype(np.uint32)
    tf2 = np.concatenate([tfb[es], tfa[ss]])
    args = (ha[f].astype(np.uint32), tfa[f], h2, tf2)
    minus_inf = req.security_margin == -np.inf
    if minus_inf or len(f) == 0:
        rec = np.zeros(0, dtype=P.contact_dtype)
    else:
        rec = orc.batch_collide(*args, req=req, nthreads=0)
    pr = np.full(n_cfg, False)
    pl = np.full(n_cfg, False)
    for g in range(g0, g1):
        pr[g] = not np.isnan(r[g * links:(g + 1) * links]).any()
        pl[g] = not np.isnan(left[g * links:(g + 1) * links]).any()
    collides = np.zeros(n_cfg, bool)
    n_env = len(ef)
    for p in range(len(rec)):
        a = int(f[p])
        b = int(es[p]) if p < n_env else int(ss[p - n_env])
        g = a // links
        sr, sl = r[a], left[a]
        if p >= n_env:
            sr, sl = add_ru(sr, r[b]), add_ru(sl, left[b])
        unsup = P.status_path(rec["status"][p]) == P.PATH_UNSUPPORTED
        clear = rec["num_contacts"][p] == 0 and not unsup
        with np.errstate(over="ignore"):  # (DBL_MAX doubles to +inf)
            d2 = 2.0 * rec["distance_lower_bound"][p]
        pr[g] &= bool(clear and d2 > sr)
        pl[g] &= bool(clear and d2 > sl)
        y = bb_b[b] if p < n_env else bb_a[b]
        x = bb_a[a]
        if rec["num_contacts"][p] > 0 and not (x[:3] > y[3:]).any() and not (x[3:] < y[:3]).any():
            collides[g] = True
    fi = np.full(n_m, -1, np.int32)
    fu = np.full(n_m, -1, np.int32)
    cert = np.zeros(n_cfg, np.uint8)
    n_unc = 0
    for m in range(m0, m0 + nm):
        a, b = int(off[m]), int(off[m + 1])
        hit = np.flatnonzero(collides[a:b])
        if len(hit):
            fi[m] = hit[0]
        for g in range(a, b - 1):
            cert[g] = pr[g] and pl[g + 1]
            if not cert[g]:
                n_unc += 1
                if fu[m] < 0:
                    fu[m] = g - a
    unsup = int((P.status_path(rec["status"]) == P.PATH_UNSUPPORTED).sum()) if len(rec) else 0
    return fi, fu, cert, (n_env, len(sf), unsup, n_unc), args, rec


def hand_sample(sc):
    """configurations of two spheres (radius 0.25), each at its own place, environment spheres placed next to them,
    and a mesh link next to a plane -> (ha, tfa, hb, tfb, links, tpl, offsets, sweep, names)"""
    sph = int(sc.register_shapes(P.make_shapes([P.GEOM_SPHERE], [[0.25, 0, 0]]))[0])
    verts, tris = W.sphere_mesh(0.25, 8, 4)
    bid = sc.register_bvh(verts, tris)[0]
    mesh = int(sc.register_shapes(P.make_shapes([P.BV_OBBRSS], [[0, 0, 0]], data=[bid]))[0])
    plane = int(sc.register_halfspaces(P.GEOM_PLANE, [[1, 0, 0, 1000.0]])[0])
    apart = [(0, 0, 0), (2, 0, 0)]
    # (links, environment spheres near link 0 as offsets, link handles)
    kinds = {
        "F": (apart, []),                                  # nothing within reach: certified through culled pairs
        "D": (apart, [(0.6, 0.6, 0)]),                     # a candidate whose lower bound, 0.349, certifies 0.6
        "X": (apart, [(1.0, 0, 0)]),                       # distance 0.5 exactly: 2 lb == s = 1.0, uncertified
        "M": (apart, [(0.55, 0.55, 0)]),                   # box gap 0.05, distance 0.278: a contact under a margin
                                                           # of 0.3 only
    }
    motions = [("culled", ["F", "F", "F"], 0.5), ("lower bounds", ["D", "D"], 0.6), ("2 lb == s", ["F", "X"], 1.0),
               ("margin", ["F", "M", "F"], 0.2), ("NaN sweep", ["F", "F"], np.nan), ("one sample", ["F"], 0.5),
               ("empty", [], 0.5), ("mesh and plane", ["F", "P"], 0.1), ("overlap", ["F", "O"], 0.1)]
    T, HA, B, SW = [], [], [], []
    g = 0
    for _, samples, s in motions:
        for k in samples:
            x0 = 10.0 * g
            if k == "P":  # the mesh link's box 0.012 short of the plane (reach 0.05); the sphere link far from it
                T += [(999.75, 0, 5.0 * g), (990.0, 0, 5.0 * g)]
                HA += [mesh, sph]
            elif k == "O":  # an environment sphere on link 0: the sample collides
                T += [(x0, 0, 0), (x0 + 2, 0, 0)]
                HA += [sph, sph]
                B.append((x0 + 0.3, 0, 0))
            else:
                links, env = kinds[k]
                T += [(x0 + x, y, z) for x, y, z in links]
                HA += [sph, sph]
                B += [(x0 + x, y, z) for x, y, z in env]
            SW += [s, s]
            g += 1
    off = np.concatenate([[0], np.cumsum([len(m[1]) for m in motions])]).astype(np.uint32)
    hb = np.array([sph] * len(B) + [plane], dtype=np.uint32)
    tfb = W.identity_transforms(len(B) + 1, T=B + [(0, 0, 0)])
    return (np.array(HA, dtype=np.uint32), W.identity_transforms(len(T), T=T), hb, tfb, 2, [(0, 1)], off,
            np.array(SW, dtype=np.float64), [m[0] for m in motions])


def margin_request(m):
    req = P.CollisionRequestPOD()
    req.security_margin = m
    return req


def reference_sample(sc):
    """the hand sample under margins 0 and 0.3 -> ([(scene, request, answer)], all candidates as (h1, tf1, h2, tf2,
    request, oracle records))"""
    scene = hand_sample(sc)
    sc.commit()
    orc, emu = sc.b["oracle"], sc.b["emu"]
    out, used = [], []
    for m in (0.0, 0.3):
        req = margin_request(m)
        ans = contract(orc, emu, *scene[:8], req=req)
        out.append((scene, req, ans))
        used.append((ans[4], req, ans[5]))
    return out, used


def check_against_reference(sc, used):
    """the reference build's collide() on every candidate of the sample gives the oracle's record"""
    for args, req, orec in used:
        rr = sc.b["ref"].batch_collide(*args, req=req)
        # an unsupported pair (a mesh against a plane, which the library does not collide): its record is the cleared
        # one, distance_lower_bound DBL_MAX, and no lower bound of it is used -- the pair fails every side
        un = P.status_path(orec["status"]) == P.PATH_UNSUPPORTED
        assert (orec["distance_lower_bound"][un] == DMAX).all() and (orec["num_contacts"][un] == 0).all()
        rr, orec = rr[~un], orec[~un]
        # the fields the reference's collide() defines (test_reference_build's set), the lower bound among them
        for f in ("p1", "p2", "normal", "pos", "distance_lower_bound", "b1", "b2", "num_contacts"):
            x, y = rr[f], orec[f]
            ok = (x == y) | (np.isnan(x) & np.isnan(y)) if x.dtype.kind == "f" else x == y
            assert np.all(ok), "%s differs from the reference build at rows %s" % (f, np.flatnonzero(~ok.reshape(len(x), -1).all(1)))


def test_certify_reference_sample():
    """each rule of the contract decides a segment of the hand sample, on records the reference build agrees with"""
    oracle_lib.build_ref()
    load_recorded()
    sc = make_scenes(ref=True, emu=True)
    out, used = reference_sample(sc)
    check_against_reference(sc, used)
    names = out[0][0][8]
    ix = {n: k for k, n in enumerate(names)}
    off = out[0][0][6]
    (fi, fu, cert, counts, _, rec), (fi1, fu1, cert1, counts1, _, rec1) = out[0][2], out[1][2]
    seg = lambda name: cert[int(off[ix[name]]):int(off[ix[name] + 1]) - 1].tolist()  # noqa: E731
    assert seg("culled") == [1, 1]
    assert seg("lower bounds") == [1]
    assert seg("2 lb == s") == [0]
    assert seg("margin") == [1, 1]
    assert seg("NaN sweep") == [0]
    assert seg("one sample") == [] and seg("empty") == []
    # the mesh link widened onto the plane: an HFB_PATH_UNSUPPORTED record, whose cleared lower bound (DBL_MAX) would
    # pass any threshold -- the unsupported rule alone fails the segment
    assert seg("mesh and plane") == [0] and counts[2] == 1
    m = ix["mesh and plane"]
    unsup = P.status_path(rec["status"]) == P.PATH_UNSUPPORTED
    assert unsup.sum() == 1 and rec["distance_lower_bound"][unsup][0] == DMAX
    assert fi.tolist() == [-1] * 8 + [1]
    assert fu.tolist() == [-1, -1, 0, -1, 0, -1, -1, 0, 0]
    # the exact tie: a lower bound of 0.5 against a threshold of 1.0
    assert (rec["distance_lower_bound"] == 0.5).sum() == 2  # (both links are 0.5 from the sphere)
    # under a margin of 0.3 the widened-only pair reports a contact: the sample stays valid, its segments fail
    m = ix["margin"]
    assert fi1[m] == -1 and fu1[m] == 0
    assert cert1[int(off[m]):int(off[m + 1]) - 1].tolist() == [0, 0]
    assert (rec1["num_contacts"] > 0).sum() > (rec["num_contacts"] > 0).sum()


def test_certified_segments_are_free_on_the_cpu():
    """chain_sweep_bounds + 2e-6 m: every certified segment of a few robot motions, resampled at 16 interior points by
    forward kinematics, has no colliding interior sample (the oracle's collide() on every box candidate)"""
    sc = make_scenes(emu=True)
    w = W.robot_motions(6, n_env=300, room=3.0, seed=71)
    hs = w["register"](sc, oracle=True)
    sc.commit()
    ha, tfa = hs[w["geom_a"]].astype(np.uint32), w["tf_a"]
    hb, tfb = hs[w["geom_b"][1:]].astype(np.uint32), w["tf_b"][1:]  # (without the floor)
    sweep = W.chain_sweep_bounds(w) + 2e-6
    L, tpl, off = 16, W.chain_self_pairs(16), w["offsets"]
    fi, fu, cert, counts, _, _ = contract(sc.b["oracle"], sc.b["emu"], ha, tfa, hb, tfb, L, tpl, off, sweep)
    assert cert.any()
    fine = W.resample_motions(w, np.flatnonzero(cert), 16)
    hf_ = hs[np.tile(w["geom_a"][:L], len(fine) // L)].astype(np.uint32)
    orc, emu = sc.b["oracle"], sc.b["emu"]
    bb = emu.scene_aabbs(hf_, fine)
    ef, es = hf.broadphase_cross_pairs(bb, emu.scene_aabbs(hb, tfb))
    sf, ss = hf.broadphase_config_pairs(bb, L, tpl)
    er = orc.batch_collide(hf_[ef], fine[ef], hb[es], tfb[es], nthreads=0)
    sr = orc.batch_collide(hf_[sf], fine[sf], hf_[ss], fine[ss], nthreads=0)
    assert (er["num_contacts"] == 0).all() and (sr["num_contacts"] == 0).all()
