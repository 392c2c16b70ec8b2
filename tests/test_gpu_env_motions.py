"""The motions query (hfb_env_collide_motions*): per motion, a run of robot configurations, the first sample that
collides with the resident environment or with itself, and the first colliding pair there.  It must equal the
composition of the configurations query (hfb_env_collide_configs with every pair, then the host reduction by the
contract: environment pairs by link, then by B index, then self pairs in template order)."""
import numpy as np
import pytest

from tests.common import P, compare_distance, hf, make_scenes
from tests.test_env_motions_reference import MESH_FIELDS, cleared_contact, contract, load_recorded, reference_sample
from tests.test_gpu_edge_inputs import NONFINITE_FIELDS, same_fields
from tests.test_gpu_env_configs import BIG_CAP, dev
from hppfcl_b200 import workloads as W

pytestmark = pytest.mark.gpu

LINKS = 16
TPL = W.chain_self_pairs(LINKS)
NONE = 0xFFFFFFFF


def motion_scene(eng, n_motions=1024, n_env=500, room=3.0, seed=37, oracle=False):
    """robot_motions with the bending joints in +-2.8 rad (some samples fold onto themselves), a Plane wall added to B,
    the floor and the large boxes moved out of reach as in test_gpu_env_configs.config_scene -> (w, ha, tfa, hb, tfb)"""
    w = W.robot_motions(n_motions, n_env=n_env, room=room, seed=seed, joint_range=2.8)
    hs = w["register"](eng, oracle=oracle)
    ha, tfa = hs[w["geom_a"]].astype(np.uint32), w["tf_a"]
    hb, tfb = hs[w["geom_b"]].astype(np.uint32), w["tf_b"].copy()
    wall = eng.register_halfspaces(P.GEOM_PLANE, [[1, 0, 0, -0.5]])
    hb[-1] = wall[0]
    tfb[-1] = W.identity_transforms(1)[0]
    tfb[0] = W.identity_transforms(1, T=[[0.0, 0.0, -2.0]])[0]
    tfb["T"][(w["geom_b"] >= LINKS + 64) & (w["geom_b"] < LINKS + 80), 2] += 10.0  # the tables and shelves
    eng.commit()
    return w, ha, tfa, hb, tfb


def reduce_motions(off, n_b, env_pairs, self_pairs, tpl=TPL, links=LINKS, m0=0, nm=None):
    """the contract's reduction on the host: env_pairs / self_pairs = (first, second, records) of the colliding pairs
    (second: index in B / in A) -> (first_invalid, kind, first, second, records)"""
    n = len(off) - 1
    nm = n - m0 if nm is None else nm
    entry = {(int(i), int(j)): k for k, (i, j) in enumerate(np.asarray(tpl).reshape(-1, 2))}
    best = {}  # configuration -> (ordinal, kind, first, second, record)
    for kind, (f, s, rec) in enumerate((env_pairs, self_pairs)):
        for a, b, r in zip(np.asarray(f).tolist(), np.asarray(s).tolist(), rec):
            g = a // links
            o = (a % links) * n_b + b if kind == 0 else links * n_b + entry[(a % links, b % links)]
            if g not in best or o < best[g][0]:
                best[g] = (o, kind, a, b, r)
    fi = np.full(n, -1, dtype=np.int32)
    kd = np.full(n, -1, dtype=np.int8)
    first = np.full(n, NONE, dtype=np.uint32)
    second = np.full(n, NONE, dtype=np.uint32)
    recs = np.full(n, cleared_contact(), dtype=P.contact_dtype)
    for m in range(m0, m0 + nm):
        for g in range(int(off[m]), int(off[m + 1])):
            if g in best:
                _, kd[m], first[m], second[m], recs[m] = best[g]
                fi[m] = g - int(off[m])
                break
    return fi, kd, first, second, recs


def composition(eng, env, ha, tfa, n_b, off, tpl=TPL, req=None, m0=0, nm=None):
    """the motions query composed from hfb_env_collide_configs: every colliding pair of the range's configurations,
    then reduce_motions -> (first_invalid, kind, first, second, records, counts)"""
    n = len(off) - 1
    nm = n - m0 if nm is None else nm
    g0, g1 = int(off[m0]), int(off[m0 + nm])
    _, e, s = eng.env_collide_configs(env, ha, tfa, LINKS, tpl, req, BIG_CAP, BIG_CAP, first_config=g0,
                                      num_configs=g1 - g0)
    assert e[4] <= BIG_CAP and s[4] <= BIG_CAP
    return reduce_motions(off, n_b, e[:3], s[:3], tpl, m0=m0, nm=nm) + ((e[3], e[4], s[3], s[4]),)


def assert_same(got, want):
    for k in range(4):
        assert np.array_equal(got[k], want[k]), k
    assert got[4].tobytes() == want[4].tobytes()
    assert tuple(got[5]) == tuple(want[5])


def test_motions_match_the_composition():
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = motion_scene(eng)
    env = eng.env_create(hb, tfb)
    off = w["offsets"]
    n = len(off) - 1
    got = eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off)
    want = composition(eng, env, ha, tfa, len(hb), off)
    assert_same(got, want)
    fi, kind = got[0], got[1]
    samples = np.diff(off)
    # every case occurs: valid motions, invalid at the first sample, in the middle, at the last; both witness kinds
    assert (fi < 0).sum() >= 20 and (fi == 0).sum() >= 5 and ((fi > 0) & (fi < samples - 1)).sum() >= 20
    assert (kind == 0).sum() >= 20 and (kind == 1).sum() >= 5 and got[5][1] > 100 and got[5][3] > 40
    assert (fi == samples - 1).sum() >= 1
    # past every grid cap the configurations tests reach
    assert len(ha) > 300_000 and got[5][0] > 100_000
    # first_invalid alone
    only = eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off, witness=False)
    assert np.array_equal(only[0], fi) and only[1] is None and only[5] == got[5]
    # motion ranges add up to the whole; the motions outside a range get the no-witness values
    cleared = np.full(n, cleared_contact(), dtype=P.contact_dtype)
    counts = np.zeros(4, dtype=np.int64)
    merged = [np.full(n, -1, dtype=np.int32), np.full(n, -1, dtype=np.int8), np.full(n, NONE, dtype=np.uint32),
              np.full(n, NONE, dtype=np.uint32), cleared.copy()]
    for m0, nm in ((0, 300), (300, 1), (301, 0), (301, n - 301)):
        r = eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off, first_motion=m0, num_motions=nm)
        assert_same(r, composition(eng, env, ha, tfa, len(hb), off, m0=m0, nm=nm))
        out = np.ones(n, dtype=bool)
        out[m0:m0 + nm] = False
        assert (r[0][out] == -1).all() and (r[1][out] == -1).all() and (r[2][out] == NONE).all()
        assert r[4][out].tobytes() == cleared[out].tobytes()
        for k in range(5):
            merged[k][m0:m0 + nm] = r[k][m0:m0 + nm]
        counts += r[5]
    assert all(np.array_equal(a, b) for a, b in zip(merged[:4], got[:4])) and merged[4].tobytes() == got[4].tobytes()
    assert tuple(counts) == got[5]
    # an empty template: environment pairs only
    empty = np.zeros((0, 2), dtype=np.uint32)
    assert_same(eng.env_collide_motions(env, ha, tfa, LINKS, empty, off), composition(eng, env, ha, tfa, len(hb), off, empty))
    # security_margin = -inf: candidates counted, no contacts, every motion valid
    req = P.CollisionRequestPOD()
    req.security_margin = -np.inf
    r = eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off, req)
    assert (r[0] == -1).all() and (r[1] == -1).all() and r[4].tobytes() == cleared.tobytes()
    assert r[5] == (got[5][0], 0, got[5][2], 0)
    eng.env_destroy(env)


def test_small_scene_and_every_refusal():
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = motion_scene(eng, n_motions=40, seed=41)
    env = eng.env_create(hb, tfb)
    off = w["offsets"]
    n_configs = len(ha) // LINKS
    # empty motions anywhere, one of them at each end
    off2 = np.concatenate([[0, 0], off[1:5], off[4:5], off[5:], off[-1:]]).astype(np.uint32)
    for o in (off, off2):
        assert_same(eng.env_collide_motions(env, ha, tfa, LINKS, TPL, o), composition(eng, env, ha, tfa, len(hb), o))
    r = eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off2)
    assert r[0][0] == -1 and r[0][5] == -1 and r[0][-1] == -1
    req = P.CollisionRequestPOD()
    req.num_max_contacts = 0
    for call in (lambda: eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off, req),
                 lambda: eng.env_collide_motions(env, ha, tfa, LINKS, [(0, 2), (2, 0)], off),
                 lambda: eng.env_collide_motions(env, ha, tfa, LINKS, TPL, np.concatenate([[1], off[1:]])),
                 lambda: eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off[[0, 2, 1] + list(range(3, len(off)))]),
                 lambda: eng.env_collide_motions(env, ha, tfa, LINKS, TPL, np.append(off[:-1], n_configs + 1)),
                 lambda: eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off[:-1]),
                 lambda: eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off, first_motion=len(off) - 1, num_motions=1),
                 lambda: eng.env_collide_motions(env, ha[:-1], tfa[:-1], LINKS, TPL, off),
                 lambda: eng.env_collide_motions(env, ha, tfa, 0, TPL, off)):
        with pytest.raises(hf.EngineError, match="invalid argument"):
            call()
    eng.env_destroy(env)


def test_env_without_objects_empty_template_and_empty_motions():
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = motion_scene(eng, n_motions=128, seed=43)
    off = w["offsets"]
    n = len(off) - 1
    env = eng.env_create(hb[:0], tfb[:0])
    got = eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off)
    assert_same(got, composition(eng, env, ha, tfa, 0, off))
    assert (got[1] == 1).sum() >= 5 and not (got[1] == 0).any() and got[5][:2] == (0, 0)
    # no env objects and an empty template: nothing to check
    r = eng.env_collide_motions(env, ha, tfa, LINKS, np.zeros((0, 2), dtype=np.uint32), off)
    assert (r[0] == -1).all() and r[5] == (0, 0, 0, 0)
    eng.env_destroy(env)
    env = eng.env_create(hb, tfb)
    # all motions empty: no configurations at all
    r = eng.env_collide_motions(env, ha[:0], tfa[:0], LINKS, TPL, np.zeros(5, dtype=np.uint32))
    assert (r[0] == -1).all() and len(r[0]) == 4 and r[4].tobytes() == np.full(4, cleared_contact()).tobytes()
    r = eng.env_collide_motions(env, ha[:0], tfa[:0], LINKS, TPL, [0])
    assert len(r[0]) == 0 and r[5] == (0, 0, 0, 0)
    eng.env_destroy(env)


def test_update_invalidates_a_motion():
    """an environment object moved onto a link of a middle sample of a valid motion: the motion turns invalid at the
    sample the oracle expects -- the first whose links the moved object collides with, by the oracle's collide() of
    that object against every link of every sample of the motion -- with that object and the lowest such link as the
    witness, and the oracle's record"""
    sc = make_scenes(gpu=True, emu=False)
    eng, orc = sc.b["gpu"], sc.b["oracle"]
    w, ha, tfa, hb, tfb = motion_scene(sc, n_motions=128, seed=47, oracle=True)
    tfb = tfb.copy()
    env = eng.env_create(hb, tfb)
    off = w["offsets"]
    before = eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off)
    valid = [int(m) for m in np.nonzero(before[0] < 0)[0] if off[m + 1] - off[m] >= 8]
    m = valid[len(valid) // 2]
    n_s = int(off[m + 1] - off[m])
    g = int(off[m]) + n_s // 2
    k = next(i for i in range(20, len(hb) - 1) if LINKS <= w["geom_b"][i] < LINKS + 64)  # a small object of B
    t = tfb[[k]].copy()
    t["T"] = tfa["T"][g * LINKS + 9]  # (the object's centre inside link 9: they collide at that sample)
    eng.env_update(env, [k], t)
    got = eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off)
    assert_same(got, composition(eng, env, ha, tfa, len(hb), off))
    # the oracle's expectation: the moved object against every link of every sample of motion m
    links = np.arange(int(off[m]) * LINKS, int(off[m + 1]) * LINKS)
    ro = orc.batch_collide(ha[links], tfa[links], np.repeat(hb[k], len(links)), np.repeat(t, len(links)), nthreads=0)
    hit = np.flatnonzero(ro["num_contacts"] > 0)
    assert len(hit) and hit[0] // LINKS <= n_s // 2
    k_sample, link = divmod(int(hit[0]), LINKS)
    assert got[0][m] == k_sample and got[1][m] == 0 and got[3][m] == k
    assert got[2][m] == (int(off[m]) + k_sample) * LINKS + link
    compare_distance(ro[hit[:1]], got[4][m:m + 1], what="the witness against the oracle")
    assert (got[0] != before[0]).sum() >= 1 and got[0][m] >= 0
    eng.env_destroy(env)


class DeviceOut:
    """device buffers of the motions query, pre-filled with a sentinel, and their download"""

    def __init__(self, n):
        import torch
        self.n = n
        self.fi = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        self.kind = torch.full((n,), 7, dtype=torch.int8, device="cuda")
        self.first = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        self.second = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        self.rec = torch.full((n * P.contact_dtype.itemsize,), 7, dtype=torch.uint8, device="cuda")
        self.cnt = torch.full((4,), 7, dtype=torch.int32, device="cuda")

    def ptrs(self):
        c = self.cnt.data_ptr()
        return dict(d_first_invalid=self.fi.data_ptr(), d_kind=self.kind.data_ptr(), d_first=self.first.data_ptr(),
                    d_second=self.second.data_ptr(), d_contacts=self.rec.data_ptr(), d_counts=(c, c + 4, c + 8, c + 12))

    def result(self):
        return (self.fi.cpu().numpy(), self.kind.cpu().numpy(), self.first.cpu().numpy().view(np.uint32),
                self.second.cpu().numpy().view(np.uint32), self.rec.cpu().numpy().view(P.contact_dtype),
                tuple(int(x) for x in self.cnt.cpu().numpy()))

    def untouched(self):
        return all((t.cpu().numpy() == 7).all() for t in (self.fi, self.kind, self.first, self.second, self.rec, self.cnt))


def test_device_form_equals_host_form_and_refusals_write_nothing():
    import torch
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = motion_scene(eng, n_motions=256, seed=53)
    env = eng.env_create(hb, tfb)
    off = w["offsets"]
    n = len(off) - 1
    stream = torch.cuda.Stream()
    rng = np.random.default_rng(2)
    for k, (m0, nm) in enumerate(((0, n), (40, 100), (0, n))):
        t = tfa.copy()
        t["T"] += rng.uniform(-0.2, 0.2, (len(ha) // LINKS, 1, 3)).repeat(LINKS, axis=1).reshape(-1, 3) * (k % 2)
        d = DeviceOut(n)
        d_h, d_t = dev(ha), dev(t)
        torch.cuda.synchronize()
        eng.env_collide_motions_device(env, len(ha), d_h.data_ptr(), d_t.data_ptr(), LINKS, TPL, off, **d.ptrs(),
                                       stream=stream.cuda_stream, first_motion=m0, num_motions=nm)
        stream.synchronize()
        host = eng.env_collide_motions(env, ha, t, LINKS, TPL, off, first_motion=m0, num_motions=nm)
        assert_same(d.result(), host)
        assert (host[0] >= 0).sum() > 10
    # first_invalid alone in the device form
    d = DeviceOut(n)
    d_h, d_t = dev(ha), dev(tfa)
    torch.cuda.synchronize()
    p = d.ptrs()
    eng.env_collide_motions_device(env, len(ha), d_h.data_ptr(), d_t.data_ptr(), LINKS, TPL, off, p["d_first_invalid"], None,
                                   None, None, None, stream=stream.cuda_stream)
    stream.synchronize()
    host = eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off)
    assert np.array_equal(d.fi.cpu().numpy(), host[0]) and (d.kind.cpu().numpy() == 7).all()
    # the offsets refusals on the device path write nothing
    n_configs = len(ha) // LINKS
    for bad, m0, nm in ((np.concatenate([[1], off[1:]]), 0, None), (off[[0, 2, 1] + list(range(3, len(off)))], 0, None),
                        (np.append(off[:-1], n_configs + 1), 0, None), (off, n, 1)):
        d = DeviceOut(n)
        torch.cuda.synchronize()
        with pytest.raises(hf.EngineError, match="invalid argument"):
            eng.env_collide_motions_device(env, len(ha), d_h.data_ptr(), d_t.data_ptr(), LINKS, TPL, bad, **d.ptrs(),
                                           stream=stream.cuda_stream, first_motion=m0, num_motions=nm)
        torch.cuda.synchronize()
        assert d.untouched()
    eng.env_destroy(env)


def test_device_call_then_host_env_calls_unsynchronised():
    """the device form returns while its narrow phase and reductions still run on the caller's stream; host env calls
    on the same context that follow with no synchronisation in between must wait for it: both results right"""
    import torch
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = motion_scene(eng, n_motions=256, seed=59)
    env = eng.env_create(hb, tfb)
    off = w["offsets"]
    n = len(off) - 1
    t_other = tfa.copy()
    t_other["T"] += 0.15
    want_dev = eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off)
    want_mot = eng.env_collide_motions(env, ha, t_other, LINKS, TPL[::2], off)
    want_cfg = eng.env_collide_configs(env, ha, t_other, LINKS, TPL, env_capacity=0, self_capacity=0)
    d_h, d_t = dev(ha), dev(tfa)
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    for host_call, check in ((lambda: eng.env_collide_motions(env, ha, t_other, LINKS, TPL[::2], off),
                              lambda r: assert_same(r, want_mot)),
                             (lambda: eng.env_collide_configs(env, ha, t_other, LINKS, TPL, env_capacity=0, self_capacity=0),
                              lambda r: np.array_equal(r[0], want_cfg[0]))):
        d = DeviceOut(n)
        torch.cuda.synchronize()
        eng.env_collide_motions_device(env, len(ha), d_h.data_ptr(), d_t.data_ptr(), LINKS, TPL, off, **d.ptrs(),
                                       stream=side.cuda_stream)
        got = host_call()  # no synchronisation in between
        side.synchronize()
        assert check(got) is not False
        assert_same(d.result(), want_dev)
    eng.env_destroy(env)


def test_nonfinite_and_huge_poses():
    """a sample with a NaN pose and one displaced by 1e100: the oracle's answer there -- its collide() on every
    candidate (the library's host pair finders), reduced by the contract -- and the composition's everywhere"""
    sc = make_scenes(gpu=True, emu=False)
    eng, orc = sc.b["gpu"], sc.b["oracle"]
    w, ha, tfa, hb, tfb = motion_scene(sc, n_motions=24, n_env=600, seed=61, oracle=True)
    off = w["offsets"]
    tfa = tfa.copy()
    m_nan, m_far = 3, 7
    g_nan, g_far = int(off[m_nan]) + 2, int(off[m_far]) + 1
    tfa["T"][g_nan * LINKS + 6, 1] = np.nan
    tfa["R"][g_nan * LINKS + 11, 4] = np.inf
    tfa["T"][g_far * LINKS:(g_far + 1) * LINKS] += 1e100
    env = eng.env_create(hb, tfb)
    got = eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off)
    assert_same(got, composition(eng, env, ha, tfa, len(hb), off))
    for m in (m_nan, m_far):
        sub = slice(int(off[m]) * LINKS, int(off[m + 1]) * LINKS)
        a_h, a_t = ha[sub], tfa[sub]
        bb_a, bb_b = eng.scene_aabbs(a_h, a_t), eng.scene_aabbs(hb, tfb)
        ef, es = hf.broadphase_cross_pairs(bb_a, bb_b)
        sf, ss = hf.broadphase_config_pairs(bb_a, LINKS, TPL)
        re_ = orc.batch_collide(a_h[ef], a_t[ef], hb[es], tfb[es], nthreads=0)
        rs = orc.batch_collide(a_h[sf], a_t[sf], a_h[ss], a_t[ss], nthreads=0)
        he, hs = re_["num_contacts"] > 0, rs["num_contacts"] > 0
        base = np.uint32(off[m] * LINKS)
        local = np.array([0, off[m + 1] - off[m]], dtype=np.uint32)
        want = reduce_motions(local, len(hb), (ef[he], es[he], re_[he]), (sf[hs], ss[hs], rs[hs]))
        assert got[0][m] == want[0][0] and got[1][m] == want[1][0]
        if want[1][0] < 0:
            assert m != m_far and got[4][m:m + 1].tobytes() == want[4][:1].tobytes()
            continue
        assert got[2][m] == want[2][0] + base
        assert got[3][m] == want[3][0] + (base if want[1][0] == 1 else 0)
        a = int(got[2][m])
        other = (hb, tfb) if want[1][0] == 0 else (ha, tfa)
        finite = all(np.isfinite(x["T"]).all() and np.isfinite(x["R"]).all() for x in (tfa[a], other[1][int(got[3][m])]))
        mesh = P.status_path(want[4]["status"][:1])[0] == P.PATH_BVH  # (`iterations`: the oracle's BV and leaf counters)
        if finite and not mesh:
            compare_distance(want[4][:1], got[4][m:m + 1], what="witness against the oracle")
        else:
            same_fields(want[4][:1], got[4][m:m + 1], MESH_FIELDS if finite else NONFINITE_FIELDS,
                        "witness against the oracle")
    assert got[0][m_far] >= 0 and got[0][m_far] <= 1  # the displaced sample folds every template pair onto one point
    eng.env_destroy(env)


def test_answers_equal_the_reference_sample():
    """the device's answers on the reference sample (tests/test_env_motions_reference.py) are the contract's, found by
    brute force with the oracle: first colliding samples, every tie rule's witness and its record; the reference build
    agrees with the oracle on every witness (its recorded outputs where it is not built here)"""
    load_recorded()
    sc = make_scenes(gpu=True, emu=True, ref=True)
    eng = sc.b["gpu"]
    scenes, args, orec = reference_sample(sc)
    rr = sc.b["ref"].batch_collide(*args)
    for f in MESH_FIELDS:
        x, y = rr[f], orec[f]
        assert np.all((x == y) | (np.isnan(x) & np.isnan(y)) if x.dtype.kind == "f" else x == y), f
    for ha, tfa, hb, tfb, links, tpl, off, (fi, kind, first, second, rec, counts) in scenes:
        env = eng.env_create(hb, tfb)
        got = eng.env_collide_motions(env, ha, tfa, links, tpl, off)
        assert got[0].tobytes() == fi.tobytes() and got[1].tobytes() == kind.tobytes()
        assert got[2].tobytes() == first.tobytes() and got[3].tobytes() == second.tobytes()
        assert got[5] == counts
        w = kind >= 0
        mesh = P.status_path(rec["status"]) == P.PATH_BVH
        compare_distance(rec[w & ~mesh], got[4][w & ~mesh], what="witness records against the oracle")
        for f in MESH_FIELDS:  # (mesh records: `iterations` holds the BV and leaf counters, which the device does not keep)
            x, y = rec[w & mesh][f], got[4][w & mesh][f]
            assert np.all((x == y) | (np.isnan(x) & np.isnan(y)) if x.dtype.kind == "f" else x == y), f
        assert got[4][~w].tobytes() == rec[~w].tobytes()
        assert np.array_equal(eng.env_collide_motions(env, ha, tfa, links, tpl, off, witness=False)[0], fi)
        eng.env_destroy(env)
