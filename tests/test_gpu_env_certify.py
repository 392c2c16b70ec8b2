"""The motion certification on the device (hfb_env_certify_motions*): against the brute-force contract of
tests/test_env_certify_reference.py on the hand sample and on robot motions, first_invalid against
hfb_env_collide_motions, and soundness at scale: every certified segment of 1 024 robot motions, resampled 16 times by
forward kinematics and checked by hfb_env_collide_configs, has no colliding interior sample."""
import numpy as np
import pytest

from tests.common import P, hf, make_scenes
from tests.test_env_certify_reference import (check_against_reference, contract, load_recorded, margin_request,
                                               reference_sample)
from oracle import oracle_lib
from tests.test_gpu_env_configs import dev
from tests.test_gpu_env_motions import motion_scene
from hppfcl_b200 import workloads as W

pytestmark = pytest.mark.gpu

LINKS = 16
TPL = W.chain_self_pairs(LINKS)


def assert_same(got, want):
    for k in range(3):
        assert np.array_equal(got[k], want[k]), k
    assert tuple(got[3]) == tuple(want[3])


def test_hand_sample_matches_the_contract():
    """the hand sample, whose every candidate record the reference build agrees with (live, or its recorded outputs)"""
    oracle_lib.build_ref()
    load_recorded()
    sc = make_scenes(gpu=True, emu=True, ref=True)
    eng = sc.b["gpu"]
    out, used = reference_sample(sc)
    check_against_reference(sc, used)
    for scene, req, ans in out:
        ha, tfa, hb, tfb, links, tpl, off, sweep, _ = scene
        env = eng.env_create(hb, tfb)
        assert_same(eng.env_certify_motions(env, ha, tfa, sweep, links, tpl, off, req), ans[:4])
        eng.env_destroy(env)


def test_robot_motions_match_the_contract():
    sc = make_scenes(gpu=True, emu=True)
    eng, orc, emu = sc.b["gpu"], sc.b["oracle"], sc.b["emu"]
    w, ha, tfa, hb, tfb = motion_scene(sc, n_motions=64, seed=53, oracle=True)
    off = w["offsets"]
    n = len(off) - 1
    env = eng.env_create(hb, tfb)
    rng = np.random.default_rng(5)
    sweep = W.chain_sweep_bounds(w) + 2e-6
    odd = sweep.copy()
    pick = rng.random(len(odd))
    odd[pick < 0.01] = np.nan
    odd[(pick >= 0.01) & (pick < 0.02)] = -1.0
    odd[(pick >= 0.02) & (pick < 0.03)] = np.inf
    cases = [(sweep, None), (odd, None), (np.zeros_like(sweep), None), (sweep, margin_request(0.02)),
             (sweep * 3, None)]
    for sw, req in cases:
        want = contract(orc, emu, ha, tfa, hb, tfb, LINKS, TPL, off, sw, req=req)[:4]
        got = eng.env_certify_motions(env, ha, tfa, sw, LINKS, TPL, off, req)
        assert_same(got, want)
    # all sweeps 0: certified[g] iff g has a successor and, at g and g + 1, every collide candidate (box overlap) has
    # no contact, is supported and has a lower bound > 0 -- stated from the oracle's records directly
    bb = emu.scene_aabbs(ha, tfa)
    ef, es = hf.broadphase_cross_pairs(bb, emu.scene_aabbs(hb, tfb))
    sf, ss = hf.broadphase_config_pairs(bb, LINKS, TPL)
    ok = np.ones(len(ha) // LINKS, bool)
    for f, rec in ((ef, orc.batch_collide(ha[ef], tfa[ef], hb[es], tfb[es], nthreads=0)),
                   (sf, orc.batch_collide(ha[sf], tfa[sf], ha[ss], tfa[ss], nthreads=0))):
        bad = (rec["num_contacts"] > 0) | (P.status_path(rec["status"]) == P.PATH_UNSUPPORTED) | \
              ~(rec["distance_lower_bound"] > 0)
        ok[np.asarray(f[bad], dtype=np.int64) // LINKS] = False
    last = np.zeros(len(ok), bool)
    last[off[1:][np.diff(off) > 0] - 1] = True
    want0 = ok & ~last
    want0[:-1] &= ok[1:]
    z = eng.env_certify_motions(env, ha, tfa, np.zeros_like(sweep), LINKS, TPL, off)[2]
    assert np.array_equal(z, want0.astype(np.uint8)) and z.any() and not z.all()
    # sub-ranges equal the full call's values; the rest -1 / 0
    full = eng.env_certify_motions(env, ha, tfa, sweep, LINKS, TPL, off)
    assert full[2].any() and (full[1] >= 0).any() and (full[0] >= 0).any() and (full[0] < 0).any()
    for m0, nm in ((0, 20), (20, 1), (21, 0), (21, n - 21)):
        r = eng.env_certify_motions(env, ha, tfa, sweep, LINKS, TPL, off, first_motion=m0, num_motions=nm)
        assert_same(r, contract(orc, emu, ha, tfa, hb, tfb, LINKS, TPL, off, sweep, m0=m0, nm=nm)[:4])
        g0, g1 = int(off[m0]), int(off[m0 + nm])
        assert np.array_equal(r[0][m0:m0 + nm], full[0][m0:m0 + nm])
        assert np.array_equal(r[1][m0:m0 + nm], full[1][m0:m0 + nm])
        assert np.array_equal(r[2][g0:g1], full[2][g0:g1])
        assert not r[2][:g0].any() and not r[2][g1:].any()
    # -inf margin: every motion valid, every segment with valid sweeps certified
    req = P.CollisionRequestPOD()
    req.security_margin = -np.inf
    r = eng.env_certify_motions(env, ha, tfa, odd, LINKS, TPL, off, req)
    assert_same(r, contract(orc, emu, ha, tfa, hb, tfb, LINKS, TPL, off, odd, req=req)[:4])
    assert (r[0] == -1).all() and r[3][2] == 0
    # an empty template, and an env without objects
    empty = np.zeros((0, 2), dtype=np.uint32)
    assert_same(eng.env_certify_motions(env, ha, tfa, sweep, LINKS, empty, off),
                contract(orc, emu, ha, tfa, hb, tfb, LINKS, empty, off, sweep)[:4])
    eng.env_destroy(env)
    env = eng.env_create(hb[:0], tfb[:0])
    assert_same(eng.env_certify_motions(env, ha, tfa, sweep, LINKS, TPL, off),
                contract(orc, emu, ha, tfa, hb[:0], tfb[:0], LINKS, TPL, off, sweep)[:4])
    r = eng.env_certify_motions(env, ha, tfa, sweep, LINKS, empty, off)
    assert (r[0] == -1).all() and r[3][:3] == (0, 0, 0)
    eng.env_destroy(env)


def test_soundness_at_scale_and_first_invalid():
    """1 024 motions: first_invalid equals hfb_env_collide_motions', and no certified segment has a colliding interior
    sample among 16 per segment"""
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = motion_scene(eng)
    off = w["offsets"]
    env = eng.env_create(hb, tfb)
    sweep = W.chain_sweep_bounds(w) + 2e-6
    fi, fu, cert, counts = eng.env_certify_motions(env, ha, tfa, sweep, LINKS, TPL, off)
    assert np.array_equal(fi, eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off, witness=False)[0])
    segs = np.flatnonzero(cert)
    n_seg = int(len(ha) // LINKS - (len(off) - 1))
    assert len(segs) > 1000 and counts[3] == n_seg - len(segs) and counts[3] > 0
    fine = W.resample_motions(w, segs, 16)
    hfine = np.tile(ha[:LINKS], len(fine) // LINKS)
    v = eng.env_collide_configs(env, hfine, fine, LINKS, TPL, None, 0, 0)[0]
    assert len(v) == 16 * len(segs) and not v.any()
    # the coarse samples of certified segments are valid too
    g = np.concatenate([segs, segs + 1])
    assert not eng.env_collide_configs(env, ha, tfa, LINKS, TPL, None, 0, 0)[0][g].any()
    # non-finite and huge poses: those segments are not certified, the call does not fail
    bad = tfa.copy()
    bad["T"][5 * LINKS + 3] = np.nan
    bad["T"][9 * LINKS + 1] = 1e300
    r = eng.env_certify_motions(env, ha, bad, sweep, LINKS, TPL, off)
    assert np.array_equal(r[0], eng.env_collide_motions(env, ha, bad, LINKS, TPL, off, witness=False)[0])
    # a NaN pose bounds nothing: both segments of its sample fail; the segments of samples with finite poses are as
    # before (configuration 9's far link is a pair with nothing)
    assert r[2][5] == 0 and r[2][4] == 0
    same = np.ones(len(cert), bool)
    same[[4, 5, 8, 9]] = False
    assert np.array_equal(r[2][same], cert[same])
    eng.env_destroy(env)


def test_update_uncertifies_a_segment():
    """an environment object moved between the two samples of a certified segment, next to a link but touching
    neither sample: the segment is no longer certified, and the oracle's lower bound of that pair explains it"""
    sc = make_scenes(gpu=True, emu=False)
    eng, orc = sc.b["gpu"], sc.b["oracle"]
    w, ha, tfa, hb, tfb = motion_scene(sc, n_motions=128, seed=47, oracle=True)
    tfb = tfb.copy()
    env = eng.env_create(hb, tfb)
    off = w["offsets"]
    sweep = W.chain_sweep_bounds(w) + 2e-6
    before = eng.env_certify_motions(env, ha, tfa, sweep, LINKS, TPL, off)
    k = next(i for i in range(20, len(hb) - 1) if LINKS <= w["geom_b"][i] < LINKS + 64)  # a small object of B
    # the certified segment whose link 15 sweeps farthest
    segs = np.flatnonzero(before[2])
    g = int(segs[np.argmax(sweep[segs * LINKS + 15])])
    a, b = tfa["T"][g * LINKS + 15], tfa["T"][(g + 1) * LINKS + 15]
    t = tfb[[k]].copy()
    t["T"] = 0.5 * (a + b)  # (half way between the link's two centres)
    eng.env_update(env, [k], t)
    after = eng.env_certify_motions(env, ha, tfa, sweep, LINKS, TPL, off)
    assert after[2][g] == 0
    assert np.array_equal(after[0], eng.env_collide_motions(env, ha, tfa, LINKS, TPL, off, witness=False)[0])
    # the oracle: at one end of the segment the moved object's pair with link 15 has 2 * lower bound <= the sweep, or
    # a contact
    ends = np.array([g * LINKS + 15, (g + 1) * LINKS + 15])
    ro = orc.batch_collide(ha[ends], tfa[ends], np.repeat(hb[k], 2), np.repeat(t, 2), nthreads=0)
    assert ((ro["num_contacts"] > 0) | ~(2 * ro["distance_lower_bound"] > sweep[g * LINKS + 15])).any()
    eng.env_destroy(env)


def test_device_form_and_refusals():
    import torch
    eng = hf.Engine(0)
    w, ha, tfa, hb, tfb = motion_scene(eng, n_motions=40, seed=41)
    off = w["offsets"]
    n, n_cfg = len(off) - 1, len(ha) // LINKS
    env = eng.env_create(hb, tfb)
    sweep = W.chain_sweep_bounds(w) + 2e-6
    want = eng.env_certify_motions(env, ha, tfa, sweep, LINKS, TPL, off)
    d_h, d_t, d_s = dev(ha), dev(tfa), dev(sweep)

    def run(tpl=TPL, offs=off, m0=0, nm=None):
        fi = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        fu = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        cert = torch.full((n_cfg,), 7, dtype=torch.uint8, device="cuda")
        cnt = torch.full((4,), 7, dtype=torch.int32, device="cuda")
        err = None
        try:
            eng.env_certify_motions_device(env, len(ha), d_h.data_ptr(), d_t.data_ptr(), d_s.data_ptr(), LINKS, tpl,
                                           offs, fi.data_ptr(), fu.data_ptr(), cert.data_ptr(),
                                           tuple(cnt[k:].data_ptr() for k in range(4)), first_motion=m0,
                                           num_motions=nm)
        except hf.EngineError as e:
            err = e
        torch.cuda.synchronize()
        return (fi.cpu().numpy(), fu.cpu().numpy(), cert.cpu().numpy(), tuple(cnt.cpu().numpy().tolist())), err

    got, err = run()
    assert err is None
    assert_same(got, want)
    r, err = run(m0=10, nm=5)
    assert err is None
    assert_same(r, eng.env_certify_motions(env, ha, tfa, sweep, LINKS, TPL, off, first_motion=10, num_motions=5))
    for kw in (dict(tpl=[(0, 2), (2, 0)]), dict(offs=np.concatenate([[1], off[1:]])), dict(m0=n, nm=1)):
        r, err = run(**kw)
        assert err is not None and "invalid argument" in str(err)
        assert (r[0] == 7).all() and (r[1] == 7).all() and (r[2] == 7).all() and r[3] == (7, 7, 7, 7)
    eng.env_destroy(env)
