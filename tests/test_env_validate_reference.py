"""The progressive motion validation's answers on the CPU, under the contract of hfb_env_validate_motions
(include/hppfcl_b200.h): validate_reference (tests/validate_common.py) drives the rounds through the brute-force
certification of tests/test_env_certify_reference.py -- the oracle's collide(), boxes and kinematics from the host
builds.  A hand-made scene of spheres makes each rule decide something.  tests/test_gpu_env_validate.py checks the
device against the same reference."""
import numpy as np
import pytest

from tests.common import P, make_scenes
from tests.robot_common import local_boxes
from tests.validate_common import cpu_narrow, hand_scene, q_at, validate_reference


def hand_reference(d0=1, D=6, cap=1 << 20, margin=0.0, first_motion=0, num_motions=None):
    sc = make_scenes(emu=True)
    model, hb, tfb, q0, q1, names = hand_scene(sc)
    sc.commit()
    orc, emu = sc.b["oracle"], sc.b["emu"]
    boxes = local_boxes(emu, model["handles"])
    req = P.CollisionRequestPOD()
    req.security_margin = margin
    narrow = cpu_narrow(orc, emu, model, boxes, hb, tfb, [(0, 1)], q0, q1, D, req)
    return validate_reference(narrow, len(q0), d0, D, cap, first_motion, num_motions), names


def test_each_rule_decides_a_motion():
    r, names = hand_reference()
    st = dict(zip(names, r["status"]))
    tv = dict(zip(names, r["t_valid"]))
    tc = dict(zip(names, r["t_collide"]))
    assert st["free"] == 0 and st["free2"] == 0 and st["still"] == 0  # certified, q_from == q_to included
    assert st["near"] == 0 and tv["near"] == 1.0                        # certified only after splits
    assert st["hit"] == 1 and tc["hit"] == 0.125 and 0 < tv["hit"] < 0.125  # touching at x = 0.5: position 8 of 64
    assert st["late"] == 1 and tv["late"] < tc["late"] <= 1.0
    assert st["graze"] == 2 and 0 < tv["graze"] < 1 / 3.0 and tc["graze"] == -1  # stuck at D before 1/3
    assert st["nan"] == 2 and tv["nan"] == 0.0                           # stuck at once: its sweeps are NaN
    assert r["n_rounds"] == 6  # d0 = 1 .. D = 6


def test_rounds_split_only_what_is_not_certified():
    full, names = hand_reference(d0=1, D=6)
    # D = d0: one certification of 2^d0 + 1 samples per motion
    one, _ = hand_reference(d0=3, D=3)
    assert one["n_rounds"] == 1 and one["n_samples"] == len(names) * 9
    # a deeper D never shortens the certified prefix when the cap does not bind
    deeper, _ = hand_reference(d0=1, D=7)
    assert (deeper["t_valid"] >= full["t_valid"]).all()
    assert (deeper["status"][full["status"] == 1] == 1).all()


def test_the_cap_cuts_a_motion_and_starves_the_later_ones():
    r, names = hand_reference(d0=2, D=4, cap=7)  # motion 0: 5 samples, motion 1: 2 of its 4 segments
    assert r["status"][0] == 0
    assert r["status"][1] == 2 and r["t_valid"][1] <= 0.5
    assert (r["status"][2:] == 2).all() and (r["t_valid"][2:] == 0).all() and (r["t_collide"][2:] == -1).all()


def test_minus_inf_margin_certifies_every_finite_motion():
    r, names = hand_reference(margin=-np.inf)
    st = dict(zip(names, r["status"]))
    assert all(st[n] == (2 if n == "nan" else 0) for n in names)
    assert r["n_rounds"] == 1  # (no collide() runs: every segment with finite sweeps closes in round 0)


def test_range_outside_gets_the_no_motion_values():
    r, names = hand_reference(first_motion=2, num_motions=3)
    assert (r["status"][:2] == -1).all() and (r["status"][5:] == -1).all()
    assert (r["t_valid"][:2] == 0).all() and (r["t_collide"][5:] == -1).all()
    assert r["status"][2] == 1


def test_q_at_is_the_sampling_formula():
    a, b = np.array([0.3, -1.0]), np.array([2.0, 5.5])
    assert np.array_equal(q_at(a, b, 0, 4), a) and np.array_equal(q_at(a, b, 16, 4), b)
    # depth-d positions are the samples of 2^d + 1 evenly spaced ones: t = k / 2^d exactly
    for k in range(1, 8):
        assert np.array_equal(q_at(a, b, 2 * k, 4), a + (k / 8.0) * (b - a))


M64 = (1 << 64) - 1


def _mix(x):  # splitmix64's finaliser, as tests/emu/validate_emu.cpp has it
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def _outcome(seed, kind, m, a, d, per_mille):
    return _mix(_mix(_mix(_mix(seed ^ kind) ^ m) ^ a) ^ (d if kind else 0)) % 1000 < per_mille


def _emu():
    import ctypes as C
    import os
    import subprocess
    from tests.common import EMU_DIR, ROOT
    so = os.path.join(EMU_DIR, "libvalidate_emu.so")
    src = os.path.join(EMU_DIR, "validate_emu.cpp")
    deps = [src, os.path.join(ROOT, "hpp-fcl_b200", "csrc", "hfb_validate.cuh"),
            os.path.join(ROOT, "hpp-fcl_b200", "csrc", "hfb_math.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", so,
                               src])
    L = C.CDLL(so)
    u32, vp = C.c_uint32, C.c_void_p
    L.val_emu.argtypes = [C.c_uint64, u32, u32, u32, u32, u32, u32, vp, vp, vp, vp, vp, vp]
    return L


def test_host_build_of_the_bookkeeping_matches_the_reference():
    """the device's bookkeeping (hfb_validate.cuh, driven as the k_val_* kernels drive it) against validate_reference on
    thousands of random round outcomes: caps that bind in round 0 and in later rounds, runs broken by certified and
    dropped segments, collisions at every depth, non-finite sweeps"""
    L = _emu()
    rng = np.random.default_rng(2024)
    for case in range(2000):
        seed = int(rng.integers(0, 1 << 62))
        n = int(rng.integers(1, 12))
        m0 = int(rng.integers(0, n))
        nm = int(rng.integers(0, n - m0 + 1))
        d0 = int(rng.integers(0, 4))
        D = d0 + int(rng.integers(0, 5))
        cap = int(rng.choice([2, 3, 5, 9, 17, 40, 100, 1 << 20]))
        pm = np.array([rng.integers(0, 80), rng.integers(100, 900), rng.integers(0, 60)], dtype=np.uint32)

        def narrow(depth, runs):
            fi, cert, fin = [], [], []
            for m, pos in runs:
                hit = [s for s, k in enumerate(pos) if _outcome(seed, 0, m, k, 0, pm[0])]
                fi.append(hit[0] if hit else -1)
                cert.append([_outcome(seed, 1, m, k, depth, pm[1]) for k in pos[:-1]])
                fin.append([not _outcome(seed, 2, m, k, depth, pm[2]) for k in pos[:-1]])
            return fi, cert, fin, (0, 0, 0)

        want = validate_reference(narrow, n, d0, D, cap, m0, nm)
        st, tv, tc = np.empty(n, np.int8), np.empty(n), np.empty(n)
        rounds, samples = np.zeros(1, np.uint32), np.zeros(1, np.uint64)
        assert L.val_emu(seed, n, m0, nm, d0, D, cap, pm.ctypes.data, st.ctypes.data, tv.ctypes.data, tc.ctypes.data,
                         rounds.ctypes.data, samples.ctypes.data) == 0
        got = dict(status=st, t_valid=tv, t_collide=tc, n_rounds=int(rounds[0]), n_samples=int(samples[0]))
        for f in got:
            assert np.array_equal(np.asarray(got[f]), np.asarray(want[f])), (case, f, got[f], want[f])
