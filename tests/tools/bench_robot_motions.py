#!/usr/bin/env python
"""bench_robot_motions.py -- continuous motion validation with the poses sampled on the host against sampled on the
device, on workloads.robot_motions' chain (16 links; chain_robot_model: 18 joints, two prismatic ones carrying the base)
in bench_certify_motions.py's scene at room scale 16 (100 000 environment objects, the template chain_self_pairs(16)),
at 16 and 1 024 motions.  Per call, host clock around a call that ends synchronised, warm-ups first, the forms
alternated round by round; the median and the minimum of the rounds are reported:

  host     numpy forward kinematics of every sample (robot_motions' own chain), chain_sweep_bounds, then
           hfb_env_certify_motions (host form: poses, handles and sweep bounds uploaded by the call)
  device   each motion's end points uploaded (torch), hfb_robot_sample_motions_device (poses, handles, sweep bounds),
           then hfb_env_certify_motions_device on the same stream
  sample_call    hfb_robot_sample_motions_device alone (host checks, the offsets' upload, the launch), CUDA events
                 around `--launches` back-to-back calls
  sample_kernel  k_robot alone: the library's kernel timing (hfb_set_profiling: CUDA events recorded on the stream
                 right before and after the launch), over the same calls

Also reported: the bytes each form sends to the device per call, and the share of segments certified under each
form's sweep bounds (chain_sweep_bounds, derived by hand for this chain, and the library's bound for any tree).
first_invalid must agree between the forms.  Prints one JSON line per size and one with the card's name and power
limit, read in the same run.

  python tests/tools/bench_robot_motions.py [--motions 16,1024] [--room-scale 16] [--rounds 10] [--warmup 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.tools.bench_env import gpu_info  # noqa: E402


def chain_fk(q, L, ll, P, W):
    """robot_motions' forward kinematics from the chain model's q ([x, y, q_0 .. q_{L-1}] per sample) -> transforms"""
    n = len(q)
    R = np.broadcast_to(np.eye(3), (n, 3, 3))
    p = np.zeros((n, 3))
    p[:, :2] = q[:, :2]
    Rs, Ts = np.empty((n, L, 3, 3)), np.empty((n, L, 3))
    for k in range(L):
        R = R @ W._axis_rotations(2 if k % 2 == 0 else 1, q[:, 2 + k])
        axis = R[:, :, 2]
        Rs[:, k] = R
        Ts[:, k] = p + 0.5 * ll * axis
        p = p + ll * axis
    return P.make_transforms(Rs.reshape(-1, 3, 3), Ts.reshape(-1, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--motions", default="16,1024")
    ap.add_argument("--room-scale", type=float, default=16.0)
    ap.add_argument("--links", type=int, default=16)
    ap.add_argument("--env", type=int, default=100_000)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--launches", type=int, default=50)
    a = ap.parse_args()

    import torch
    import hppfcl_b200 as hf
    from hppfcl_b200 import _pod as P, workloads as W

    L = a.links
    tpl = W.chain_self_pairs(L)
    room = W.robot_vs_environment(n_configs=1024, n_links=L, n_env=a.env)["room"] * a.room_scale
    eng = hf.Engine(0)
    req = P.CollisionRequestPOD()
    env = hs = robot = None
    for K in [int(x) for x in a.motions.split(",")]:
        w = W.robot_motions(K, n_links=L, n_env=a.env, room=room)
        if hs is None:  # (B does not depend on K: its draws come first)
            hs = w["register"](eng)
            eng.commit()
            tfb = w["tf_b"].copy()
            tfb[0] = W.identity_transforms(1, T=[[0.0, 0.0, -2.0]])[0]  # the floor below every base
            tfb["T"][(w["geom_b"] >= L + 64) & (w["geom_b"] < L + 80), 2] += 10.0  # the tables and shelves
            env = eng.env_create(hs[w["geom_b"]].astype(np.uint32), tfb)
        m = W.chain_robot_model(w)
        if robot is None:
            robot = eng.robot_create(m["parent"], m["types"], m["axis"], m["placement"], m["link_joint"],
                                     m["link_placement"], hs[m["geom"]].astype(np.uint32))
        J = len(m["parent"])
        off = w["offsets"]
        n_cfg, n = int(off[-1]), len(off) - 1
        n_a = n_cfg * L
        ha_link = hs[m["geom"]].astype(np.uint32)
        # the host form's samples: robot_motions' own, linear in q (as the library samples them, up to rounding)
        q_host = m["q"]
        qf_np, qt_np = m["q_from"], m["q_to"]
        s = torch.cuda.current_stream().cuda_stream
        d_t = torch.empty(n_a * 96, dtype=torch.uint8, device="cuda")
        d_h = torch.empty(n_a * 4, dtype=torch.uint8, device="cuda")
        d_s = torch.empty(n_a * 8, dtype=torch.uint8, device="cuda")
        fi = torch.empty(n, dtype=torch.int32, device="cuda")
        fu = torch.empty(n, dtype=torch.int32, device="cuda")
        cert = torch.empty(n_cfg, dtype=torch.uint8, device="cuda")
        cnt = torch.empty(4, dtype=torch.int32, device="cuda")

        def host():
            tfa = chain_fk(q_host, L, w["link_len"], P, W)
            sweep = W.chain_sweep_bounds(w)
            return eng.env_certify_motions(env, np.tile(ha_link, n_cfg), tfa, sweep, L, tpl, off, req)

        def sample(qf, qt):
            eng.robot_sample_motions_device(robot, off, qf.data_ptr(), qt.data_ptr(), d_t.data_ptr(), d_h.data_ptr(),
                                            None, d_s.data_ptr(), stream=s)

        def device():
            qf = torch.from_numpy(qf_np).cuda(non_blocking=False)
            qt = torch.from_numpy(qt_np).cuda(non_blocking=False)
            sample(qf, qt)
            eng.env_certify_motions_device(env, n_a, d_h.data_ptr(), d_t.data_ptr(), d_s.data_ptr(), L, tpl, off,
                                           fi.data_ptr(), fu.data_ptr(), cert.data_ptr(),
                                           tuple(cnt[k:].data_ptr() for k in range(4)), req=req, stream=s)
            torch.cuda.synchronize()
            return fi.cpu().numpy(), fu.cpu().numpy(), cert.cpu().numpy(), tuple(int(c) for c in cnt.cpu().numpy())

        forms = {"host": host, "device": device}
        res = {}
        for name, fn in forms.items():
            for _ in range(a.warmup):
                res[name] = fn()
        assert np.array_equal(res["host"][0], res["device"][0]), "first_invalid differs between the forms"
        times = {k: [] for k in forms}
        for _ in range(a.rounds):
            for name, fn in forms.items():
                t0 = time.perf_counter()
                fn()
                times[name].append(time.perf_counter() - t0)
        # the sampling kernel alone
        qf, qt = torch.from_numpy(qf_np).cuda(), torch.from_numpy(qt_np).cuda()
        for _ in range(a.warmup):
            sample(qf, qt)
        ct, kt = [], []
        for _ in range(a.rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.launches):
                sample(qf, qt)
            e1.record()
            torch.cuda.synchronize()
            ct.append(e0.elapsed_time(e1) / a.launches)
            eng.set_profiling(True)
            eng.kernel_times(reset=True)
            for _ in range(a.launches):
                sample(qf, qt)
            torch.cuda.synchronize()
            t = eng.kernel_times(reset=True)
            eng.set_profiling(False)
            assert t["other_launches"] == a.launches, t
            kt.append(t["other_ms"] / a.launches)
        n_s = np.diff(off).astype(np.int64)
        segs = int((n_s - 1).clip(0).sum())
        hand_unc, lib_unc = res["host"][3][3], res["device"][3][3]
        line = {"motions": K, "samples": n_cfg, "links": L, "joints": J, "template_pairs": len(tpl), "b_objects": a.env,
                "room": room,
                "bytes_up": {"host": n_a * (96 + 4 + 8), "device": 2 * n * J * 8 + 4 * (n + 1)},
                "segments": segs, "share_certified": {"host_hand_sweep": (segs - hand_unc) / max(segs, 1),
                                                      "device_library_sweep": (segs - lib_unc) / max(segs, 1)},
                "share_motions_valid": float((res["host"][0] < 0).mean()),
                "ms_per_call_median": {k: 1e3 * float(np.median(t)) for k, t in times.items()},
                "ms_per_call_min": {k: 1e3 * float(np.min(t)) for k, t in times.items()},
                "sample_call_ms_median": float(np.median(ct)), "sample_call_ms_min": float(np.min(ct)),
                "sample_kernel_ms_median": float(np.median(kt)), "sample_kernel_ms_min": float(np.min(kt)),
                "rounds": a.rounds}
        print(json.dumps(line), flush=True)
    eng.robot_destroy(robot)
    eng.env_destroy(env)
    print(json.dumps({"gpu": gpu_info()}))


if __name__ == "__main__":
    main()
