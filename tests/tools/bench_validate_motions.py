#!/usr/bin/env python
"""bench_validate_motions.py -- progressive motion validation as a host loop over the existing device calls against
hfb_env_validate_motions, on workloads.robot_motions' chain (chain_robot_model, 16 links) in bench_robot_motions.py's
scene (100 000 environment objects, the template chain_self_pairs(16)), at 16 and 1 024 motions.  Per call, host clock
around a call that ends synchronised, warm-ups first, the forms alternated round by round; the median and the minimum
of the rounds are reported:

  host_loop  validate_reference (tests/validate_common.py) driving the device forms of the existing calls: per round
             the runs' joint values on the host, hfb_robot_poses_device, hfb_robot_sample_motions_device over 2-sample
             motions for the sweep bounds, hfb_env_certify_motions_device, and the flags downloaded for the bookkeeping
  device     hfb_env_validate_motions_device (the end points uploaded, the outputs downloaded)

The two forms' status, t_valid, t_collide and counts must be equal.  Also reported: the rounds and samples, and the
shares of motions that end valid, colliding and unresolved against hfb_env_certify_motions alone at the initial
sampling (2^d0 + 1 samples: a motion is certified whole there, collides, or is left uncertified).  Prints one JSON line
per size and one with the card's name and power limit, read in the same run.

  python tests/tools/bench_validate_motions.py [--motions 16,1024] [--room-scale 16] [--d0 4] [--depth 8] [--rounds 5]
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
from tests.validate_common import effective_cap, run_layout, validate_reference  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--motions", default="16,1024")
    ap.add_argument("--room-scale", type=float, default=16.0)
    ap.add_argument("--links", type=int, default=16)
    ap.add_argument("--env", type=int, default=100_000)
    ap.add_argument("--d0", type=int, default=4)
    ap.add_argument("--depth", type=int, default=8, help="D - d0")
    ap.add_argument("--max-samples", type=int, default=1 << 22)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()

    import torch
    import hppfcl_b200 as hf
    from hppfcl_b200 import _pod as P, workloads as W

    L, d0 = a.links, a.d0
    D = d0 + a.depth
    tpl = W.chain_self_pairs(L)
    room = W.robot_vs_environment(n_configs=1024, n_links=L, n_env=a.env)["room"] * a.room_scale
    eng = hf.Engine(0)
    req = P.CollisionRequestPOD()
    env = hs = robot = None
    s = torch.cuda.current_stream().cuda_stream
    for K in [int(x) for x in a.motions.split(",")]:
        w = W.robot_motions(K, n_links=L, n_env=a.env, room=room)
        if hs is None:  # (B does not depend on K: its draws come first)
            hs = w["register"](eng)
            eng.commit()
            tfb = w["tf_b"].copy()
            tfb[0] = W.identity_transforms(1, T=[[0.0, 0.0, -2.0]])[0]  # the floor below every base
            tfb["T"][(w["geom_b"] >= L + 64) & (w["geom_b"] < L + 80), 2] += 10.0  # the tables and shelves
            n_b = len(tfb)
            env = eng.env_create(hs[w["geom_b"]].astype(np.uint32), tfb)
        m = W.chain_robot_model(w)
        if robot is None:
            robot = eng.robot_create(m["parent"], m["types"], m["axis"], m["placement"], m["link_joint"],
                                     m["link_placement"], hs[m["geom"]].astype(np.uint32))
        q0, q1 = m["q_from"], m["q_to"]

        def narrow(depth, runs):
            qs, off, qa, qb = run_layout(runs, q0, q1, D)
            ns, na = len(qs), len(qs) * L
            d_t = torch.empty(na * 96, dtype=torch.uint8, device="cuda")
            d_h = torch.empty(na * 4, dtype=torch.uint8, device="cuda")
            # (the uploads are kept referenced until the calls that read them are done)
            d_qs, d_qa, d_qb = (torch.from_numpy(x).cuda() for x in (qs, qa, qb))
            eng.robot_poses_device(robot, ns, d_qs.data_ptr(), d_t.data_ptr(), d_h.data_ptr(), stream=s)
            nseg = len(qa)
            sw2 = torch.empty((2 * nseg, L), dtype=torch.float64, device="cuda")
            t2, h2 = torch.empty(2 * nseg * L * 96, dtype=torch.uint8, device="cuda"), torch.empty(
                2 * nseg * L * 4, dtype=torch.uint8, device="cuda")
            eng.robot_sample_motions_device(robot, np.arange(0, 2 * nseg + 1, 2, dtype=np.uint32),
                                            d_qa.data_ptr(), d_qb.data_ptr(),
                                            t2.data_ptr(), h2.data_ptr(), None, sw2.data_ptr(), stream=s)
            # each run's segments' sweeps, then 0 at its last sample
            seg_of = np.full(ns, -1, np.int64)
            k = 0
            for r in range(len(runs)):
                n_r = int(off[r + 1] - off[r]) - 1
                seg_of[off[r]:off[r] + n_r] = 2 * np.arange(k, k + n_r)
                k += n_r
            idx = torch.from_numpy(np.maximum(seg_of, 0)).cuda()
            sweep = sw2[idx] * torch.from_numpy(seg_of >= 0).cuda()[:, None]
            fin_seg = (sw2[::2] <= np.finfo(np.float64).max).all(dim=1)
            n_r = len(runs)
            fi = torch.empty(n_r, dtype=torch.int32, device="cuda")
            cert = torch.empty(ns, dtype=torch.uint8, device="cuda")
            cnt = torch.zeros(4, dtype=torch.int32, device="cuda")
            eng.env_certify_motions_device(env, na, d_h.data_ptr(), d_t.data_ptr(), sweep.contiguous().data_ptr(), L,
                                           tpl, off, fi.data_ptr(), None, cert.data_ptr(),
                                           tuple(cnt[j:].data_ptr() for j in range(4)), req=req, stream=s)
            fi, cert, cnt, fin_seg = fi.cpu().numpy(), cert.cpu().numpy(), cnt.cpu().numpy(), fin_seg.cpu().numpy()
            certs, fins, k = [], [], 0
            for r in range(n_r):
                n_s = int(off[r + 1] - off[r]) - 1
                certs.append(cert[off[r]:off[r] + n_s])
                fins.append(fin_seg[k:k + n_s])
                k += n_s
            return fi, certs, fins, (int(cnt[0]), int(cnt[1]), int(cnt[2]))

        def host_loop():
            return validate_reference(narrow, K, d0, D, effective_cap(a.max_samples, n_b, L))

        d_out = [torch.empty(K * b, dtype=torch.uint8, device="cuda") for b in (1, 8, 8)]
        d_cnt = [torch.empty(8, dtype=torch.uint8, device="cuda") for _ in range(5)]

        def device():
            d_q0, d_q1 = torch.from_numpy(q0).cuda(), torch.from_numpy(q1).cuda()
            eng.env_validate_motions_device(env, robot, K, d_q0.data_ptr(), d_q1.data_ptr(), tpl, d0, D, a.max_samples,
                                            *[x.data_ptr() for x in d_out], d_counts=[x.data_ptr() for x in d_cnt],
                                            req=req, stream=s)
            r = {f: x.cpu().numpy().view(t) for f, x, t in zip(("status", "t_valid", "t_collide"), d_out,
                                                                 (np.int8, np.float64, np.float64))}
            r["n_rounds"] = int(d_cnt[0].cpu().numpy().view(np.uint32)[0])
            for f, x in zip(("n_samples", "n_env_candidates", "n_self_candidates", "n_unsupported"), d_cnt[1:]):
                r[f] = int(x.cpu().numpy().view(np.uint64)[0])
            return r

        forms = {"host_loop": host_loop, "device": device}
        out = {}
        for _ in range(a.warmup):
            for f in forms.values():
                f()
        times = {k: [] for k in forms}
        for _ in range(a.rounds):
            for k, f in forms.items():
                torch.cuda.synchronize()
                t = time.perf_counter()
                out[k] = f()
                torch.cuda.synchronize()
                times[k].append((time.perf_counter() - t) * 1e3)
        h, d = out["host_loop"], out["device"]
        for f in ("status", "t_valid", "t_collide", "n_rounds", "n_samples", "n_env_candidates", "n_self_candidates",
                  "n_unsupported"):
            assert np.array_equal(np.asarray(h[f]), np.asarray(d[f])), "the forms differ in " + f
        # certify alone at the initial sampling
        n0 = 1 << d0
        off = np.arange(0, (n0 + 1) * K + 1, n0 + 1, dtype=np.uint32)
        tfa, ha, _, sw = eng.robot_sample_motions(robot, q0, q1, off)
        fi, fu, _, _ = eng.env_certify_motions(env, ha, tfa, sw, L, tpl, off, req)
        st = d["status"]
        line = {"motions": K, "room_scale": a.room_scale, "d0": d0, "D": D,
                "ms": {k: {"median": float(np.median(v)), "min": float(np.min(v))} for k, v in times.items()},
                "rounds": d["n_rounds"], "samples": d["n_samples"],
                "validate_share": {"valid": float((st == 0).mean()), "collides": float((st == 1).mean()),
                                   "unresolved": float((st == 2).mean())},
                "certify_share": {"valid": float(((fi < 0) & (fu < 0)).mean()), "collides": float((fi >= 0).mean()),
                                  "uncertified": float(((fi < 0) & (fu >= 0)).mean())}}
        print(json.dumps(line), flush=True)
    print(json.dumps({"gpu": gpu_info()}))


if __name__ == "__main__":
    main()
