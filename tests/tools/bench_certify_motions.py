#!/usr/bin/env python
"""bench_certify_motions.py -- a planner's continuous motion validation (hfb_env_certify_motions) against discrete
validation (hfb_env_collide_motions) on the same samples and at 4x the sampling density, on workloads.robot_motions
with chain_sweep_bounds: 100 000 environment objects, 16 links, the self-pair template chain_self_pairs(16) (105
pairs), at 16 and 1 024 motions.  bench_motions.py's room is so dense that every motion collides; here the room is
`--room-scale` times as wide in x and y (the objects spread over room-scale^2 the floor area), so that a share of the
motions is valid, and, as in test_gpu_env_configs' scene, the floor (B's object 0), which every base stands on, is lowered and
the large boxes (tables and shelves, 1 % of B) are lifted out of reach; the small objects and the meshes stay.  Per call, host clock around a call that ends synchronised, warm-ups first, the forms alternated
round by round; the median and the minimum of the rounds are reported:

  certify           hfb_env_certify_motions (host form): first_invalid, first_uncertified, certified
  collide           hfb_env_collide_motions on the same samples, first_invalid only
  collide_4x        hfb_env_collide_motions on the same motions sampled 4 times as densely, first_invalid only

certify's first_invalid must equal collide's.  Also reported: the candidate counts of each call, the share of segments
certified, and the shares of motions that are valid and that are certified whole (every segment, two samples or more).
Prints one JSON line per (room, size) and one with the card's name and power limit, read in the same run.

  python tests/tools/bench_certify_motions.py [--motions 16,1024] [--room-scale 4,16,32] [--rounds 10] [--warmup 3]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--motions", default="16,1024")
    ap.add_argument("--room-scale", default="4,16,32")
    ap.add_argument("--links", type=int, default=16)
    ap.add_argument("--env", type=int, default=100_000)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()

    import hppfcl_b200 as hf
    from hppfcl_b200 import _pod as P, workloads as W

    L = a.links
    tpl = W.chain_self_pairs(L)
    base_room = W.robot_vs_environment(n_configs=1024, n_links=L, n_env=a.env)["room"]
    eng = hf.Engine(0)
    req = P.CollisionRequestPOD()
    for scale in [float(x) for x in a.room_scale.split(",")]:
        room = base_room * scale
        env = hs = None
        for K in [int(x) for x in a.motions.split(",")]:
            w = W.robot_motions(K, n_links=L, n_env=a.env, room=room)
            w4 = W.robot_motions(K, n_links=L, n_env=a.env, room=room, resolution=0.025 / 4)  # (the same motions)
            if hs is None:  # (B does not depend on K: its draws come first)
                hs = w["register"](eng)
                eng.commit()
                tfb = w["tf_b"].copy()
                tfb[0] = W.identity_transforms(1, T=[[0.0, 0.0, -2.0]])[0]  # the floor below every base (see above)
                tfb["T"][(w["geom_b"] >= L + 64) & (w["geom_b"] < L + 80), 2] += 10.0  # the tables and shelves
                env = eng.env_create(hs[w["geom_b"]].astype(np.uint32), tfb)
            ha, tfa, off = hs[w["geom_a"]].astype(np.uint32), w["tf_a"], w["offsets"]
            ha4, tfa4, off4 = hs[w4["geom_a"]].astype(np.uint32), w4["tf_a"], w4["offsets"]
            sweep = W.chain_sweep_bounds(w)

            forms = {"certify": lambda: eng.env_certify_motions(env, ha, tfa, sweep, L, tpl, off, req),
                     "collide": lambda: eng.env_collide_motions(env, ha, tfa, L, tpl, off, req, witness=False),
                     "collide_4x": lambda: eng.env_collide_motions(env, ha4, tfa4, L, tpl, off4, req, witness=False)}
            res = {}
            for name, fn in forms.items():
                for _ in range(a.warmup):
                    res[name] = fn()
            fi, fu, cert, cnt = res["certify"]
            assert np.array_equal(fi, res["collide"][0]), "certify: first_invalid differs from collide_motions'"
            times = {k: [] for k in forms}
            for _ in range(a.rounds):
                for name, fn in forms.items():
                    t0 = time.perf_counter()
                    fn()
                    times[name].append(time.perf_counter() - t0)
            n_s = np.diff(off).astype(np.int64)
            segs = int((n_s - 1).clip(0).sum())
            whole = (fu < 0) & (n_s >= 2)
            c1, c4 = res["collide"][5], res["collide_4x"][5]
            line = {"room_scale": scale, "room": room, "motions": K, "samples": int(off[-1]),
                    "samples_4x": int(off4[-1]), "links": L, "template_pairs": len(tpl), "b_objects": a.env,
                    "candidates": {"certify_env": cnt[0], "certify_self": cnt[1], "collide_env": c1[0],
                                   "collide_self": c1[2], "collide_4x_env": c4[0], "collide_4x_self": c4[2]},
                    "unsupported": cnt[2], "segments": segs, "segments_certified": segs - cnt[3],
                    "share_segments_certified": (segs - cnt[3]) / max(segs, 1),
                    "share_motions_valid": float((fi < 0).mean()),
                    "share_motions_valid_4x": float((res["collide_4x"][0] < 0).mean()),
                    "share_motions_certified": float(whole.mean()),
                    "ms_per_call_median": {k: 1e3 * float(np.median(t)) for k, t in times.items()},
                    "ms_per_call_min": {k: 1e3 * float(np.min(t)) for k, t in times.items()}, "rounds": a.rounds}
            print(json.dumps(line), flush=True)
        eng.env_destroy(env)
    print(json.dumps({"gpu": gpu_info()}))


if __name__ == "__main__":
    main()
