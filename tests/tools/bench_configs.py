#!/usr/bin/env python
"""bench_configs.py -- a planner's validity check: robot configurations against the resident environment AND against
themselves (hfb_env_collide_configs*), against today's composition of existing calls, on workloads.robot_vs_environment
with the bending joints in +-2.8 rad (so that some configurations fold onto themselves): bench_env.py's room of 100 000
environment objects, 16 links, at 1, 16 and 1 024 configurations, the self-pair template chain_self_pairs(16) (105
pairs).  Per call, host clock around a call that ends synchronised, warm-ups first, the forms alternated round by round;
the median of the rounds is reported:

  configs_verdicts  hfb_env_collide_configs, verdicts only (A up, one byte per configuration down)
  configs_pairs     hfb_env_collide_configs with verdicts and both kinds of pairs (records down)
  configs_device    hfb_env_collide_configs_device, verdicts and pairs into device buffers
  composition       hfb_env_collide flags-only, then hfb_batch_collide_objects (compact) over all K x 105 template
                    pairs (expanded on the host once, outside the timing), then the OR per configuration on the host

The verdicts of configs_verdicts and composition must be equal.  Prints one JSON line per size and one with the card's
name and power limit, read in the same run.

  python tests/tools/bench_configs.py [--configs 1,16,1024] [--env 100000] [--rounds 20] [--warmup 3]
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
    ap.add_argument("--configs", default="1,16,1024")
    ap.add_argument("--links", type=int, default=16)
    ap.add_argument("--env", type=int, default=100_000)
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()

    import torch
    import hppfcl_b200 as hf
    from hppfcl_b200 import _pod as P, workloads as W

    sizes = [int(x) for x in a.configs.split(",")]
    L = a.links
    tpl = W.chain_self_pairs(L)
    room = W.robot_vs_environment(n_configs=1024, n_links=L, n_env=a.env)["room"]
    eng = hf.Engine(0)
    req = P.CollisionRequestPOD()
    stream = torch.cuda.current_stream().cuda_stream
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1)).cuda()  # noqa: E731
    dcap = 2_000_000
    d_kinds = [(torch.empty(dcap, dtype=torch.int32, device="cuda"), torch.empty(dcap, dtype=torch.int32, device="cuda"),
                torch.empty(dcap * P.contact_dtype.itemsize, dtype=torch.uint8, device="cuda")) for _ in range(2)]
    d_n = torch.zeros(4, dtype=torch.int32, device="cuda")
    hs = env = None
    for K in sizes:
        w = W.robot_vs_environment(n_configs=K, n_links=L, n_env=a.env, room=room, joint_range=2.8)
        if hs is None:  # (B does not depend on K: its draws come first)
            hs = w["register"](eng)
            eng.commit()
            env = eng.env_create(hs[w["geom_b"]].astype(np.uint32), w["tf_b"])
        ha, tfa = hs[w["geom_a"]].astype(np.uint32), w["tf_a"]
        na = len(ha)
        d_ha, d_tfa = dev(ha), dev(tfa)
        d_v = torch.empty(K, dtype=torch.uint8, device="cuda")
        g = np.repeat(np.arange(K, dtype=np.uint32) * L, len(tpl))
        pf, ps = g + np.tile(tpl[:, 0], K), g + np.tile(tpl[:, 1], K)
        outs = [(f.data_ptr(), s.data_ptr(), r.data_ptr(), dcap, d_n.data_ptr() + 8 * k, d_n.data_ptr() + 8 * k + 4)
                for k, (f, s, r) in enumerate(d_kinds)]

        def configs_verdicts():
            return eng.env_collide_configs(env, ha, tfa, L, tpl, req, 0, 0)[0]

        _, e0, s0 = eng.env_collide_configs(env, ha, tfa, L, tpl, req, 0, 0)
        caps = (max(e0[4], 1), max(s0[4], 1))  # room for every colliding pair

        def configs_pairs():
            v, e, s = eng.env_collide_configs(env, ha, tfa, L, tpl, req, *caps)
            return v, e[3:], s[3:]

        def configs_device():
            eng.env_collide_configs_device(env, na, d_ha.data_ptr(), d_tfa.data_ptr(), L, tpl, d_v.data_ptr(), *outs, req,
                                           stream)
            torch.cuda.current_stream().synchronize()
            return None

        def composition():
            flags = eng.env_collide(env, ha, tfa, req, capacity=0, flags=True)[5]
            _, _, ids, _ = eng.batch_collide_objects(ha, tfa, pf, ps, req, compact_capacity=len(pf))
            v = flags.reshape(K, L).max(axis=1)
            v[pf[ids] // L] = 1
            return v

        forms = {"configs_verdicts": configs_verdicts, "configs_pairs": configs_pairs, "configs_device": configs_device,
                 "composition": composition}
        res = {}
        for name, fn in forms.items():
            for _ in range(a.warmup):
                res[name] = fn()
        assert np.array_equal(res["configs_verdicts"], res["composition"]), "verdicts differ from the composition's"
        assert np.array_equal(res["configs_pairs"][0], res["composition"])
        assert np.array_equal(d_v.cpu().numpy(), res["composition"])
        times = {k: [] for k in forms}
        for _ in range(a.rounds):
            for name, fn in forms.items():
                t0 = time.perf_counter()
                fn()
                times[name].append(time.perf_counter() - t0)
        v, e, s = res["configs_pairs"]
        line = {"configs": K, "links": L, "template_pairs": len(tpl), "a_objects": na, "b_objects": a.env,
                "colliding_configs": int(v.sum()), "env_candidates": e[0], "env_colliding": e[1], "self_candidates": s[0],
                "self_colliding": s[1],
                "ms_per_call_median": {k: 1e3 * float(np.median(t)) for k, t in times.items()},
                "ms_per_call_min": {k: 1e3 * float(np.min(t)) for k, t in times.items()}, "rounds": a.rounds}
        print(json.dumps(line), flush=True)
    eng.env_destroy(env)
    print(json.dumps({"gpu": gpu_info()}))


if __name__ == "__main__":
    main()
