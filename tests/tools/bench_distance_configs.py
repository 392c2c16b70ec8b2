#!/usr/bin/env python
"""bench_distance_configs.py -- each configuration's clearance, its nearest environment or self pair
(hfb_env_distance_configs_device), against the composition of existing calls on the device, on
workloads.robot_vs_environment: bench_env.py's room of 100 000 environment objects, 16 links and the chain template
(chain_self_pairs(16), 105 pairs), at 1, 16 and 1 024 configurations, max_distance in {0, 0.05, 0.3, inf}.  Per call: the
device time between CUDA events around the call (warm-ups first, the forms alternated round by round, the median
reported) and the self candidates per configuration.

  configs      hfb_env_distance_configs_device: kind, first, second, min_distance and records into device buffers
  composition  hfb_env_distance_device over all links, hfb_batch_distance_objects_device over the template expanded
               over every configuration (every pair: that path has no box cutoff), then a torch argmin per
               configuration (smallest eligible distance; environment pairs by link before self pairs by template entry)

kind, first, second and min_distance of both forms must be equal.  Prints one JSON line per size and cutoff and one
with the card's name and power limit, read in the same run.

  python tests/tools/bench_distance_configs.py [--configs 1,16,1024] [--env 100000] [--rounds 20] [--warmup 3]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.tools.bench_env import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="1,16,1024")
    ap.add_argument("--links", type=int, default=16)
    ap.add_argument("--env", type=int, default=100_000)
    ap.add_argument("--cutoffs", default="0,0.05,0.3,inf")
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()

    import torch
    import hppfcl_b200 as hf
    from hppfcl_b200 import _pod as P, workloads as W

    sizes = [int(x) for x in a.configs.split(",")]
    cutoffs = [float(x) for x in a.cutoffs.split(",")]
    L = a.links
    tpl = W.chain_self_pairs(L)
    npairs = len(tpl)
    room = W.robot_vs_environment(n_configs=1024, n_links=L, n_env=a.env)["room"]
    eng = hf.Engine(0)
    req = P.DistanceRequestPOD()
    cs = torch.cuda.current_stream()
    stream = cs.cuda_stream
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1)).cuda()  # noqa: E731
    rec_size = P.distance_result_dtype.itemsize
    hs = env = None
    for K in sizes:
        w = W.robot_vs_environment(n_configs=K, n_links=L, n_env=a.env, room=room)
        if hs is None:  # (B does not depend on K: its draws come first)
            hs = w["register"](eng)
            eng.commit()
            hb, tfb = hs[w["geom_b"]].astype(np.uint32), w["tf_b"]
            env = eng.env_create(hb, tfb)
            nb = len(hb)
        ha, tfa = hs[w["geom_a"]].astype(np.uint32), w["tf_a"]
        na = len(ha)
        d_ha, d_tfa = dev(ha), dev(tfa)
        out = {"kind": torch.empty(K, dtype=torch.int8, device="cuda"),
               "first": torch.empty(K, dtype=torch.int32, device="cuda"),
               "second": torch.empty(K, dtype=torch.int32, device="cuda"),
               "min": torch.empty(K, dtype=torch.float64, device="cuda"),
               "rec": torch.empty(K * rec_size, dtype=torch.uint8, device="cuda")}
        d_cnt = torch.zeros(3, dtype=torch.int32, device="cuda")
        # the composition's buffers: per-link results, the expanded template and its records
        d_near = torch.empty(na, dtype=torch.int32, device="cuda")
        d_lmin = torch.empty(na, dtype=torch.float64, device="cuda")
        d_lrec = torch.empty(na * rec_size, dtype=torch.uint8, device="cuda")
        g = torch.arange(K, device="cuda", dtype=torch.int64).repeat_interleave(npairs)
        t_pairs = torch.from_numpy(tpl.astype(np.int64)).cuda().repeat(K, 1)
        sf = (g * L + t_pairs[:, 0]).to(torch.int32).contiguous()
        ss = (g * L + t_pairs[:, 1]).to(torch.int32).contiguous()
        ns = K * npairs
        d_srec = torch.empty(ns * rec_size, dtype=torch.uint8, device="cuda")
        ordinal = torch.cat([torch.arange(na, device="cuda") % L,
                             L + torch.arange(npairs, device="cuda").repeat(K)])
        cfg = torch.cat([torch.arange(na, device="cuda") // L, g])

        for maxd in cutoffs:
            def configs():
                eng.env_distance_configs_device(env, na, d_ha.data_ptr(), d_tfa.data_ptr(), L, tpl, out["kind"].data_ptr(),
                                                out["first"].data_ptr(), out["second"].data_ptr(), out["min"].data_ptr(),
                                                out["rec"].data_ptr(), d_cnt.data_ptr(), d_cnt.data_ptr() + 4,
                                                d_cnt.data_ptr() + 8, req, maxd, stream)

            def composition():
                eng.env_distance_device(env, na, d_ha.data_ptr(), d_tfa.data_ptr(), d_near.data_ptr(), d_lmin.data_ptr(),
                                        d_lrec.data_ptr(), None, None, req, maxd, stream)
                eng.batch_distance_objects_device(na, d_ha.data_ptr(), d_tfa.data_ptr(), ns, sf.data_ptr(), ss.data_ptr(),
                                                  d_srec.data_ptr(), req, stream)
                r = d_srec.view(ns, rec_size)
                sd = r[:, :8].contiguous().view(torch.float64).reshape(-1)
                status = r[:, 88:92].contiguous().view(torch.int32).reshape(-1)
                selig = (sd <= maxd) & (((status >> 16) & 0xff) != P.PATH_UNSUPPORTED)
                d = torch.cat([d_lmin, sd])
                elig = torch.cat([d_near >= 0, selig])
                best = torch.full((K,), np.inf, dtype=torch.float64, device="cuda")
                best.scatter_reduce_(0, cfg[elig], d[elig], "amin")
                at = elig & (d == best[cfg])
                word = torch.full((K,), 1 << 40, dtype=torch.int64, device="cuda")
                word.scatter_reduce_(0, cfg[at], ordinal[at], "amin")
                won = at & (ordinal == word[cfg])
                kind = torch.full((K,), -1, dtype=torch.int8, device="cuda")
                first = torch.full((K,), -1, dtype=torch.int32, device="cuda")
                second = torch.full((K,), -1, dtype=torch.int32, device="cuda")
                dist = torch.full((K,), P.DBL_MAX, dtype=torch.float64, device="cuda")
                idx = torch.nonzero(won).reshape(-1)
                gw = cfg[idx]
                is_self = idx >= na
                kind[gw] = is_self.to(torch.int8)
                li = torch.clamp(idx, max=na - 1)
                si = torch.clamp(idx - na, min=0)
                first[gw] = torch.where(is_self, sf[si], li.to(torch.int32))
                second[gw] = torch.where(is_self, ss[si], d_near[li])
                dist[gw] = d[idx]
                return kind, first, second, dist

            forms = {"configs": configs, "composition": composition}
            res = {}
            for name, fn in forms.items():
                for _ in range(a.warmup):
                    res[name] = fn()
            torch.cuda.synchronize()
            kind, first, second, dist = res["composition"]
            assert torch.equal(kind, out["kind"]), "kind differs from the composition's"
            assert torch.equal(first, out["first"]) and torch.equal(second, out["second"]), "winners differ"
            assert torch.equal(dist, out["min"]), "min_distance differs from the composition's"
            cnt = d_cnt.cpu().numpy()
            times = {k: [] for k in forms}
            for _ in range(a.rounds):
                for name, fn in forms.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(cs)
                    fn()
                    e1.record(cs)
                    e1.synchronize()
                    times[name].append(e0.elapsed_time(e1))
            k = out["kind"].cpu().numpy()
            line = {"configs": K, "links": L, "self_pairs": npairs, "b_objects": nb, "max_distance": maxd,
                    "env_candidates": int(cnt[0]), "self_candidates": int(cnt[1]),
                    "self_candidates_per_config": int(cnt[1]) / K,
                    "winners": {"env": int((k == 0).sum()), "self": int((k == 1).sum()), "none": int((k < 0).sum())},
                    "ms_per_call_median": {n: float(np.median(t)) for n, t in times.items()},
                    "ms_per_call_min": {n: float(np.min(t)) for n, t in times.items()}, "timed_rounds": a.rounds}
            print(json.dumps(line), flush=True)
    eng.env_destroy(env)
    print(json.dumps({"gpu": gpu_info()}))


if __name__ == "__main__":
    main()
