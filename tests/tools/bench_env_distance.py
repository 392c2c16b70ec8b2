#!/usr/bin/env python
"""bench_env_distance.py -- each robot object's nearest environment object (hfb_env_distance_device) against the
composition of existing calls on the device, on workloads.robot_vs_environment: bench_env.py's room of 100 000
environment objects, 16 links, at 1, 16 and 1 024 configurations, max_distance in {0, 0.05, 0.3, inf}.  Per call: the
device time between CUDA events around the call (warm-ups first, the forms alternated round by round, the median
reported), the number of rounds of growing radius that ran candidates (k_dist_boxes launches in one profiled call, less
the last one, which only finds every object settled) and the candidates per robot object.

  env_distance  hfb_env_distance_device: nearest, min_distance and records into device buffers
  composition   A's boxes (hfb_scene_aabbs_device) inflated by max_distance in torch (rounded outward), then
                hfb_broadphase_cross_pairs_device against B's boxes, hfb_batch_distance_objects_device over [A; B]
                and a torch argmin per A object (smallest eligible distance, lowest B index on ties); finite cutoffs
                only (at inf every pair is a candidate)

nearest and min_distance of both forms must be equal.  Prints one JSON line per size and cutoff and one with the card's
name and power limit, read in the same run.

  python tests/tools/bench_env_distance.py [--configs 1,16,1024] [--env 100000] [--rounds 20] [--warmup 3]
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
            d_hb, d_tfb = dev(hb), dev(tfb)
            d_bbb = torch.empty(nb * 6, dtype=torch.float64, device="cuda")
            eng.scene_aabbs_device(nb, d_hb.data_ptr(), d_tfb.data_ptr(), d_bbb.data_ptr(), stream)
        ha, tfa = hs[w["geom_a"]].astype(np.uint32), w["tf_a"]
        na = len(ha)
        d_ha, d_tfa = dev(ha), dev(tfa)
        d_table_h, d_table_t = dev(np.concatenate([ha, hb])), dev(np.concatenate([tfa, tfb]))
        d_near = torch.empty(na, dtype=torch.int32, device="cuda")
        d_min = torch.empty(na, dtype=torch.float64, device="cuda")
        d_rec = torch.empty(na * rec_size, dtype=torch.uint8, device="cuda")
        d_cnt = torch.zeros(2, dtype=torch.int32, device="cuda")
        d_bba = torch.empty(na * 6, dtype=torch.float64, device="cuda")
        d_np = torch.zeros(1, dtype=torch.int32, device="cuda")
        comp_cap = [1 << 20]
        bufs = {}

        def grow(cap):
            bufs["f"] = torch.empty(cap, dtype=torch.int32, device="cuda")
            bufs["s"] = torch.empty(cap, dtype=torch.int32, device="cuda")
            bufs["r"] = torch.empty(cap * rec_size, dtype=torch.uint8, device="cuda")

        grow(comp_cap[0])
        for maxd in cutoffs:
            def env_distance():
                eng.env_distance_device(env, na, d_ha.data_ptr(), d_tfa.data_ptr(), d_near.data_ptr(), d_min.data_ptr(),
                                        d_rec.data_ptr(), d_cnt.data_ptr(), d_cnt.data_ptr() + 4, req, maxd, stream)

            def composition():
                eng.scene_aabbs_device(na, d_ha.data_ptr(), d_tfa.data_ptr(), d_bba.data_ptr(), stream)
                bq = d_bba.view(na, 6)
                inf = torch.tensor(np.inf, dtype=torch.float64, device="cuda")
                lo = torch.nextafter(bq[:, :3] - maxd, -inf)
                hi = torch.nextafter(bq[:, 3:] + maxd, inf)
                bq = torch.cat([lo, hi], 1).contiguous()
                while True:
                    eng.broadphase_cross_pairs_device(na, bq.data_ptr(), nb, d_bbb.data_ptr(), bufs["f"].data_ptr(),
                                                      bufs["s"].data_ptr(), comp_cap[0], d_np.data_ptr(), stream=stream)
                    n = int(d_np.item())
                    if n <= comp_cap[0]:
                        break
                    comp_cap[0] = n + n // 8
                    grow(comp_cap[0])
                f, s = bufs["f"][:n], (bufs["s"][:n] + na).contiguous()
                if n:
                    eng.batch_distance_objects_device(na + nb, d_table_h.data_ptr(), d_table_t.data_ptr(), n, f.data_ptr(),
                                                      s.data_ptr(), bufs["r"].data_ptr(), req, stream)
                r = bufs["r"][:n * rec_size].view(n, rec_size)
                d = r[:, :8].contiguous().view(torch.float64).reshape(-1)
                status = r[:, 88:92].contiguous().view(torch.int32).reshape(-1)
                elig = (d <= maxd) & (((status >> 16) & 0xff) != P.PATH_UNSUPPORTED)
                fi = f.long()
                best = torch.full((na,), np.inf, dtype=torch.float64, device="cuda")
                best.scatter_reduce_(0, fi[elig], d[elig], "amin")
                won = elig & (d == best[fi])
                j = torch.full((na,), 1 << 31, dtype=torch.int64, device="cuda")
                j.scatter_reduce_(0, fi[won], (s[won] - na).long(), "amin")
                near = torch.where(j == 1 << 31, torch.full_like(j, -1), j).to(torch.int32)
                dist = torch.full((na,), P.DBL_MAX, dtype=torch.float64, device="cuda")
                dist[fi[won]] = d[won]
                return near, dist, n

            forms = {"env_distance": env_distance}
            if np.isfinite(maxd):
                forms["composition"] = composition
            res = {}
            for name, fn in forms.items():
                for _ in range(a.warmup):
                    res[name] = fn()
            torch.cuda.synchronize()
            cand = int(d_cnt[0].item())
            if "composition" in res:
                near, dist, _ = res["composition"]
                assert torch.equal(near, d_near), "nearest differs from the composition's"
                assert torch.equal(dist, d_min), "min_distance differs from the composition's"
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                env_distance()
                torch.cuda.synchronize()
            # (the last k_dist_boxes launch only finds every object settled: it runs no candidates)
            rounds = sum(e.count for e in prof.key_averages() if "k_dist_boxes" in e.key) - 1
            times = {k: [] for k in forms}
            for _ in range(a.rounds):
                for name, fn in forms.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(cs)
                    fn()
                    e1.record(cs)
                    e1.synchronize()
                    times[name].append(e0.elapsed_time(e1))
            near = d_near.cpu().numpy()
            line = {"configs": K, "links": L, "a_objects": na, "b_objects": nb, "max_distance": maxd, "rounds": rounds,
                    "candidates": cand, "candidates_per_link": cand / na, "found": int((near >= 0).sum()),
                    "ms_per_call_median": {k: float(np.median(t)) for k, t in times.items()},
                    "ms_per_call_min": {k: float(np.min(t)) for k, t in times.items()}, "timed_rounds": a.rounds}
            print(json.dumps(line), flush=True)
    eng.env_destroy(env)
    print(json.dumps({"gpu": gpu_info()}))


if __name__ == "__main__":
    main()
