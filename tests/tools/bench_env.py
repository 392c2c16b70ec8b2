#!/usr/bin/env python
"""bench_env.py -- the resident environment (hfb_env_*) against the one-shot two-set call (hfb_scene_collide_sets) on
workloads.robot_vs_environment: 100 000 environment objects, 16 links, at 1, 16 and 1 024 configurations (one
environment for all three: the room of the 1 024-configuration workload).  Per call, host clock around a call that
ends synchronised, warm-ups first, the forms alternated round by round; the median of the rounds is reported:

  sets           hfb_scene_collide_sets, pinned host buffers (A and B up, colliding pairs and records down)
  env_pairs      hfb_env_collide, pairs mode (A up, colliding pairs and records down)
  env_flags      hfb_env_collide, flags only (A up, one byte per A object down)
  sets_device    the device-side form bench_sets.py times: boxes of [A; B], hfb_broadphase_cross_pairs_device, the
                 count to the host, collide() of the candidates (hfb_batch_collide_objects_device)
  env_device     hfb_env_collide_device, pairs and flags into device buffers
  env_update     hfb_env_update with 1 % of B moved (poses up, boxes and the grid redone)

Prints one JSON line per size and one with the card's name and power limit, read in the same run.

  python tests/tools/bench_env.py [--configs 1,16,1024] [--env 100000] [--rounds 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [x.strip() for x in q[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


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
    room = W.robot_vs_environment(n_configs=1024, n_links=a.links, n_env=a.env)["room"]
    eng = hf.Engine(0)
    req = P.CollisionRequestPOD()
    stream = torch.cuda.current_stream().cuda_stream
    pin = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1)).pin_memory().numpy()  # noqa: E731
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1)).cuda()  # noqa: E731
    ccap = 2_000_000
    bufs = tuple(torch.empty(ccap * it, dtype=torch.uint8).pin_memory().numpy().view(dt) for it, dt in
                 ((4, np.uint32), (4, np.uint32), (P.contact_dtype.itemsize, P.contact_dtype)))
    dcap = 4_000_000
    d_f = torch.empty(dcap, dtype=torch.int32, device="cuda")
    d_s = torch.empty(dcap, dtype=torch.int32, device="cuda")
    d_out = torch.empty(dcap * P.contact_dtype.itemsize, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(2, dtype=torch.int32, device="cuda")
    h_n = torch.zeros(1, dtype=torch.int32).pin_memory()
    hs = None
    rng = np.random.default_rng(3)
    for K in sizes:
        w = W.robot_vs_environment(n_configs=K, n_links=a.links, n_env=a.env, room=room)
        if hs is None:
            hs = w["register"](eng)
            eng.commit()
        ha, hb = pin(hs[w["geom_a"]].astype(np.uint32)).view(np.uint32), pin(hs[w["geom_b"]].astype(np.uint32)).view(np.uint32)
        tfa, tfb = pin(w["tf_a"]).view(P.transform_dtype), pin(w["tf_b"]).view(P.transform_dtype)
        na, nb = len(ha), len(hb)
        env = eng.env_create(hb, tfb)
        d_ha, d_tfa = dev(ha), dev(tfa)
        d_h, d_tf = dev(np.concatenate([ha, hb])), dev(np.concatenate([tfa, tfb]))
        d_bb = torch.empty((na + nb) * 6, dtype=torch.float64, device="cuda")
        d_fl = torch.empty(na, dtype=torch.uint8, device="cuda")
        moved = np.sort(rng.choice(np.arange(1, nb), nb // 100, replace=False)).astype(np.uint32)
        moved_tf = pin(tfb[moved]).view(P.transform_dtype)

        def sets():
            return eng.scene_collide_sets(ha, tfa, hb, tfb, req, capacity=ccap, bufs=bufs)[3:5]

        def env_pairs():
            return eng.env_collide(env, ha, tfa, req, capacity=ccap, bufs=bufs)[3:5]

        def env_flags():
            r = eng.env_collide(env, ha, tfa, req, capacity=0, flags=True)
            return r[3], r[4]

        def sets_device():
            eng.scene_aabbs_device(na + nb, d_h.data_ptr(), d_tf.data_ptr(), d_bb.data_ptr(), stream)
            eng.broadphase_cross_pairs_device(na, d_bb.data_ptr(), nb, d_bb.data_ptr() + 48 * na, d_f.data_ptr(),
                                              d_s.data_ptr(), dcap, d_n.data_ptr(), stream)
            h_n.copy_(d_n[:1], non_blocking=True)
            torch.cuda.current_stream().synchronize()
            k = int(h_n.item())
            d_s[:k] += na
            eng.batch_collide_objects_device(na + nb, d_h.data_ptr(), d_tf.data_ptr(), k, d_f.data_ptr(), d_s.data_ptr(),
                                             d_out.data_ptr(), req, stream=stream)
            torch.cuda.current_stream().synchronize()
            return k, None

        def env_device():
            eng.env_collide_device(env, na, d_ha.data_ptr(), d_tfa.data_ptr(), d_f.data_ptr(), d_s.data_ptr(),
                                   d_out.data_ptr(), dcap, d_n.data_ptr(), d_n.data_ptr() + 4, d_fl.data_ptr(), req, stream)
            torch.cuda.current_stream().synchronize()
            return int(d_n[1].item()), int(d_n[0].item())

        def env_update():
            eng.env_update(env, moved, moved_tf)
            return None, None

        forms = {"sets": sets, "env_pairs": env_pairs, "env_flags": env_flags, "sets_device": sets_device,
                 "env_device": env_device, "env_update": env_update}
        counts = {}
        for name, fn in forms.items():
            for _ in range(a.warmup):
                counts[name] = fn()
        assert counts["sets"] == counts["env_pairs"] == counts["env_flags"] == counts["env_device"], counts
        assert counts["sets_device"][0] == counts["sets"][0]
        times = {k: [] for k in forms}
        for _ in range(a.rounds):
            for name, fn in forms.items():
                t0 = time.perf_counter()
                fn()
                times[name].append(time.perf_counter() - t0)
        eng.env_destroy(env)
        line = {"configs": K, "links": a.links, "a_objects": na, "b_objects": nb,
                "candidate_pairs": counts["sets"][0], "colliding_pairs": counts["sets"][1],
                "ms_per_call_median": {k: 1e3 * float(np.median(v)) for k, v in times.items()},
                "ms_per_call_min": {k: 1e3 * float(np.min(v)) for k, v in times.items()},
                "rounds": a.rounds, "env_update_objects": int(len(moved))}
        print(json.dumps(line), flush=True)
    print(json.dumps({"gpu": gpu_info()}))


if __name__ == "__main__":
    main()
