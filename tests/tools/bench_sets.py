#!/usr/bin/env python
"""bench_sets.py -- robot against environment: set A (K configurations x L links) collided with set B (a static
environment of about 10^5 objects), workloads.robot_vs_environment at about 10^6 candidate pairs.  Prints one JSON line:

  value            candidate pairs/s with the poses resident on the device: boxes + cross pair finder
                   (hfb_broadphase_cross_pairs_device) + collide() of the candidates over the object table [A; B]
  split_ms         the same step cut by CUDA events: boxes + pair finder / narrow phase
  e2e              candidate pairs/s through hfb_scene_collide_sets with pinned host buffers (poses in, colliding pairs
                   and their records out)
  cpu_baseline     the host cross finder on one thread + the reference build's collide() (the oracle where the
                   reference build is absent) on a sample of the candidates, all cores, as bench.py's config 5 arm
  gpu              the card's name and power limit, read in the same run

  python tests/tools/bench_sets.py [--configs 1024] [--env 100000] [--steps 20] [--warmup 3]
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
    ap.add_argument("--configs", type=int, default=1024)
    ap.add_argument("--links", type=int, default=16)
    ap.add_argument("--env", type=int, default=100_000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-sample", type=int, default=100_000)
    a = ap.parse_args()

    import torch
    import hppfcl_b200 as hf
    from hppfcl_b200 import _pod as P, workloads as W
    from oracle import oracle_lib

    w = W.robot_vs_environment(n_configs=a.configs, n_links=a.links, n_env=a.env)
    eng = hf.Engine(0)
    hs = w["register"](eng)
    eng.commit()
    ha, hb = hs[w["geom_a"]].astype(np.uint32), hs[w["geom_b"]].astype(np.uint32)
    tfa, tfb = w["tf_a"], w["tf_b"]
    na, nb = len(ha), len(hb)
    req = P.CollisionRequestPOD()

    def dev(x):
        return torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1)).cuda()

    # the object table [A; B] on the device; boxes of both sets in one array
    d_h, d_tf = dev(np.concatenate([ha, hb])), dev(np.concatenate([tfa, tfb]))
    d_bb = torch.empty((na + nb) * 6, dtype=torch.float64, device="cuda")
    cap = 4_000_000
    d_f = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_s = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int32, device="cuda")
    d_out = torch.empty(cap * P.contact_dtype.itemsize, dtype=torch.uint8, device="cuda")
    h_n = torch.zeros(1, dtype=torch.int32).pin_memory()
    stream = torch.cuda.current_stream().cuda_stream
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    acc = {"bp": 0.0, "np": 0.0}

    def step(timed=False):
        if timed:
            ev[0].record()
        eng.scene_aabbs_device(na + nb, d_h.data_ptr(), d_tf.data_ptr(), d_bb.data_ptr(), stream)
        eng.broadphase_cross_pairs_device(na, d_bb.data_ptr(), nb, d_bb.data_ptr() + 48 * na, d_f.data_ptr(), d_s.data_ptr(),
                                          cap, d_n.data_ptr(), stream)
        h_n.copy_(d_n, non_blocking=True)
        if timed:
            ev[1].record()
        torch.cuda.current_stream().synchronize()  # the narrow phase is launched for the number of candidates found
        k = int(h_n.item())
        assert k <= cap, "candidate buffer too small"
        d_s[:k] += na  # index in B -> index in the table [A; B]
        eng.batch_collide_objects_device(na + nb, d_h.data_ptr(), d_tf.data_ptr(), k, d_f.data_ptr(), d_s.data_ptr(),
                                         d_out.data_ptr(), req, stream=stream)
        if timed:
            ev[2].record()
            torch.cuda.synchronize()
            acc["bp"] += ev[0].elapsed_time(ev[1])
            acc["np"] += ev[1].elapsed_time(ev[2])
        return k

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    pairs = 0
    e0.record()
    for _ in range(a.steps):
        pairs += step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    n_split = 3
    for _ in range(n_split):
        step(timed=True)
    # e2e: hfb_scene_collide_sets with pinned host buffers
    pin = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1)).pin_memory().numpy()  # noqa: E731
    pha, ptfa = pin(ha).view(np.uint32), pin(tfa).view(P.transform_dtype)
    phb, ptfb = pin(hb).view(np.uint32), pin(tfb).view(P.transform_dtype)
    ccap = 2_000_000
    bufs = tuple(torch.empty(ccap * it, dtype=torch.uint8).pin_memory().numpy().view(dt) for it, dt in
                 ((4, np.uint32), (4, np.uint32), (P.contact_dtype.itemsize, P.contact_dtype)))
    for _ in range(2):
        eng.scene_collide_sets(pha, ptfa, phb, ptfb, req, capacity=ccap, bufs=bufs)
    e2e_steps = max(3, min(a.steps, 10))
    cand = hits = 0
    t0 = time.perf_counter()
    for _ in range(e2e_steps):
        _, _, _, c, h = eng.scene_collide_sets(pha, ptfa, phb, ptfb, req, capacity=ccap, bufs=bufs)
        cand += c
        hits += h
    dt = time.perf_counter() - t0
    gpu = gpu_info()
    del eng

    # CPU arm: host cross finder on one thread + the reference's collide() on a sample of the candidates
    emu_boxes = None
    from tests.common import EmuScene
    emu = EmuScene()
    he = w["register"](emu)
    emu_boxes = (emu.scene_aabbs(he[w["geom_a"]], tfa), emu.scene_aabbs(he[w["geom_b"]], tfb))
    t0 = time.perf_counter()
    f, s = hf.broadphase_cross_pairs(*emu_boxes)
    t_bp = time.perf_counter() - t0
    ref = oracle_lib.ref_available()
    orc = oracle_lib.RefScene(P) if ref else oracle_lib.OracleScene(P)
    ho = w["register"](orc, oracle=True)
    m = min(a.cpu_sample, len(f))
    sel = np.random.default_rng(1).choice(len(f), m, replace=False)
    oa, ob = ho[w["geom_a"]][f[sel]].astype(np.uint32), ho[w["geom_b"]][s[sel]].astype(np.uint32)
    t0 = time.perf_counter()
    orc.batch_collide(oa, tfa[f[sel]], ob, tfb[s[sel]], req, nthreads=0)
    t_np = time.perf_counter() - t0
    rate_np = m / t_np
    cpu_total = t_bp + len(f) / rate_np

    per_step = pairs / a.steps
    line = {"workload": "robot_vs_environment: %d configurations x %d links against %d environment objects, about %d "
                        "candidate pairs per step" % (a.configs, a.links, a.env, per_step),
            "unit": "candidate pairs/s", "value": pairs / (ms * 1e-3), "ms_per_step": ms / a.steps,
            "candidate_pairs_per_step": per_step,
            "split_ms_per_step": {"boxes_cross_pair_finder": acc["bp"] / n_split, "narrow_phase": acc["np"] / n_split},
            "e2e": {"value": cand / dt, "unit": "candidate pairs/s", "api": "hfb_scene_collide_sets (pinned host buffers)",
                    "steps": e2e_steps, "colliding_pairs_per_step": hits / e2e_steps,
                    "h2d_bytes_per_step": int((na + nb) * 100)},
            "cpu_baseline": {"value": len(f) / cpu_total, "unit": "candidate pairs/s", "broadphase_ms": 1e3 * t_bp,
                             "narrow_phase_only_value": rate_np,
                             "kind": "reference build" if ref else "oracle (reference build absent)",
                             "sample": "host cross finder on 1 thread (%d candidates) + collide() of %d of them, all cores"
                                       % (len(f), m)},
            "gpu": gpu}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
