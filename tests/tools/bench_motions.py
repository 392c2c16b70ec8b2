#!/usr/bin/env python
"""bench_motions.py -- a planner's motion validation: per motion, the first sample that collides with the resident
environment or with itself and the pair that collides there (hfb_env_collide_motions*), against today's composition of
hfb_env_collide_configs and a host reduction, on workloads.robot_motions with the bending joints in +-2.8 rad:
bench_env.py's room of 100 000 environment objects, 16 links, at 16 and 1 024 motions (about 25 samples each), the
self-pair template chain_self_pairs(16) (105 pairs).  Per call, host clock around a call that ends synchronised,
warm-ups first, the forms alternated round by round; the median and the minimum of the rounds are reported:

  motions_first         hfb_env_collide_motions, first_invalid only (no witness sought, no records down)
  motions_witness       hfb_env_collide_motions with kind, indices and records
  motions_device        hfb_env_collide_motions_device, everything into device buffers
  composition_verdicts  hfb_env_collide_configs verdicts only, then the first colliding sample per motion on the host
                        (first_invalid only)
  composition_pairs     hfb_env_collide_configs with every colliding pair (records down), then the witness per motion
                        on the host by the contract's order

The forms must agree: first_invalid of all five, and kind, indices and records of motions_witness, motions_device and
composition_pairs.  Prints one JSON line per size and one with the card's name and power limit, read in the same run.

  python tests/tools/bench_motions.py [--motions 16,1024] [--env 100000] [--rounds 20] [--warmup 3]
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


def host_witness(off, L, n_b, tpl, e, s):
    """the contract's reduction on the host, vectorised: -> (first_invalid, kind, first, second, records index into
    the concatenated pair records)"""
    n = len(off) - 1
    entry = np.full((L, L), -1, dtype=np.int64)
    entry[tpl[:, 0], tpl[:, 1]] = np.arange(len(tpl))
    f = np.concatenate([e[0], s[0]]).astype(np.int64)
    sec = np.concatenate([e[1], s[1]]).astype(np.int64)
    kind = np.concatenate([np.zeros(len(e[0]), np.int8), np.ones(len(s[0]), np.int8)])
    ordv = np.concatenate([(e[0].astype(np.int64) % L) * n_b + e[1], L * n_b + entry[s[0] % L, s[1] % L]])
    g = f // L
    motion = np.searchsorted(off, g, side="right") - 1
    sample = g - off[motion].astype(np.int64)
    order = np.lexsort((ordv, sample, motion))
    ms, at = np.unique(motion[order], return_index=True)
    win = order[at]
    fi = np.full(n, -1, np.int32)
    kd = np.full(n, -1, np.int8)
    first = np.full(n, 0xFFFFFFFF, np.uint32)
    second = np.full(n, 0xFFFFFFFF, np.uint32)
    fi[ms], kd[ms], first[ms], second[ms] = sample[win], kind[win], f[win], sec[win]
    return fi, kd, first, second, ms, win


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--motions", default="16,1024")
    ap.add_argument("--links", type=int, default=16)
    ap.add_argument("--env", type=int, default=100_000)
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()

    import torch
    import hppfcl_b200 as hf
    from hppfcl_b200 import _pod as P, workloads as W

    sizes = [int(x) for x in a.motions.split(",")]
    L = a.links
    tpl = W.chain_self_pairs(L)
    room = W.robot_vs_environment(n_configs=1024, n_links=L, n_env=a.env)["room"]
    eng = hf.Engine(0)
    req = P.CollisionRequestPOD()
    stream = torch.cuda.current_stream().cuda_stream
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1)).cuda()  # noqa: E731
    hs = env = None
    for K in sizes:
        w = W.robot_motions(K, n_links=L, n_env=a.env, room=room, joint_range=2.8)
        if hs is None:  # (B does not depend on K: its draws come first)
            hs = w["register"](eng)
            eng.commit()
            env = eng.env_create(hs[w["geom_b"]].astype(np.uint32), w["tf_b"])
        ha, tfa, off = hs[w["geom_a"]].astype(np.uint32), w["tf_a"], w["offsets"]
        na, n_b = len(ha), a.env
        d_ha, d_tfa = dev(ha), dev(tfa)
        d_fi = torch.empty(K, dtype=torch.int32, device="cuda")
        d_kind = torch.empty(K, dtype=torch.int8, device="cuda")
        d_f = torch.empty(K, dtype=torch.int32, device="cuda")
        d_s = torch.empty(K, dtype=torch.int32, device="cuda")
        d_rec = torch.empty(K * P.contact_dtype.itemsize, dtype=torch.uint8, device="cuda")
        d_n = torch.zeros(4, dtype=torch.int32, device="cuda")

        def motions_first():
            return eng.env_collide_motions(env, ha, tfa, L, tpl, off, req, witness=False)[0]

        def motions_witness():
            return eng.env_collide_motions(env, ha, tfa, L, tpl, off, req)

        def motions_device():
            c = d_n.data_ptr()
            eng.env_collide_motions_device(env, na, d_ha.data_ptr(), d_tfa.data_ptr(), L, tpl, off, d_fi.data_ptr(),
                                           d_kind.data_ptr(), d_f.data_ptr(), d_s.data_ptr(), d_rec.data_ptr(),
                                           (c, c + 4, c + 8, c + 12), req, stream)
            torch.cuda.current_stream().synchronize()
            return None

        def composition_verdicts():
            v = eng.env_collide_configs(env, ha, tfa, L, tpl, req, 0, 0)[0]
            hit = np.flatnonzero(v)
            m = np.searchsorted(off, hit, side="right") - 1
            fi = np.full(K, -1, np.int32)
            ms, at = np.unique(m, return_index=True)
            fi[ms] = hit[at] - off[ms]
            return fi

        _, e0, s0 = eng.env_collide_configs(env, ha, tfa, L, tpl, req, 0, 0)
        caps = (max(e0[4], 1), max(s0[4], 1))  # room for every colliding pair

        def composition_pairs():
            _, e, s = eng.env_collide_configs(env, ha, tfa, L, tpl, req, *caps)
            fi, kd, first, second, ms, win = host_witness(off, L, n_b, tpl, e, s)
            rec = np.full(K, eng_cleared, dtype=P.contact_dtype)
            rec[ms] = np.concatenate([e[2], s[2]])[win]
            return fi, kd, first, second, rec

        # the record of a motion without a witness (every motion of an empty range gets it)
        eng_cleared = eng.env_collide_motions(env, ha, tfa, L, tpl, off, req, num_motions=0)[4][0]

        forms = {"motions_first": motions_first, "motions_witness": motions_witness, "motions_device": motions_device,
                 "composition_verdicts": composition_verdicts, "composition_pairs": composition_pairs}
        res = {}
        for name, fn in forms.items():
            for _ in range(a.warmup):
                res[name] = fn()
        wit, cp = res["motions_witness"], res["composition_pairs"]
        for name in ("motions_first", "composition_verdicts"):
            assert np.array_equal(res[name], wit[0]), name + ": first_invalid differs"
        for k in range(4):
            assert np.array_equal(cp[k], wit[k]), "composition_pairs differs from motions_witness"
        assert cp[4].tobytes() == wit[4].tobytes(), "records differ from the composition's"
        dv = (d_fi.cpu().numpy(), d_kind.cpu().numpy(), d_f.cpu().numpy().view(np.uint32),
              d_s.cpu().numpy().view(np.uint32), d_rec.cpu().numpy().view(P.contact_dtype))
        for k in range(4):
            assert np.array_equal(dv[k], wit[k]), "motions_device differs from motions_witness"
        assert dv[4].tobytes() == wit[4].tobytes() and tuple(int(x) for x in d_n.cpu().numpy()) == wit[5]
        times = {k: [] for k in forms}
        for _ in range(a.rounds):
            for name, fn in forms.items():
                t0 = time.perf_counter()
                fn()
                times[name].append(time.perf_counter() - t0)
        fi = wit[0]
        line = {"motions": K, "samples": int(off[-1]), "links": L, "template_pairs": len(tpl), "a_objects": na,
                "b_objects": a.env, "invalid_motions": int((fi >= 0).sum()), "env_witness": int((wit[1] == 0).sum()),
                "self_witness": int((wit[1] == 1).sum()), "env_candidates": wit[5][0], "env_colliding": wit[5][1],
                "self_candidates": wit[5][2], "self_colliding": wit[5][3],
                "ms_per_call_median": {k: 1e3 * float(np.median(t)) for k, t in times.items()},
                "ms_per_call_min": {k: 1e3 * float(np.min(t)) for k, t in times.items()}, "rounds": a.rounds}
        print(json.dumps(line), flush=True)
    eng.env_destroy(env)
    print(json.dumps({"gpu": gpu_info()}))


if __name__ == "__main__":
    main()
