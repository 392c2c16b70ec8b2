"""Config 4 timing (test tooling, not bench.py: the tree is built by the oracle's restatement of the
reference builder): 10 000-triangle OBBRSS mesh vs N capsules, distance + nearest points.
Prints one JSON line with GPU queries/s (device-resident and host-API), the traversal counters that
define the algorithmic bytes, and the CPU oracle on the same queries."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import hppfcl_b200 as hf  # noqa: E402
from hppfcl_b200 import _pod as P, workloads as W  # noqa: E402
from oracle import oracle_lib  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 100_000
w = W.config4_mesh_vs_capsules(n)
orc = oracle_lib.OracleScene(P)
bid, nodes = orc.register_bvh(w["verts"], w["tris"])
ob = orc.register_shapes(P.make_shapes([P.BV_OBBRSS], [[0, 0, 0]], data=[bid]))
oc = orc.register_shapes(w["capsules"])
eng = hf.Engine(0)
gb = eng.register_bvh_obbrss(nodes, w["verts"], w["tris"])
hb = eng.register_shapes(P.make_shapes([P.BV_OBBRSS], [[0, 0, 0]], data=[gb]))
hc = eng.register_shapes(w["capsules"])
eng.commit()
hm = np.full(n, hb[0], dtype=np.uint32)
hs = hc[w["hc"]]


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()


d = [dev(hm), dev(w["tf_mesh"]), dev(hs), dev(w["tf_caps"])]
d_out = torch.empty(n * P.distance_result_dtype.itemsize, dtype=torch.uint8, device="cuda")
req = P.DistanceRequestPOD()
stream = torch.cuda.current_stream().cuda_stream
for _ in range(3):
    eng.batch_distance_device(n, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), d[3].data_ptr(), d_out.data_ptr(), req, stream=stream)
torch.cuda.synchronize()
s0 = eng.stats()
eng.set_profiling(True)
eng.kernel_times(reset=True)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
steps = 5
e0.record()
for _ in range(steps):
    eng.batch_distance_device(n, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), d[3].data_ptr(), d_out.data_ptr(), req, stream=stream)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / steps
kt = eng.kernel_times(reset=True)
s1 = eng.stats()
t0 = time.perf_counter()
got = eng.batch_distance(hm, w["tf_mesh"], hs, w["tf_caps"], req)
t_host = time.perf_counter() - t0
ns = min(n, 20000)
t0 = time.perf_counter()
ref = orc.batch_distance(np.full(ns, ob[0], dtype=np.uint32), w["tf_mesh"][:ns], oc[w["hc"][:ns]], w["tf_caps"][:ns], req, nthreads=0)
t_cpu = time.perf_counter() - t0
t0 = time.perf_counter()
orc.batch_distance(np.full(2000, ob[0], dtype=np.uint32), w["tf_mesh"][:2000], oc[w["hc"][:2000]], w["tf_caps"][:2000], req, nthreads=1)
t_cpu1 = time.perf_counter() - t0
same = bool(np.array_equal(ref["min_distance"], got["min_distance"][:ns]) and np.array_equal(ref["b1"], got["b1"][:ns])
            and np.array_equal(ref["iterations"], got["iterations"][:ns]))
bv = (s1["bv_tests"] - s0["bv_tests"]) / steps
lf = (s1["leaf_tests"] - s0["leaf_tests"]) / steps
alg_bytes = 136 * bv + 96 * lf + (136 + 96) * n  # SURVEY 8d: RSS half of the node + header, leaf triangle, capsule+pose, result
import ctypes as _C
_prof = (_C.c_ulonglong * 5)()
eng.L.hfb_debug_bvh_profile.argtypes = [_C.c_void_p, _C.c_void_p]
eng.L.hfb_debug_bvh_profile(eng.h, _prof)
_calls = steps + 3
# k_bvhq runs at most one block per SM (bvhq_blocks); the counters are SM clock cycles
_nb = min(torch.cuda.get_device_properties(0).multi_processor_count, (n + 63) // 64)
_cyc_per_us = torch.cuda.clock_rate(0)  # current SM clock, MHz
phase = {"bv_us_per_block": _prof[0] / _cyc_per_us / _nb / _calls, "leaf_us_per_block": _prof[1] / _cyc_per_us / _nb / _calls,
         "epa_us_per_block": _prof[2] / _cyc_per_us / _nb / _calls, "cycles_per_block": _prof[3] / _nb / _calls,
         "epa_phases_per_block": _prof[4] / _nb / _calls}
print(json.dumps({"phase_profile": phase, "workload": "config4: 10k-tri OBBRSS mesh vs %d capsules, distance" % n, "queries_per_s": n / (ms * 1e-3),
                  "ms_per_batch": ms, "k_bvh_ms": kt["bvh_ms"] / steps, "host_api_queries_per_s": n / t_host,
                  "bv_tests_per_query": bv / n, "leaf_tests_per_query": lf / n,
                  "algorithmic_GBps": alg_bytes / (kt["bvh_ms"] / steps * 1e-3) / 1e9,
                  "cpu_oracle_queries_per_s": ns / t_cpu, "cpu_threads": oracle_lib.lib().oracle_max_threads(),
                  "cpu_single_thread_queries_per_s": 2000 / t_cpu1, "bit_identical_to_oracle": same,
                  "watchdog_trips": s1["watchdog_trips"]}))
