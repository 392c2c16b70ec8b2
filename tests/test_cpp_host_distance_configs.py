"""The C++ host mirror's ResidentEnvironment::distance_configurations / configuration_clearance: compiles and links
against the C-ABI library everywhere; on the GPU box it runs on the scene the Python mirror runs on, and both must give
the same winner and distance per configuration (tests/cpp/test_host_distance_configs.cpp)."""
import os
import subprocess

import numpy as np
import pytest

from tests.common import ROOT

SRC = os.path.join(ROOT, "tests", "cpp", "test_host_distance_configs.cpp")


def _build(exe):
    lib = os.path.join(ROOT, "hpp-fcl_b200")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-o", str(exe), SRC, "-L", lib,
                           "-lhppfcl_b200", "-Wl,-rpath," + lib])


def test_cpp_host_distance_configs_compiles_and_refuses_cpu(built, tmp_path):
    import torch
    exe = tmp_path / "test_host_distance_configs.bin"
    _build(exe)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode != 0 and "no CPU fallback" in r.stderr


@pytest.mark.gpu
def test_cpp_and_python_configs_mirrors_agree(built, tmp_path):
    import hppfcl_b200 as hf
    from hppfcl_b200 import workloads as W
    from tests.test_gpu_env_configs import link_kind, mirror_geoms, mirror_scene
    links, robot, env = mirror_scene(np.random.default_rng(29))
    link_geom = [hf.Capsule(0.05, 0.14), hf.Box(0.08, 0.08, 0.22)]
    ro = [hf.CollisionObject(link_geom[link_kind(k, links)], hf.Transform3f(R, T)) for k, (R, T) in enumerate(robot)]
    geoms = mirror_geoms()
    eo = [hf.CollisionObject(geoms[gi], hf.Transform3f(R, T)) for gi, R, T in env]
    mr, me = hf.DynamicAABBTreeCollisionManager(), hf.DynamicAABBTreeCollisionManager()
    mr.registerObjects(ro)
    me.registerObjects(eo)
    mr.setup()
    me.setup()
    exe = tmp_path / "test_host_distance_configs.bin"
    _build(exe)
    path = tmp_path / "scene.txt"  # every pose with every digit (hexadecimal floating point)
    with open(path, "w") as fh:
        fh.write("%d %d\n" % (len(robot), len(env)))
        rows = [(link_kind(k, links), R, T) for k, (R, T) in enumerate(robot)] + list(env)
        for kind, R, T in rows:
            fh.write("%d %s\n" % (kind, " ".join(float(x).hex() for x in list(np.ravel(R)) + list(T))))
    tpl = W.chain_self_pairs(links, 2)
    with hf.ResidentEnvironment(me) as re:
        for maxd in (0.1, np.inf):
            kind, first, second, dist, rec = re.distance_configurations(mr, links, tpl, max_distance=maxd)
            assert (kind >= 0).any() and (maxd == np.inf) == (kind >= 0).all()
            r = subprocess.run([str(exe), str(path), repr(float(maxd)), str(links)], capture_output=True, text=True,
                               timeout=300)
            assert r.returncode == 0 and "HOST-DISTANCE-CONFIGS-OK" in r.stdout, r.stdout + r.stderr
            cpp = [ln.split() for ln in r.stdout.split("\n") if ln.startswith("cfg ")]
            assert [int(p[2]) for p in cpp] == kind.tolist()
            assert [int(p[3]) for p in cpp] == first.tolist() and [int(p[4]) for p in cpp] == second.tolist()
            assert [float.fromhex(p[5]) for p in cpp] == dist.tolist()
