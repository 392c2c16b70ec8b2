"""The C++ host mirror's ResidentEnvironment::certify_motions: compiles and links against the C-ABI library
everywhere; on the GPU box it runs on the scene the Python mirror runs on, and both must give the same first colliding
and first uncertified sample per motion and the same certified flag per configuration
(tests/cpp/test_host_certify.cpp)."""
import os
import subprocess

import numpy as np
import pytest

from tests.common import ROOT
from tests.test_cpp_host_motions import motion_offsets

SRC = os.path.join(ROOT, "tests", "cpp", "test_host_certify.cpp")


def _build(exe):
    lib = os.path.join(ROOT, "hpp-fcl_b200")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-o", str(exe), SRC, "-L", lib,
                           "-lhppfcl_b200", "-Wl,-rpath," + lib])


def test_cpp_host_certify_compiles_and_refuses_cpu(built, tmp_path):
    import torch
    exe = tmp_path / "test_host_certify.bin"
    _build(exe)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode != 0 and "no CPU fallback" in r.stderr


@pytest.mark.gpu
def test_cpp_and_python_certify_mirrors_agree(built, tmp_path):
    import hppfcl_b200 as hf
    from hppfcl_b200 import workloads as W
    from tests.test_gpu_env_configs import link_kind, mirror_geoms, mirror_scene
    rng = np.random.default_rng(33)
    links, robot, env = mirror_scene(rng)
    link_geom = [hf.Capsule(0.05, 0.14), hf.Box(0.08, 0.08, 0.22)]
    ro = [hf.CollisionObject(link_geom[link_kind(k, links)], hf.Transform3f(R, T)) for k, (R, T) in enumerate(robot)]
    geoms = mirror_geoms()
    eo = [hf.CollisionObject(geoms[gi], hf.Transform3f(R, T)) for gi, R, T in env]
    mr, me = hf.DynamicAABBTreeCollisionManager(), hf.DynamicAABBTreeCollisionManager()
    mr.registerObjects(ro)
    me.registerObjects(eo)
    mr.setup()
    me.setup()
    exe = tmp_path / "test_host_certify.bin"
    _build(exe)
    path = tmp_path / "scene.txt"  # every pose with every digit (hexadecimal floating point)
    with open(path, "w") as fh:
        fh.write("%d %d\n" % (len(robot), len(env)))
        rows = [(link_kind(k, links), R, T) for k, (R, T) in enumerate(robot)] + list(env)
        for kind, R, T in rows:
            fh.write("%d %s\n" % (kind, " ".join(float(x).hex() for x in list(np.ravel(R)) + list(T))))
    off = motion_offsets(len(robot) // links, rng)
    opath = tmp_path / "offsets.txt"
    opath.write_text("\n".join(str(int(v)) for v in off) + "\n")
    # bounds of every size, some invalid
    sweep = rng.choice([0.0, 0.001, 0.005, 0.02, 1.0, np.nan, -1.0], len(robot),
                       p=[0.3, 0.3, 0.2, 0.1, 0.096, 0.002, 0.002])
    spath = tmp_path / "sweep.txt"
    spath.write_text("\n".join(float(v).hex() if np.isfinite(v) else ("nan" if np.isnan(v) else "-inf") for v in sweep)
                     + "\n")
    tpl = W.chain_self_pairs(links, 2)
    with hf.ResidentEnvironment(me) as re:
        fi, fu, cert = re.certify_motions(mr, links, tpl, off, sweep)
        assert (fi >= 0).any() and (fu >= 0).any() and (fu != 0).any()
        with pytest.raises(ValueError):
            re.certify_motions(mr, links, tpl, off, sweep[:-1])
        r = subprocess.run([str(exe), str(path), str(opath), str(links), str(spath)], capture_output=True, text=True,
                           timeout=300)
        assert r.returncode == 0 and "HOST-CERTIFY-OK" in r.stdout, r.stdout + r.stderr
        mot = [ln.split() for ln in r.stdout.split("\n") if ln.startswith("mot ")]
        cfg = [ln.split() for ln in r.stdout.split("\n") if ln.startswith("cfg ")]
        assert [int(p[2]) for p in mot] == fi.tolist() and [int(p[3]) for p in mot] == fu.tolist()
        assert [int(p[2]) for p in cfg] == cert.tolist()
