"""The C++ host mirror's ResidentEnvironment::collide_motions / first_invalid_samples: compiles and links against the
C-ABI library everywhere; on the GPU box it runs on the scene the Python mirror runs on, and both must give the same
first colliding sample and witness per motion (tests/cpp/test_host_motions.cpp)."""
import os
import subprocess

import numpy as np
import pytest

from tests.common import ROOT

SRC = os.path.join(ROOT, "tests", "cpp", "test_host_motions.cpp")


def _build(exe):
    lib = os.path.join(ROOT, "hpp-fcl_b200")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-o", str(exe), SRC, "-L", lib,
                           "-lhppfcl_b200", "-Wl,-rpath," + lib])


def test_cpp_host_motions_compiles_and_refuses_cpu(built, tmp_path):
    import torch
    exe = tmp_path / "test_host_motions.bin"
    _build(exe)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode != 0 and "no CPU fallback" in r.stderr


def motion_offsets(n_configs, rng):
    """motions of 0 to 12 configurations, one after another, covering all n_configs"""
    sizes = []
    while sum(sizes) < n_configs:
        sizes.append(min(int(rng.integers(0, 13)), n_configs - sum(sizes)))
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)


@pytest.mark.gpu
def test_cpp_and_python_motions_mirrors_agree(built, tmp_path):
    import hppfcl_b200 as hf
    from hppfcl_b200 import workloads as W
    from tests.test_gpu_env_configs import link_kind, mirror_geoms, mirror_scene
    rng = np.random.default_rng(31)
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
    exe = tmp_path / "test_host_motions.bin"
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
    tpl = W.chain_self_pairs(links, 2)
    with hf.ResidentEnvironment(me) as re:
        fi, kind, first, second, rec = re.collide_motions(mr, links, tpl, off)
        assert (fi >= 0).any() and (fi < 0).any()
        assert np.array_equal(re.first_invalid_samples(mr, links, tpl, off), fi)
        r = subprocess.run([str(exe), str(path), str(opath), str(links)], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0 and "HOST-MOTIONS-OK" in r.stdout, r.stdout + r.stderr
        cpp = [ln.split() for ln in r.stdout.split("\n") if ln.startswith("mot ")]
        assert [int(p[2]) for p in cpp] == fi.tolist() and [int(p[3]) for p in cpp] == kind.tolist()
        assert [int(p[4]) for p in cpp] == first.tolist() and [int(p[5]) for p in cpp] == second.tolist()
        # every field of every record, a NaN equal to a NaN
        doubles = np.array([[float.fromhex(x) for x in p[6:20]] for p in cpp])
        want = np.concatenate([rec["distance"][:, None], rec["p1"], rec["p2"], rec["normal"], rec["pos"],
                               rec["distance_lower_bound"][:, None]], axis=1)
        assert np.array_equal(doubles, want, equal_nan=True)
        ints = np.array([[int(x) for x in p[20:25]] for p in cpp])
        assert np.array_equal(ints, np.stack([rec[f].astype(np.int64) for f in ("b1", "b2", "status", "num_contacts",
                                                                                  "iterations")], axis=1))
