"""The C++ host mirror's ResidentEnvironment::validate_motions: compiles and links against the C-ABI library
everywhere; on the GPU box it validates the motions the Python mirror validates here, and both must give the same
status, t_valid, t_collide, witness and counts, field by field and bit for bit (tests/cpp/test_host_validate.cpp).
The C++ program also checks that the refusals throw std::invalid_argument; the Python mirror raises ValueError."""
import os
import subprocess

import numpy as np
import pytest

from tests.common import ROOT

SRC = os.path.join(ROOT, "tests", "cpp", "test_host_validate.cpp")


def _build(exe):
    lib = os.path.join(ROOT, "hpp-fcl_b200")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-o", str(exe), SRC, "-L", lib,
                           "-lhppfcl_b200", "-Wl,-rpath," + lib])


def test_cpp_host_validate_compiles_and_refuses_cpu(built, tmp_path):
    import torch
    exe = tmp_path / "test_host_validate.bin"
    _build(exe)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode != 0 and "no CPU fallback" in r.stderr


@pytest.mark.gpu
def test_cpp_and_python_validate_mirrors_agree(built, tmp_path):
    import hppfcl_b200 as hf
    up = hf.Transform3f(np.eye(3), [0, 0, 0.1])
    joints = [(-1, hf.JOINT_REVOLUTE, [0, 0, 1], hf.Transform3f()),
              (0, hf.JOINT_REVOLUTE, [0, 1, 0], hf.Transform3f(np.eye(3), [0, 0, 0.2]))]
    links = [(0, up, hf.Box(0.05, 0.05, 0.2)), (1, up, hf.Capsule(0.03, 0.1)),
             (-1, hf.Transform3f(np.eye(3), [0.5, 0, 0]), hf.Sphere(0.05))]
    exe = tmp_path / "test_host_validate.bin"
    _build(exe)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "HOST-VALIDATE-OK" in r.stdout, r.stdout + r.stderr
    val = [ln.split()[1:] for ln in r.stdout.split("\n") if ln.startswith("val ")]
    cnt = [ln.split()[1:] for ln in r.stdout.split("\n") if ln.startswith("cnt ")]
    q0 = np.array([[0.0, 0.0], [1.0, -0.5], [-2.0, 0.3], [0.4, 0.4]])
    q1 = np.array([[1.5, 1.0], [-1.0, 0.5], [2.0, 0.3], [0.4, 0.4]])
    with hf.RobotModel(joints, links) as robot:
        mgr = hf.DynamicAABBTreeCollisionManager()
        mgr.registerObjects([hf.CollisionObject(hf.Box(0.1, 0.1, 0.1), hf.Transform3f(np.eye(3), [0.2, 0.1, 0.25]))])
        with hf.ResidentEnvironment(mgr) as env:
            runs = [env.validate_motions(robot, q0, q1, [(0, 2)], initial_depth=1, max_depth=7, max_samples=1 << 20),
                    env.validate_motions(robot, q0, q1, [(0, 2)], initial_depth=2, max_depth=6, max_samples=9,
                                         first_motion=1, num_motions=2)]
            with pytest.raises(ValueError):
                env.validate_motions(robot, q0, q1[:3], [(0, 2)], initial_depth=1, max_depth=4, max_samples=100)
    assert len(val) == 8 and len(cnt) == 2
    for row in val:
        p, m = int(row[0]), int(row[1])
        v = runs[p]
        assert int(row[2]) == v.status[m]
        assert float.fromhex(row[3]) == v.t_valid[m] and float.fromhex(row[4]) == v.t_collide[m]
        assert int(row[5]) == v.kind[m] and int(row[6]) == v.first[m] and int(row[7]) == v.second[m]
        assert bytes.fromhex(row[8]) == v.contacts[m:m + 1].tobytes()
    for row in cnt:
        v = runs[int(row[0])]
        assert [int(x) for x in row[1:]] == [v.n_rounds, v.n_samples, v.n_env_candidates, v.n_self_candidates,
                                             v.n_unsupported]
    assert runs[1].status[0] == -1 and runs[1].status[3] == -1
