"""The C++ host mirror's RobotModel: compiles and links against the C-ABI library everywhere; on the GPU box it builds
the model the Python mirror builds here, and both must give the same link handles, poses and sweep bounds bit for bit,
and, fed to ResidentEnvironment, the same certify_motions and configuration_flags outputs (tests/cpp/test_host_robot.cpp).
The C++ program also checks that malformed input throws std::invalid_argument; the Python mirror raises ValueError."""
import os
import subprocess

import numpy as np
import pytest

from tests.common import ROOT

SRC = os.path.join(ROOT, "tests", "cpp", "test_host_robot.cpp")


def _build(exe):
    lib = os.path.join(ROOT, "hpp-fcl_b200")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-o", str(exe), SRC, "-L", lib,
                           "-lhppfcl_b200", "-Wl,-rpath," + lib])


def test_cpp_host_robot_compiles_and_refuses_cpu(built, tmp_path):
    import torch
    exe = tmp_path / "test_host_robot.bin"
    _build(exe)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode != 0 and "no CPU fallback" in r.stderr


@pytest.mark.gpu
def test_cpp_and_python_robot_mirrors_agree(built, tmp_path):
    import hppfcl_b200 as hf
    up = hf.Transform3f(np.eye(3), [0, 0, 0.1])
    joints = [(-1, hf.JOINT_REVOLUTE, [0, 0, 1], hf.Transform3f()),
              (0, hf.JOINT_REVOLUTE, [0, 1, 0], hf.Transform3f(np.eye(3), [0, 0, 0.2]))]
    links = [(0, up, hf.Box(0.05, 0.05, 0.2)), (1, up, hf.Capsule(0.03, 0.1)),
             (-1, hf.Transform3f(np.eye(3), [0.5, 0, 0]), hf.Sphere(0.05))]
    exe = tmp_path / "test_host_robot.bin"
    _build(exe)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "HOST-ROBOT-OK" in r.stdout, r.stdout + r.stderr
    rows = {k: [ln.split()[1:] for ln in r.stdout.split("\n") if ln.startswith(k + " ")] for k in ("tf", "mot", "cfg", "flag")}
    with hf.RobotModel(joints, links) as robot:
        s = robot.sample_motions([[0.0, 0.0], [1.0, -0.5]], [[1.5, 1.0], [-1.0, 0.5]], [0, 20, 45])
        with pytest.raises(ValueError):
            robot.poses(np.zeros(3))
        with pytest.raises(ValueError):
            robot.sample_motions([[0.0, 0.0], [1.0, -0.5]], [[1.5, 1.0], [-1.0, 0.5]], [0, 20, 10])
        assert len(rows["tf"]) == len(s.tfs) == 135
        cpp_h = np.array([int(row[1]) for row in rows["tf"]], dtype=np.uint32)
        cpp_v = np.array([[float.fromhex(x) for x in row[2:]] for row in rows["tf"]])
        # (the handles are each process's own arena's: compared as the same link-per-object pattern)
        assert np.array_equal(cpp_h, np.tile(cpp_h[:3], 45)) and len(set(cpp_h[:3].tolist())) == 3
        assert np.array_equal(s.handles, np.tile(s.handles[:3], 45))
        py_v = np.concatenate([s.tfs["R"], s.tfs["T"], s.sweep[:, None]], axis=1)
        assert cpp_v.tobytes() == py_v.tobytes()
        mgr = hf.DynamicAABBTreeCollisionManager()
        mgr.registerObjects([hf.CollisionObject(hf.Box(0.1, 0.1, 0.1), hf.Transform3f(np.eye(3), [0.2, 0.1, 0.25]))])
        with hf.ResidentEnvironment(mgr) as env:
            fi, fu, cert = env.certify_motions(s, 3, [(0, 2)], s.offsets, s.sweep)
            flags = env.configuration_flags(robot.poses(s.q), 3, [(0, 2)])
        assert [int(m[1]) for m in rows["mot"]] == fi.tolist() and [int(m[2]) for m in rows["mot"]] == fu.tolist()
        assert [int(c[1]) for c in rows["cfg"]] == cert.tolist()
        assert [int(c[1]) for c in rows["flag"]] == flags.tolist()
