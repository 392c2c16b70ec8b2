"""The C++ host mirror's ResidentEnvironment::collide_configurations / configuration_flags: compiles and links against
the C-ABI library everywhere; on the GPU box it runs on the scene the Python mirror runs on, and both must give the same
verdicts and pairs (tests/cpp/test_host_configs.cpp)."""
import os
import subprocess

import numpy as np
import pytest

from tests.common import ROOT

SRC = os.path.join(ROOT, "tests", "cpp", "test_host_configs.cpp")
EXE = os.path.join(ROOT, "tests", "cpp", "test_host_configs.bin")


def _build():
    lib = os.path.join(ROOT, "hpp-fcl_b200")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-o", EXE, SRC, "-L", lib,
                           "-lhppfcl_b200", "-Wl,-rpath," + lib])


def test_cpp_host_configs_compiles_and_refuses_cpu(built):
    import torch
    _build()
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([EXE], capture_output=True, text=True)
    assert r.returncode != 0 and "no CPU fallback" in r.stderr


@pytest.mark.gpu
def test_cpp_and_python_mirrors_agree(built, tmp_path):
    from tests.test_gpu_env_configs import link_kind, python_mirror
    links, robot, env, tpl, v, ep, sp = python_mirror(np.random.default_rng(19))
    _build()
    path = tmp_path / "scene.txt"  # every pose with every digit (hexadecimal floating point)
    with open(path, "w") as fh:
        fh.write("%d %d %d %d\n" % (links, len(robot) // links, len(tpl), len(env)))
        fh.write(" ".join("%d %d" % (i, j) for i, j in tpl) + "\n")
        rows = [(link_kind(k, links), R, T) for k, (R, T) in enumerate(robot)] + list(env)
        for kind, R, T in rows:
            fh.write("%d %s\n" % (kind, " ".join(float(x).hex() for x in list(np.ravel(R)) + list(T))))
    r = subprocess.run([EXE, str(path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "HOST-CONFIGS-OK" in r.stdout, r.stdout + r.stderr
    lines = r.stdout.split("\n")
    assert lines[0] == "verdicts " + "".join(str(int(x)) for x in v)
    cpp = {"env": set(), "self": set()}
    for ln in lines[1:]:
        parts = ln.split()
        if parts and parts[0] in cpp:
            cpp[parts[0]].add((int(parts[1]), int(parts[2]), int(parts[3]), float.fromhex(parts[4])))
    mine = lambda pr: {(int(a), int(b), int(x["num_contacts"]), float(x["distance"])) for a, b, x in zip(*pr)}  # noqa: E731
    assert cpp["env"] == mine(ep) and cpp["self"] == mine(sp)
    assert len(cpp["env"]) > 5 and len(cpp["self"]) > 5
