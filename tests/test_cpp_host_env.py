"""The C++ host mirror's ResidentEnvironment and the manager's update(obj) / update(objs): compiles and links against the
C-ABI library everywhere; on the GPU box the queries run (tests/cpp/test_host_env.cpp)."""
import os
import subprocess

import pytest

from tests.common import ROOT

SRC = os.path.join(ROOT, "tests", "cpp", "test_host_env.cpp")
EXE = os.path.join(ROOT, "tests", "cpp", "test_host_env.bin")


def _build():
    lib = os.path.join(ROOT, "hpp-fcl_b200")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-o", EXE, SRC, "-L", lib,
                           "-lhppfcl_b200", "-Wl,-rpath," + lib])


def test_cpp_host_env_compiles_and_refuses_cpu(built):
    import torch
    _build()
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([EXE], capture_output=True, text=True)
    assert r.returncode != 0 and "no CPU fallback" in r.stderr


@pytest.mark.gpu
def test_cpp_host_env_on_gpu(built):
    _build()
    r = subprocess.run([EXE], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "HOST-ENV-OK" in r.stdout, r.stdout + r.stderr
