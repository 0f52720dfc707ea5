import importlib
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
GOLDEN = ROOT / "tests" / "golden"


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with `pytest -m gpu`)")


@pytest.fixture(scope="session")
def orc():
    """The CPU oracle (test infrastructure)."""
    from oracle import pyoracle
    pyoracle.build()
    return pyoracle


@pytest.fixture(scope="session")
def b2():
    """The product bindings (ctypes over libb200post.so). Built if missing; never falls back."""
    mod = importlib.import_module("go-spacemesh_b200")
    if not mod.LIB_PATH.exists():
        mod.build()
    return mod


@pytest.fixture(scope="session")
def golden():
    return {p.stem: json.loads(p.read_text()) for p in GOLDEN.glob("*.json")}


@pytest.fixture(scope="session")
def host_emul(tmp_path_factory):
    """post_device.cuh (the kernels' per-thread arithmetic) compiled as plain C++ for the CPU."""
    import ctypes
    out = tmp_path_factory.mktemp("emul") / "host_emul.so"
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-o", str(out), str(ROOT / "tests" / "host_emul.cpp")],
                   check=True)
    return ctypes.CDLL(str(out))


@pytest.fixture(scope="session")
def gpu_ready(b2):
    provs = b2.providers()
    if not provs:
        pytest.fail("GPU test selected but libb200post reports no CUDA device (there is no CPU fallback)")
    return provs
