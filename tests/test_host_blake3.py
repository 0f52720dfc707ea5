"""CPU tier: the product's host BLAKE3 (csrc/host_hash.cpp: blake3_single_chunk, which hashes the Subset seed, the
commitment and the AES keys) against the `blake3` wheel, across the block seams of the one chunk it accepts and the
XOF output lengths the Subset stream reaches."""
import ctypes
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
OUT_LENS = (1, 16, 32, 63, 64, 65, 256, 512, 1000, 8192)


@pytest.fixture(scope="module")
def host_blake3(tmp_path_factory):
    out = tmp_path_factory.mktemp("blake3") / "host_blake3.so"
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-o", str(out), str(ROOT / "tests" / "host_blake3_shim.cpp"),
                    str(ROOT / "go-spacemesh_b200" / "csrc" / "host_hash.cpp")], check=True)
    lib = ctypes.CDLL(str(out))
    lib.shim_blake3.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t]
    lib.shim_blake3.restype = ctypes.c_int

    def run(msg: bytes, outlen: int):
        buf = ctypes.create_string_buffer(outlen + 1)
        buf.raw = b"\xa5" * (outlen + 1)                  # a canary after the output
        ok = lib.shim_blake3(msg, len(msg), buf, outlen)
        assert buf.raw[outlen] == 0xA5, "wrote past the output"
        return bool(ok), buf.raw[:outlen]
    return run


def _lengths():
    rng = np.random.default_rng(7)
    return [0, 1, 63, 64, 65, 127, 128, 129, 512, 1023, 1024] + sorted(int(n) for n in rng.integers(0, 1025, 200))


def test_single_chunk_against_wheel(host_blake3):
    blake3 = pytest.importorskip("blake3")
    rng = np.random.default_rng(8)
    for n in _lengths():
        msg = bytes(rng.integers(0, 256, n, dtype=np.uint8))
        want = blake3.blake3(msg).digest(max(OUT_LENS))
        for outlen in OUT_LENS:
            assert host_blake3(msg, outlen) == (True, want[:outlen]), (n, outlen)


def test_input_above_one_chunk_is_refused(host_blake3):
    ok, _ = host_blake3(bytes(1025), 32)
    assert not ok
    ok, _ = host_blake3(bytes(4096), 32)
    assert not ok
