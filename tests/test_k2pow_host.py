"""CPU tier for k2pow: the product's host half of RandomX (cache + SuperscalarHash generator, csrc/randomx_host.cpp)
against the oracle, and the C ABI's behaviour without a device."""
import ctypes
import importlib
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def host_rx(tmp_path_factory):
    """csrc/randomx_host.cpp compiled on its own (it is plain C++) behind a two-function C shim."""
    d = tmp_path_factory.mktemp("rxhost")
    shim = d / "shim.cpp"
    shim.write_text('''
#include "randomx_host.h"
#include <cstring>
using namespace b200post::rx;
static CacheImage g;
extern "C" void rxh_build(const char *key, size_t n) { build_cache(key, n, g); }
extern "C" const uint64_t *rxh_memory() { return g.memory.data(); }
extern "C" uint32_t rxh_prog(int i, uint8_t *out /* 8 bytes per op: opcode,dst,src,shift,imm32 */, uint64_t *rcp, uint32_t *addr) {
    *addr = g.programs[i].address_reg;
    for (size_t j = 0; j < g.programs[i].ops.size(); j++) { memcpy(out + 8 * j, &g.programs[i].ops[j], 8); rcp[j] = g.programs[i].ops[j].rcp; }
    return (uint32_t)g.programs[i].ops.size();
}
extern "C" uint64_t rxh_reciprocal(uint32_t d) { return reciprocal(d); }
extern "C" void rxh_blake2b(void *o, size_t ol, const void *i, size_t il) { blake2b(o, ol, i, il); }
''')
    out = d / "librxhost.so"
    src = ROOT / "go-spacemesh_b200" / "csrc"
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", f"-I{src}", "-o", str(out), str(shim), str(src / "randomx_host.cpp")], check=True)
    L = ctypes.CDLL(str(out))
    L.rxh_memory.restype = ctypes.POINTER(ctypes.c_uint64)
    L.rxh_reciprocal.restype = ctypes.c_uint64
    return L


def test_product_host_cache_and_programs_equal_oracle(host_rx):
    from oracle import pyrandomx as orx
    key = b"test key 000"
    host_rx.rxh_build(key, len(key))
    mem = np.ctypeslib.as_array(host_rx.rxh_memory(), shape=(256 * 1024 * 1024 // 8,))
    assert int(mem[0]) == 0x191e0e1d23c02186 and int(mem[1568413]) == 0xf1b62fe6210bf8b1 and int(mem[33554431]) == 0x1f47f056d05cd99b
    c = orx.Cache(key)
    try:
        assert np.array_equal(mem, c.memory())
        # oracle opcode numbering -> the product's device numbering (7/8/9-byte immediates collapse)
        to_dev = {0: 0, 1: 1, 2: 2, 3: 3, 4: 4, 5: 5, 6: 6, 7: 5, 8: 6, 9: 5, 10: 6, 11: 7, 12: 8, 13: 9}
        for i, ref in enumerate(c.programs()):
            buf = ctypes.create_string_buffer(8 * 512)
            rcp = (ctypes.c_uint64 * 512)()
            addr = ctypes.c_uint32()
            n = host_rx.rxh_prog(i, buf, rcp, ctypes.byref(addr))
            assert n == ref.size and addr.value == ref.address_reg
            for j in range(n):
                op, dst, src, shift = buf.raw[8 * j:8 * j + 4]
                imm = int.from_bytes(buf.raw[8 * j + 4:8 * j + 8], "little")
                r = ref.ins[j]
                assert (op, dst, src, imm) == (to_dev[r.opcode], r.dst, r.src, r.imm32), (i, j)
                if r.opcode == 2:
                    assert shift == (r.mod >> 2) & 3
                if r.opcode == 13:
                    assert rcp[j] == r.rcp
    finally:
        c.close()
    for d, e in ((3, 12297829382473034410), (0xffffffff, 9223372039002259456), (15000001, 10316166306300415204)):
        assert host_rx.rxh_reciprocal(d) == e
    import hashlib
    for n in (0, 1, 64, 128, 129, 300):
        o = ctypes.create_string_buffer(64)
        m = bytes(range(256)) * 2
        host_rx.rxh_blake2b(o, 64, m[:n], n)
        assert o.raw == hashlib.blake2b(m[:n]).digest()


def test_k2pow_api_without_a_device(b2):
    k2 = importlib.import_module("go-spacemesh_b200.k2pow")
    d = bytes.fromhex("000dfb23b0979b4b" + "00" * 24)          # config/mainnet.go:41
    assert k2.scale_difficulty(d, 1) == d
    assert int.from_bytes(k2.scale_difficulty(d, 4), "big") == int.from_bytes(d, "big") // 4
    assert int.from_bytes(k2.scale_difficulty(b"\xff" * 32, 3), "big") == (2**256 - 1) // 3
    assert k2.scale_difficulty(d, 0) == d                              # num_units 0 counts as 1
    from oracle import pyrandomx as orx
    for first, count in ((orx.DATASET_ITEMS - 1, 2), (orx.DATASET_ITEMS + 1, 0), (2**64 - 1, 2)):
        with pytest.raises(b2.B200PostError) as e:                     # checked before any device is looked for
            k2.dataset(first, count)
        assert e.value.code == b2.ERR_INVALID_ARGUMENT
    if b2.providers():
        pytest.skip("a CUDA device is present: the no-device contract is covered on CPU-only boxes")
    for call in (lambda: k2.prepare(), lambda: k2.hashes(0, bytes(8), bytes(32), 0, 1), lambda: k2.search(0, bytes(8), bytes(32), b"\xff" * 32, 0, 1),
                 lambda: k2.verify(0, 0, bytes(8), bytes(32), b"\xff" * 32), lambda: k2.randomx_hash(b"k", [b"x"]),
                 lambda: k2.dataset(0, 1), lambda: k2.search_groups(bytes(8), bytes(32), b"\xff" * 32, 2)):
        with pytest.raises(b2.B200PostError) as e:
            call()
        assert e.value.code == b2.ERR_NO_DEVICE
    with pytest.raises(b2.B200PostError) as e:
        k2.prepare(provider=b2.CPU_PROVIDER_ID)
    assert e.value.code == b2.ERR_UNSUPPORTED


def test_scale_difficulty_is_exact_integer_division(b2):
    """The one division the prover, the verifier and the export share: floor(difficulty / num_units) over 256 bits."""
    k2 = importlib.import_module("go-spacemesh_b200.k2pow")
    rng = np.random.default_rng(31)
    values = [0, 1, 2**256 - 1, 2**255, 2**224 - 1] + [int.from_bytes(bytes(rng.integers(0, 256, 32, dtype=np.uint8)), "big")
                                                      for _ in range(40)]
    for v in values:
        for units in (1, 2, 3, 4, 7, 255, 256, 65537, 2**31 - 1, 2**32 - 1):
            assert int.from_bytes(k2.scale_difficulty(v.to_bytes(32, "big"), units), "big") == v // units, (hex(v), units)
