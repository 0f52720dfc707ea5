"""CPU ORACLE for k2pow (RandomX), Python side — TEST INFRASTRUCTURE ONLY.

ctypes bindings of oracle/librandomx_oracle.so (randomx_oracle.c: a from-spec restatement of tevador/RandomX v1.1.x,
the function behind go-spacemesh's k2pow: cmd/root.go:254-259, activation/post_types.go:116-121,
activation/nipost.go:171, activation/post_verifier.go:150-160).  Pinned on RandomX's own known-answer vectors
(tests/test_randomx_oracle.py).  Nothing in the product package imports this module.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
_LIB_PATH = _HERE / "librandomx_oracle.so"
_lib = None

# post-rs pow/randomx.rs (recollection, "parity unpinned"): the RandomX cache key of spacemesh's k2pow
K2POW_CACHE_KEY = b"spacemesh-randomx-cache-key"
# RandomX dataset: (2 GiB base + 32 MiB - 64 B extra) / 64-byte items
DATASET_ITEMS = (2**31 + 33554368) // 64


class SsInstr(ctypes.Structure):
    _fields_ = [("opcode", ctypes.c_uint8), ("dst", ctypes.c_uint8), ("src", ctypes.c_uint8), ("mod", ctypes.c_uint8),
                ("imm32", ctypes.c_uint32), ("rcp", ctypes.c_uint64)]


class SsProgram(ctypes.Structure):
    _fields_ = [("ins", SsInstr * 512), ("size", ctypes.c_uint32), ("address_reg", ctypes.c_uint32)]


def build(force: bool = False) -> Path:
    src = _HERE / "randomx_oracle.c"
    if force or not _LIB_PATH.exists() or _LIB_PATH.stat().st_mtime < src.stat().st_mtime:
        subprocess.run(["make", "-C", str(_HERE), "-s", "librandomx_oracle.so"] + (["-B"] if force else []), check=True)
    return _LIB_PATH


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(str(_LIB_PATH))
        vp, u64, sz = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_size_t
        L.rxo_blake2b.argtypes = [vp, sz, ctypes.c_char_p, sz]
        L.rxo_argon2d_fill.argtypes = [vp, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32,
                                       ctypes.c_char_p, ctypes.c_uint32, ctypes.c_uint32, vp]
        L.rxo_reciprocal.restype = u64
        L.rxo_reciprocal.argtypes = [ctypes.c_uint32]
        L.rxo_cache_new.restype = vp
        L.rxo_cache_new.argtypes = [ctypes.c_char_p, sz]
        L.rxo_cache_free.argtypes = [vp]
        L.rxo_cache_memory.restype = ctypes.POINTER(ctypes.c_uint64)
        L.rxo_cache_memory.argtypes = [vp]
        L.rxo_cache_programs.restype = ctypes.POINTER(SsProgram)
        L.rxo_cache_programs.argtypes = [vp]
        L.rxo_dataset_item.argtypes = [vp, u64, vp]
        L.rxo_dataset_init.argtypes = [vp, ctypes.c_int]
        L.rxo_has_dataset.argtypes = [vp]
        L.rxo_dataset_memory.restype = ctypes.POINTER(ctypes.c_uint64)
        L.rxo_dataset_memory.argtypes = [vp]
        L.rxo_hash.argtypes = [vp, ctypes.c_char_p, sz, vp]
        L.rxo_vm_new.restype = vp
        L.rxo_vm_free.argtypes = [vp]
        L.rxo_hash_vm.argtypes = [vp, vp, ctypes.c_char_p, sz, vp, vp]
        L.rxo_k2pow_input.argtypes = [u64, ctypes.c_uint8, ctypes.c_char_p, ctypes.c_char_p, vp]
        L.rxo_k2pow_scan.restype = ctypes.c_double
        L.rxo_k2pow_scan.argtypes = [vp, ctypes.c_uint8, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, u64, u64,
                                     ctypes.c_int, vp, ctypes.POINTER(u64)]
        L.rxo_fill_aes_1rx4.argtypes = [vp, sz, vp]
        L.rxo_fill_aes_4rx4.argtypes = [ctypes.c_char_p, sz, vp]
        L.rxo_hash_aes_1rx4.argtypes = [ctypes.c_char_p, sz, vp]
        _lib = L
    return _lib


def default_threads() -> int:
    return max(1, len(os.sched_getaffinity(0)))


def blake2b(msg: bytes, outlen: int = 64) -> bytes:
    o = ctypes.create_string_buffer(outlen)
    lib().rxo_blake2b(o, outlen, msg, len(msg))
    return o.raw


class Cache:
    """RandomX cache for one key (256 MiB Argon2d memory + 8 SuperscalarHash programs); optional full dataset."""

    def __init__(self, key: bytes):
        self.key = key
        self._h = lib().rxo_cache_new(key, len(key))
        if not self._h:
            raise MemoryError("rxo_cache_new failed")

    def close(self):
        if self._h:
            lib().rxo_cache_free(self._h)
            self._h = None

    def __del__(self):
        self.close()

    @property
    def handle(self):
        return self._h

    def memory(self) -> np.ndarray:
        """The 256 MiB cache as a (33554432,) uint64 view (owned by the cache)."""
        p = lib().rxo_cache_memory(self._h)
        return np.ctypeslib.as_array(p, shape=(256 * 1024 * 1024 // 8,))

    def programs(self):
        p = lib().rxo_cache_programs(self._h)
        return [p[i] for i in range(8)]

    def program_bytes(self, i: int) -> bytes:
        """Program i as RandomX's 8-byte Instruction records (opcode, dst, src, mod, imm32)."""
        import struct
        pr = self.programs()[i]
        return b"".join(struct.pack("<BBBBI", pr.ins[j].opcode, pr.ins[j].dst, pr.ins[j].src, pr.ins[j].mod, pr.ins[j].imm32)
                        for j in range(pr.size))

    def dataset_item(self, n: int) -> np.ndarray:
        out = np.zeros(8, dtype=np.uint64)
        lib().rxo_dataset_item(self._h, n, out.ctypes.data)
        return out

    def init_dataset(self, threads: int | None = None):
        if lib().rxo_dataset_init(self._h, threads or default_threads()) != 0:
            raise MemoryError("dataset allocation failed")

    def dataset(self) -> np.ndarray:
        """The fast-mode dataset as a (DATASET_ITEMS, 8) uint64 view (owned by the cache); init_dataset() first."""
        p = lib().rxo_dataset_memory(self._h)
        if not p:
            raise ValueError("no dataset: call init_dataset() first")
        return np.ctypeslib.as_array(p, shape=(DATASET_ITEMS, 8))

    def hash(self, data: bytes, trace: bool = False):
        o = ctypes.create_string_buffer(32)
        if not trace:
            lib().rxo_hash(self._h, data, len(data), o)
            return o.raw
        tr = np.zeros(8 * 256, dtype=np.uint8)
        vm = lib().rxo_vm_new()
        lib().rxo_hash_vm(vm, self._h, data, len(data), o, tr.ctypes.data)
        lib().rxo_vm_free(vm)
        return o.raw, tr.reshape(8, 256)

    def k2pow_scan(self, nonce_group: int, challenge8: bytes, node_id: bytes, start: int, count: int,
                   difficulty: bytes | None = None, threads: int | None = None, want_hashes: bool = True):
        """hashes of pow = start..start+count-1 (count x 32 uint8), the smallest pow below `difficulty` (or None), seconds."""
        hashes = np.zeros((count, 32), dtype=np.uint8) if want_hashes else None
        found = ctypes.c_uint64(0)
        secs = lib().rxo_k2pow_scan(self._h, nonce_group, challenge8, node_id, difficulty, start, count,
                                    threads or default_threads(), hashes.ctypes.data if want_hashes else None,
                                    ctypes.byref(found))
        return hashes, (None if found.value == 2**64 - 1 else found.value), secs


def k2pow_input(pow_: int, nonce_group: int, challenge8: bytes, node_id: bytes) -> bytes:
    o = ctypes.create_string_buffer(48)
    lib().rxo_k2pow_input(pow_, nonce_group, challenge8, node_id, o)
    return o.raw


def scale_pow_difficulty(difficulty32: bytes, num_units: int) -> bytes:
    """post-rs: the configured difficulty (256-bit big-endian) divided by num_units (recollection, unpinned)."""
    return (int.from_bytes(difficulty32, "big") // max(1, num_units)).to_bytes(32, "big")
