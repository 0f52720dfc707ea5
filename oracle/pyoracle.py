"""CPU ORACLE, Python side — TEST INFRASTRUCTURE ONLY (see oracle/post_oracle.h for parity status).

Two independent restatements of the POST label function live here:

* ``py_*``  — numpy + hashlib + the ``blake3`` wheel: scrypt-jane's scrypt (ChaCha20/8 mix, HMAC-Keccak-512
  PBKDF2) written array-at-a-time; its Keccak-f is pinned against ``hashlib.sha3_512`` (same permutation, other
  pad byte) and the whole function against the real VRF nonces of the reference's checkpoint fixture
  (tests/golden/checkpoint_vrf.json).  Used to pin the C oracle and to generate tests/golden/*.json.
* ``c_*``   — ctypes bindings of oracle/libpost_oracle.so (post_oracle.c), the fast checker the
  GPU parity tests and bench.py's cpu_baseline use.

Reference anchors: activation/post.go:295,355-361 (Initialize), activation/post_verifier.go:159
(Verify), activation/validation.go:261-282 (VerifyVRFNonce), hash/hash.go:16-25 (blake3).
The proof-side conventions (verify / prove helpers below) are "parity unpinned".

Nothing in the product package imports this module.
"""
from __future__ import annotations

import ctypes
import hashlib
import os
import subprocess
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
_LIB_PATH = _HERE / "libpost_oracle.so"
_lib = None


def build(force: bool = False) -> Path:
    """Compile oracle/libpost_oracle.so with the committed Makefile (gcc only)."""
    src = _HERE / "post_oracle.c"
    if force or not _LIB_PATH.exists() or _LIB_PATH.stat().st_mtime < src.stat().st_mtime:
        subprocess.run(["make", "-C", str(_HERE), "-s"] + (["-B"] if force else []), check=True)
    return _LIB_PATH


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(str(_LIB_PATH))
        u8p, u64 = ctypes.c_char_p, ctypes.c_uint64
        L.oracle_scrypt.argtypes = [u8p, ctypes.c_size_t, u8p, ctypes.c_size_t, u64, ctypes.c_uint32,
                                    ctypes.c_uint32, ctypes.c_void_p, ctypes.c_size_t]
        L.oracle_scrypt.restype = ctypes.c_int
        L.oracle_scrypt_jane.argtypes = L.oracle_scrypt.argtypes
        L.oracle_scrypt_jane.restype = ctypes.c_int
        L.oracle_labels_range.argtypes = [u8p, u64, ctypes.c_uint32, ctypes.c_uint32, u64, u64, ctypes.c_void_p,
                                          ctypes.c_void_p, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(u64),
                                          ctypes.c_void_p, ctypes.c_int]
        L.oracle_labels_range.restype = ctypes.c_int
        L.oracle_labels_gather.argtypes = [ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, u64, ctypes.c_uint32,
                                           ctypes.c_uint32, ctypes.c_void_p, ctypes.c_int]
        L.oracle_labels_gather.restype = ctypes.c_int
        L.oracle_time_labels.argtypes = [u8p, u64, u64, u64, ctypes.c_int, ctypes.c_void_p]
        L.oracle_time_labels.restype = ctypes.c_double
        L.oracle_label32.argtypes = [u8p, u64, u64, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p]
        L.oracle_label32.restype = ctypes.c_int
        _lib = L
    return _lib


# ----------------------------------------------------------------------------- python restatement
def py_commitment(node_id: bytes, commitment_atx: bytes) -> bytes:
    import blake3  # third-party wheel, present in this image

    assert len(node_id) == 32 and len(commitment_atx) == 32
    return blake3.blake3(node_id + commitment_atx).digest()


# --- Keccak-512 with the original 0x01 padding (scrypt-jane's SCRYPT_KECCAK512); pad=0x06 is SHA3-512
_KRC = [0x0000000000000001, 0x0000000000008082, 0x800000000000808A, 0x8000000080008000, 0x000000000000808B,
        0x0000000080000001, 0x8000000080008081, 0x8000000000008009, 0x000000000000008A, 0x0000000000000088,
        0x0000000080008009, 0x000000008000000A, 0x000000008000808B, 0x800000000000008B, 0x8000000000008089,
        0x8000000000008003, 0x8000000000008002, 0x8000000000000080, 0x000000000000800A, 0x800000008000000A,
        0x8000000080008081, 0x8000000000008080, 0x0000000080000001, 0x8000000080008008]
_KROT = [[0, 36, 3, 41, 18], [1, 44, 10, 45, 2], [62, 6, 43, 15, 61], [28, 55, 25, 21, 56], [27, 20, 39, 8, 14]]
_M64 = (1 << 64) - 1


def _keccak_f(A):
    for rc in _KRC:
        C = [A[x][0] ^ A[x][1] ^ A[x][2] ^ A[x][3] ^ A[x][4] for x in range(5)]
        D = [C[(x - 1) % 5] ^ (((C[(x + 1) % 5] << 1) | (C[(x + 1) % 5] >> 63)) & _M64) for x in range(5)]
        A = [[A[x][y] ^ D[x] for y in range(5)] for x in range(5)]
        B = [[0] * 5 for _ in range(5)]
        for x in range(5):
            for y in range(5):
                r, v = _KROT[x][y], A[x][y]
                B[y][(2 * x + 3 * y) % 5] = ((v << r) | (v >> (64 - r))) & _M64 if r else v
        A = [[B[x][y] ^ ((~B[(x + 1) % 5][y]) & B[(x + 2) % 5][y]) for y in range(5)] for x in range(5)]
        A[0][0] ^= rc
    return A


def py_keccak512(data: bytes, pad: int = 0x01) -> bytes:
    rate = 72
    m = bytearray(data)
    m.append(pad)
    m.extend(b"\0" * ((-len(m)) % rate))
    m[-1] |= 0x80
    A = [[0] * 5 for _ in range(5)]
    for off in range(0, len(m), rate):
        for i in range(rate // 8):
            A[i % 5][i // 5] ^= int.from_bytes(m[off + 8 * i: off + 8 * i + 8], "little")
        A = _keccak_f(A)
    return b"".join(A[i % 5][i // 5].to_bytes(8, "little") for i in range(8))


def py_hmac_keccak512(key: bytes, msg: bytes) -> bytes:
    bs = 72                                     # HMAC block size = the sponge rate
    if len(key) > bs:
        key = py_keccak512(key)
    key = key.ljust(bs, b"\0")
    return py_keccak512(bytes(k ^ 0x5C for k in key) + py_keccak512(bytes(k ^ 0x36 for k in key) + msg))


def py_pbkdf2_keccak512(pw: bytes, salt: bytes, dklen: int) -> bytes:
    out, i = b"", 1
    while len(out) < dklen:
        out += py_hmac_keccak512(pw, salt + i.to_bytes(4, "big"))
        i += 1
    return out[:dklen]


def _rotl32(x, k):
    return (x << np.uint32(k)) | (x >> np.uint32(32 - k))


def py_chacha20_8(B: np.ndarray) -> np.ndarray:
    """ChaCha20/8 core of scrypt-jane on a batch: B is (n, 16) uint32, the block is the whole state."""
    x = [B[:, i].copy() for i in range(16)]

    def qr(a, b, c, d):
        x[a] += x[b]; x[d] = _rotl32(x[d] ^ x[a], 16)
        x[c] += x[d]; x[b] = _rotl32(x[b] ^ x[c], 12)
        x[a] += x[b]; x[d] = _rotl32(x[d] ^ x[a], 8)
        x[c] += x[d]; x[b] = _rotl32(x[b] ^ x[c], 7)
    for _ in range(4):
        qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15)
        qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14)
    return B + np.stack(x, axis=1)


def _py_blockmix_r1(B):
    y0 = py_chacha20_8(B[:, 16:] ^ B[:, :16])
    y1 = py_chacha20_8(y0 ^ B[:, 16:])
    return np.concatenate([y0, y1], axis=1)


def py_scrypt_jane_batch(pws: list[bytes], salts: list[bytes], n: int, dklen: int = 32) -> list[bytes]:
    """scrypt-jane (ChaCha20/8 + Keccak-512), r = p = 1, for a batch of (password, salt) pairs at once."""
    old = np.seterr(over="ignore")
    try:
        X = np.stack([np.frombuffer(py_pbkdf2_keccak512(p, s, 128), dtype="<u4") for p, s in zip(pws, salts)]).astype(np.uint32)
        m = X.shape[0]
        V = np.empty((n, m, 32), dtype=np.uint32)
        for i in range(n):
            V[i] = X
            X = _py_blockmix_r1(X)
        rows = np.arange(m)
        for i in range(n):
            j = X[:, 16] & np.uint32(n - 1)
            X = _py_blockmix_r1(X ^ V[j, rows])
    finally:
        np.seterr(**old)
    return [py_pbkdf2_keccak512(p, X[i].astype("<u4").tobytes(), dklen) for i, p in enumerate(pws)]


def py_label_password(commitment: bytes, index: int) -> bytes:
    """commitment || LE64(index) || 32 zero bytes: the 72-byte scrypt password of a label (the salt is empty)."""
    assert len(commitment) == 32
    return commitment + int(index).to_bytes(8, "little") + bytes(32)


def py_label32_batch(commitments: list[bytes], indices: list[int], n: int) -> list[bytes]:
    out: list[bytes] = []
    for off in range(0, len(indices), 256):        # 1 MiB of scratch per label at N = 8192
        pws = [py_label_password(c, i) for c, i in zip(commitments[off:off + 256], indices[off:off + 256])]
        out += py_scrypt_jane_batch(pws, [b""] * len(pws), n)
    return out


def py_label32(commitment: bytes, index: int, n: int, r: int = 1, p: int = 1) -> bytes:
    assert r == 1 and p == 1, "the numpy restatement covers the network's r = p = 1 only"
    return py_label32_batch([commitment], [index], n)[0]


def py_labels_range(commitment: bytes, n: int, start: int, count: int) -> bytes:
    return b"".join(l[:16] for l in py_label32_batch([commitment] * count, list(range(start, start + count)), n))


def py_vrf_difficulty(num_labels: int) -> bytes:
    if num_labels <= 1:
        return b"\xff" * 32
    return ((1 << 256) // num_labels).to_bytes(32, "big")


def py_vrf_scan(commitment: bytes, n: int, start: int, count: int, difficulty: bytes):
    best, best_idx = difficulty, None
    for i, l32 in enumerate(py_label32_batch([commitment] * count, list(range(start, start + count)), n)):
        if l32 < best:
            best, best_idx = l32, start + i
    return best_idx, (best if best_idx is not None else None)


# ----------------------------------------------------------------------------- C oracle wrappers
def _buf(b):
    return ctypes.c_char_p(bytes(b))


def c_scrypt(pw: bytes, salt: bytes, n: int, r: int, p: int, dklen: int) -> bytes:
    out = ctypes.create_string_buffer(dklen)
    rc = lib().oracle_scrypt(pw, len(pw), salt, len(salt), n, r, p, out, dklen)
    if rc:
        raise ValueError("oracle_scrypt: bad parameters")
    return out.raw


def c_scrypt_jane(pw: bytes, salt: bytes, n: int, r: int, p: int, dklen: int) -> bytes:
    out = ctypes.create_string_buffer(dklen)
    rc = lib().oracle_scrypt_jane(pw, len(pw), salt, len(salt), n, r, p, out, dklen)
    if rc:
        raise ValueError("oracle_scrypt_jane: bad parameters")
    return out.raw


def c_keccak512(msg: bytes, pad: int = 0x01) -> bytes:
    out = ctypes.create_string_buffer(64)
    lib().oracle_keccak512(msg, ctypes.c_size_t(len(msg)), ctypes.c_uint8(pad), out)
    return out.raw


def c_hmac_keccak512(key: bytes, msg: bytes) -> bytes:
    out = ctypes.create_string_buffer(64)
    lib().oracle_hmac_keccak512(key, ctypes.c_size_t(len(key)), msg, ctypes.c_size_t(len(msg)), out)
    return out.raw


def c_pbkdf2_keccak512(pw: bytes, salt: bytes, dklen: int) -> bytes:
    out = ctypes.create_string_buffer(dklen)
    lib().oracle_pbkdf2_keccak512(pw, ctypes.c_size_t(len(pw)), salt, ctypes.c_size_t(len(salt)), out, ctypes.c_size_t(dklen))
    return out.raw


def c_chacha20_8(block: bytes) -> bytes:
    buf = ctypes.create_string_buffer(block, 64)
    lib().oracle_chacha20_8(buf)
    return buf.raw


def _hash32(fn_name: str, msg: bytes) -> bytes:
    out = ctypes.create_string_buffer(32)
    getattr(lib(), fn_name)(msg, ctypes.c_size_t(len(msg)), out)
    return out.raw


def c_sha256(msg: bytes) -> bytes:
    return _hash32("oracle_sha256", msg)


def c_blake3(msg: bytes, outlen: int = 32) -> bytes:
    out = ctypes.create_string_buffer(outlen)
    lib().oracle_blake3_xof(msg, ctypes.c_size_t(len(msg)), out, ctypes.c_size_t(outlen))
    return out.raw


def c_hmac_sha256(key: bytes, msg: bytes) -> bytes:
    out = ctypes.create_string_buffer(32)
    lib().oracle_hmac_sha256(key, ctypes.c_size_t(len(key)), msg, ctypes.c_size_t(len(msg)), out)
    return out.raw


def c_pbkdf2(pw: bytes, salt: bytes, iters: int, dklen: int) -> bytes:
    out = ctypes.create_string_buffer(dklen)
    lib().oracle_pbkdf2_sha256(pw, ctypes.c_size_t(len(pw)), salt, ctypes.c_size_t(len(salt)),
                               ctypes.c_uint32(iters), out, ctypes.c_size_t(dklen))
    return out.raw


def c_aes128(key: bytes, block: bytes) -> bytes:
    out = ctypes.create_string_buffer(16)
    lib().oracle_aes128_encrypt(key, block, out)
    return out.raw


def c_commitment(node_id: bytes, commitment_atx: bytes) -> bytes:
    out = ctypes.create_string_buffer(32)
    lib().oracle_commitment(node_id, commitment_atx, out)
    return out.raw


def c_vrf_difficulty(num_labels: int) -> bytes:
    out = ctypes.create_string_buffer(32)
    lib().oracle_vrf_difficulty(ctypes.c_uint64(num_labels), out)
    return out.raw


def c_label32(commitment: bytes, index: int, n: int, r: int = 1, p: int = 1) -> bytes:
    out = ctypes.create_string_buffer(32)
    if lib().oracle_label32(commitment, index, n, r, p, out):
        raise ValueError("oracle_label32: bad parameters")
    return out.raw


def default_threads() -> int:
    return len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)


def c_labels_range(commitment: bytes, n: int, start: int, count: int, vrf_difficulty: bytes | None = None,
                   threads: int | None = None):
    """Returns (labels uint8[count,16], found, best_index, best_label32)."""
    out = np.empty((count, 16), dtype=np.uint8)
    found = ctypes.c_int(0)
    best_idx = ctypes.c_uint64(0)
    best = ctypes.create_string_buffer(32)
    rc = lib().oracle_labels_range(commitment, n, 1, 1, start, count, out.ctypes.data,
                                   ctypes.cast(ctypes.c_char_p(vrf_difficulty), ctypes.c_void_p)
                                   if vrf_difficulty is not None else None,
                                   ctypes.byref(found), ctypes.byref(best_idx), best,
                                   threads or default_threads())
    if rc:
        raise ValueError("oracle_labels_range failed")
    if vrf_difficulty is None or not found.value:
        return out, False, None, None
    return out, True, best_idx.value, best.raw


def c_labels_gather(commitments: np.ndarray, indices: np.ndarray, n: int, threads: int | None = None) -> np.ndarray:
    commitments = np.ascontiguousarray(commitments, dtype=np.uint8).reshape(-1, 32)
    indices = np.ascontiguousarray(indices, dtype=np.uint64)
    assert commitments.shape[0] == indices.shape[0]
    out = np.empty((indices.shape[0], 16), dtype=np.uint8)
    rc = lib().oracle_labels_gather(indices.shape[0], commitments.ctypes.data, indices.ctypes.data, n, 1, 1,
                                    out.ctypes.data, threads or default_threads())
    if rc:
        raise ValueError("oracle_labels_gather failed")
    return out


def c_time_labels(commitment: bytes, n: int, start: int, count: int, threads: int) -> float:
    out = np.empty((count, 16), dtype=np.uint8)
    return float(lib().oracle_time_labels(commitment, n, start, count, threads, out.ctypes.data))


# ----------------------------------------------------------------------------- verify-path restatement
# Python restatement of the post-rs v0.7.x proof verifier (ASSUMED conventions, "parity unpinned"): used by
# the tests as the checker of go-spacemesh_b200's batched verifier, and to build synthetic valid proofs.
def py_bits_per_index(num_labels: int) -> int:
    return 0 if num_labels == 0 else int(num_labels).bit_length()          # floor(log2(n)) + 1


def py_proving_difficulty(k1: int, num_labels: int) -> int:
    return min((k1 << 64) // num_labels, (1 << 64) - 1)


def py_pack_indices(indices, bits: int) -> bytes:
    acc = 0
    for i, v in enumerate(indices):
        acc |= (int(v) & ((1 << bits) - 1)) << (i * bits)
    return acc.to_bytes((len(indices) * bits + 7) // 8, "little")


def py_unpack_indices(packed: bytes, bits: int, count: int):
    acc = int.from_bytes(packed, "little")
    return [(acc >> (i * bits)) & ((1 << bits) - 1) for i in range(count)]


def py_cipher_key(challenge: bytes, nonce_group: int, pow_: int, nonce: int | None = None) -> bytes:
    import blake3
    msg = challenge + nonce_group.to_bytes(4, "little") + pow_.to_bytes(8, "little")
    if nonce is not None:
        msg += nonce.to_bytes(4, "little")
    return blake3.blake3(msg).digest()[:16]


def py_aes128(key: bytes, block: bytes) -> bytes:
    from cryptography.hazmat.primitives.ciphers import Cipher, algorithms, modes
    return Cipher(algorithms.AES(key), modes.ECB()).encryptor().update(block)


def py_label_passes(label16: bytes, challenge: bytes, nonce: int, pow_: int, difficulty: int) -> bool:
    ng = nonce // 16
    out = py_aes128(py_cipher_key(challenge, ng, pow_), label16)
    msb, dmsb = out[nonce % 16], difficulty >> 56
    if msb != dmsb:
        return msb < dmsb
    out = py_aes128(py_cipher_key(challenge, ng, pow_, nonce), label16)
    return (int.from_bytes(out[:8], "little") & ((1 << 56) - 1)) < (difficulty & ((1 << 56) - 1))


def py_subset_positions(values, seed: bytes, nonce: int, packed: bytes, pow_: int, k3: int, with_positions: bool = False,
                        stream_bytes: int = 256):
    """RandomValuesIterator: BLAKE3-XOF driven partial Fisher-Yates; returns the first k3 selected values
    (with_positions: pairs (value, position in `values`)).  The XOF stream starts at `stream_bytes` and doubles
    whenever the next draw would run past its end, so any number of draws reads real stream bytes."""
    import blake3
    xof = blake3.blake3(seed + nonce.to_bytes(4, "little") + packed + pow_.to_bytes(8, "little"))
    stream = xof.digest(stream_bytes)
    vals, pos, out, idx = list(values), 0, [], 0
    where = list(range(len(vals)))
    while len(out) < min(k3, len(vals)):
        remaining = len(vals) - idx
        max_allowed = 0xFFFF - 0xFFFF % remaining
        while True:
            while pos + 2 > len(stream):
                stream = xof.digest(max(2 * len(stream), 2))
            r = int.from_bytes(stream[pos:pos + 2], "little")
            pos += 2
            if r < max_allowed:
                break
        vals[idx], vals[idx + r % remaining] = vals[idx + r % remaining], vals[idx]
        where[idx], where[idx + r % remaining] = where[idx + r % remaining], where[idx]
        out.append((vals[idx], where[idx]) if with_positions else vals[idx])
        idx += 1
    return out


def py_verify(nonce: int, packed: bytes, pow_: int, node_id: bytes, atx: bytes, challenge: bytes, num_units: int,
              labels_per_unit: int, k1: int, k2: int, n: int, mode: str = "all", k3: int = 0, seed: bytes = b"",
              selected: int = 0):
    """Returns (ok, position of the failing index in the proof's K2 list or None) — the position is what
    verifying.ErrInvalidIndex carries (activation/handler_v1.go:248, activation/malfeasance.go:165).  Labels come from the C oracle."""
    if not packed:
        raise ValueError("proof indices are empty")
    num_labels = num_units * labels_per_unit
    bits = py_bits_per_index(num_labels)
    if len(packed) != (k2 * bits + 7) // 8:
        raise ValueError("wrong indices length")
    idx = py_unpack_indices(packed, bits, k2)
    where = list(range(k2))
    if mode == "subset":
        pairs = py_subset_positions(idx, seed, nonce, packed, pow_, k3, with_positions=True)
        idx, where = [p[0] for p in pairs], [p[1] for p in pairs]
    elif mode == "selected":
        idx, where = [idx[selected]], [selected]
    c = py_commitment(node_id, atx)
    comms = np.tile(np.frombuffer(c, dtype=np.uint8), (len(idx), 1))
    labels = c_labels_gather(comms, np.array(idx, dtype=np.uint64), n, threads=4)
    diff = py_proving_difficulty(k1, num_labels)
    for w, lab in zip(where, labels):
        if not py_label_passes(lab.tobytes(), challenge, nonce, pow_, diff):
            return False, w
    return True, None


def py_prove(node_id: bytes, atx: bytes, challenge: bytes, num_units: int, labels_per_unit: int, k1: int, k2: int,
             n: int, nonce: int = 0, pow_: int = 0):
    """Scan all labels (small spaces only) and return the packed first-K2 passing indices, or None."""
    num_labels = num_units * labels_per_unit
    c = py_commitment(node_id, atx)
    labels, _, _, _ = c_labels_range(c, n, 0, num_labels, threads=4)
    diff = py_proving_difficulty(k1, num_labels)
    hits = []
    for i in range(num_labels):
        if py_label_passes(labels[i].tobytes(), challenge, nonce, pow_, diff):
            hits.append(i)
            if len(hits) == k2:
                return py_pack_indices(hits, py_bits_per_index(num_labels)), hits
    return None, hits


def py_prove_multi(labels: np.ndarray, challenge: bytes, nonces: int, pows, k1: int, k2: int, num_labels: int):
    """Multi-nonce scan over `labels` (uint8[n,16], label indices 0..n-1) with the product's deterministic
    selection rule: among nonces reaching K2 hits, lowest K2-th hit index wins, ties to the lower nonce.
    Returns (nonce, hits) or (None, None)."""
    diff = py_proving_difficulty(k1, num_labels)
    best = None
    for nonce in range(nonces):
        pow_ = pows[nonce // 16]
        hits = []
        for i in range(len(labels)):
            if py_label_passes(labels[i].tobytes(), challenge, nonce, pow_, diff):
                hits.append(i)
                if len(hits) == k2:
                    break
        if len(hits) == k2 and (best is None or hits[-1] < best[1][-1]):
            best = (nonce, hits)
    return best if best else (None, None)


def np_stored_argmin(stored: np.ndarray):
    """The arg-min of stored 16-byte label prefixes (uint8[n,16]), compared as big-endian 128-bit integers, which is
    how label32 orders.  Returns (the lowest position at the minimum prefix, int64 array of every position holding
    it, ascending).  Array-at-a-time, so 2^24 rows take well under a second."""
    stored = np.ascontiguousarray(stored, dtype=np.uint8).reshape(-1, 16)
    assert len(stored), "np_stored_argmin: no rows"
    words = stored.view(">u8")
    hi = words[:, 0].astype(np.uint64)
    at_hi = np.flatnonzero(hi == hi.min())
    lo = words[at_hi, 1].astype(np.uint64)
    ties = at_hi[lo == lo.min()]
    return int(ties[0]), ties


def _np_aes128_ecb(key: bytes, blocks: np.ndarray) -> np.ndarray:
    from cryptography.hazmat.primitives.ciphers import Cipher, algorithms, modes
    enc = Cipher(algorithms.AES(key), modes.ECB()).encryptor()
    return np.frombuffer(enc.update(blocks.tobytes()) + enc.finalize(), dtype=np.uint8).reshape(-1, 16)


def np_prove_hits(labels: np.ndarray, challenge: bytes, nonces: int, pows, k1: int, k2: int, num_labels: int):
    """{nonce: the first (up to) k2 positions in `labels` (uint8[n,16]) that pass py_label_passes, ascending},
    array-at-a-time: one AES-128-ECB call per nonce group over all labels, and one per nonce over the labels whose
    byte equals the difficulty MSB (the nonce's lazy cipher then compares its low 56 bits, little-endian)."""
    labels = np.ascontiguousarray(labels, dtype=np.uint8).reshape(-1, 16)
    diff = py_proving_difficulty(k1, num_labels)
    msb, lsb = diff >> 56, diff & ((1 << 56) - 1)
    out = {}
    for g in range(nonces // 16):
        ct = _np_aes128_ecb(py_cipher_key(challenge, g, int(pows[g])), labels)
        rows, cols = np.nonzero(ct <= msb)                  # row-major: ascending label position
        keep = ct[rows, cols] != msb
        for b in np.unique(cols[~keep]):
            sel = np.flatnonzero((cols == b) & ~keep)
            lz = _np_aes128_ecb(py_cipher_key(challenge, g, int(pows[g]), 16 * g + int(b)), labels[rows[sel]])
            low56 = lz[:, :8].copy().view("<u8")[:, 0] & np.uint64((1 << 56) - 1)
            keep[sel[low56 < np.uint64(lsb)]] = True
        rows, cols = rows[keep], cols[keep]
        for b in range(16):
            out[16 * g + b] = rows[cols == b][:k2]
    return out


def np_prove_multi(labels: np.ndarray, challenge: bytes, nonces: int, pows, k1: int, k2: int, num_labels: int,
                   first_index: int = 0):
    """py_prove_multi, vectorised, for labels holding indices first_index .. first_index + n - 1: the same
    selection rule (lowest K2-th hit index wins, ties to the lower nonce).  Returns (nonce, [global indices]) or
    (None, None)."""
    best = None
    for nonce, hits in np_prove_hits(labels, challenge, nonces, pows, k1, k2, num_labels).items():   # ascending nonce
        if len(hits) == k2 and (best is None or hits[-1] < best[1][-1]):
            best = (nonce, hits)
    return (best[0], [first_index + int(i) for i in best[1]]) if best else (None, None)
