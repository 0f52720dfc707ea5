"""k2pow (RandomX proof of work) — ctypes harness over include/b200post_k2pow.h (test / bench use only; the product is
libb200post.so).  Reference seam: activation/nipost.go:171 (the search, in the external post-service) and
activation/post_verifier.go:150-160 (the check)."""
from __future__ import annotations

import ctypes

import numpy as np

from . import _check, lib

NOT_FOUND = 2**64 - 1
DEFAULT_KEY = b"spacemesh-randomx-cache-key"


class _Params(ctypes.Structure):
    _fields_ = [("cache_key", ctypes.c_char_p), ("cache_key_len", ctypes.c_size_t), ("nonce_group", ctypes.c_uint8),
                ("challenge8", ctypes.c_uint8 * 8), ("node_id", ctypes.c_uint8 * 32), ("difficulty", ctypes.c_uint8 * 32)]


class _Job(ctypes.Structure):
    _fields_ = [("node_id", ctypes.c_uint8 * 32), ("challenge8", ctypes.c_uint8 * 8), ("nonce_group", ctypes.c_uint8),
                ("difficulty", ctypes.c_uint8 * 32)]


_bound = False


def _bind():
    global _bound
    L = lib()
    if not _bound:
        u32, u64, sz, vp = ctypes.c_uint32, ctypes.c_uint64, ctypes.c_size_t, ctypes.c_void_p
        L.b200post_k2pow_scale_difficulty.argtypes = [ctypes.c_char_p, u32, vp]
        L.b200post_k2pow_scale_difficulty.restype = None
        L.b200post_randomx_prepare.argtypes = [u32, ctypes.c_char_p, sz]
        L.b200post_randomx_hash.argtypes = [u32, ctypes.c_char_p, sz, vp, sz, sz, vp]
        L.b200post_k2pow_hashes.argtypes = [u32, ctypes.POINTER(_Params), u64, u64, vp]
        L.b200post_k2pow_search.argtypes = [u32, ctypes.POINTER(_Params), u64, u64, ctypes.POINTER(u64), ctypes.POINTER(u64), vp]
        L.b200post_k2pow_search_multi.argtypes = [ctypes.POINTER(u32), ctypes.c_int, ctypes.POINTER(_Params), u64, u64,
                                                  ctypes.POINTER(u64), ctypes.POINTER(u64), vp]
        L.b200post_k2pow_search_groups.argtypes = [u32, ctypes.POINTER(_Params), u32, u64, vp, ctypes.POINTER(u64), vp]
        L.b200post_k2pow_search_groups_multi.argtypes = [ctypes.POINTER(u32), ctypes.c_int, ctypes.POINTER(_Params), u32, u64, vp,
                                                         ctypes.POINTER(u64), vp]
        L.b200post_k2pow_search_group_range.argtypes = [u32, ctypes.POINTER(_Params), u32, u32, u64, vp, ctypes.POINTER(u64), vp]
        L.b200post_k2pow_search_group_range_multi.argtypes = [ctypes.POINTER(u32), ctypes.c_int, ctypes.POINTER(_Params), u32, u32,
                                                              u64, vp, ctypes.POINTER(u64), vp]
        L.b200post_k2pow_search_jobs.argtypes = [ctypes.POINTER(u32), ctypes.c_int, ctypes.c_char_p, sz, sz, ctypes.POINTER(_Job), u64,
                                                 vp, ctypes.POINTER(u64), vp]
        L.b200post_k2pow_verify.argtypes = [u32, ctypes.POINTER(_Params), u64, ctypes.POINTER(ctypes.c_int)]
        L.b200post_randomx_dataset_read.argtypes = [u32, ctypes.c_char_p, sz, u64, u64, vp]
        L.b200post_randomx_last_timing.argtypes = [u32, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double),
                                                   ctypes.POINTER(u64), ctypes.POINTER(u64)]
        L.b200post_randomx_batch_size.argtypes = [u32, ctypes.POINTER(u64)]
        _bound = True
    return L


def _params(nonce_group: int, challenge8: bytes, node_id: bytes, difficulty: bytes | None, key: bytes | None) -> _Params:
    p = _Params()
    p.cache_key = key
    p.cache_key_len = len(key) if key is not None else 0
    p.nonce_group = nonce_group
    p.challenge8 = (ctypes.c_uint8 * 8)(*challenge8[:8])
    p.node_id = (ctypes.c_uint8 * 32)(*node_id)
    p.difficulty = (ctypes.c_uint8 * 32)(*(difficulty or b"\x00" * 32))
    return p


def scale_difficulty(pow_difficulty: bytes, num_units: int) -> bytes:
    out = ctypes.create_string_buffer(32)
    _bind().b200post_k2pow_scale_difficulty(pow_difficulty, num_units, out)
    return out.raw


def prepare(key: bytes | None = None, *, provider: int = 0) -> None:
    _check(_bind().b200post_randomx_prepare(provider, key, len(key) if key is not None else 0))


def randomx_hash(key: bytes | None, inputs: list[bytes], *, provider: int = 0) -> list[bytes]:
    """RandomX hashes of equally long inputs through the GPU engine."""
    n = len(inputs)
    ln = len(inputs[0]) if n else 0
    assert all(len(i) == ln for i in inputs)
    buf = np.frombuffer(b"".join(inputs), dtype=np.uint8) if n * ln else np.zeros(1, dtype=np.uint8)
    out = np.zeros((n, 32), dtype=np.uint8)
    _check(_bind().b200post_randomx_hash(provider, key, len(key) if key is not None else 0, buf.ctypes.data, ln, n, out.ctypes.data))
    return [bytes(r) for r in out]


def hashes(nonce_group: int, challenge8: bytes, node_id: bytes, start: int, count: int, *, key: bytes | None = None,
           provider: int = 0) -> np.ndarray:
    p = _params(nonce_group, challenge8, node_id, None, key)
    out = np.zeros((count, 32), dtype=np.uint8)
    _check(_bind().b200post_k2pow_hashes(provider, ctypes.byref(p), start, count, out.ctypes.data))
    return out


def search(nonce_group: int, challenge8: bytes, node_id: bytes, difficulty: bytes, start: int, count: int, *,
           key: bytes | None = None, provider: int = 0, providers: list[int] | None = None, cancel=None):
    """-> (found pow or None, hashes computed)."""
    p = _params(nonce_group, challenge8, node_id, difficulty, key)
    found, done = ctypes.c_uint64(0), ctypes.c_uint64(0)
    cptr = ctypes.addressof(cancel) if cancel is not None else None
    if providers is not None:
        arr = (ctypes.c_uint32 * len(providers))(*providers)
        _check(_bind().b200post_k2pow_search_multi(arr, len(providers), ctypes.byref(p), start, count, ctypes.byref(found),
                                                  ctypes.byref(done), cptr))
    else:
        _check(_bind().b200post_k2pow_search(provider, ctypes.byref(p), start, count, ctypes.byref(found), ctypes.byref(done), cptr))
    return (None if found.value == NOT_FOUND else found.value), done.value


def search_groups(challenge8: bytes, node_id: bytes, difficulty: bytes, n_groups: int, max_nonces_per_group: int = 0, *,
                  key: bytes | None = None, provider: int = 0, providers: list[int] | None = None, cancel=None):
    """The prover's search: the smallest valid pow of each nonce group 0..n_groups-1 (None where there is none below
    max_nonces_per_group; 0 = the whole nonce space).  providers: several devices (repeats allowed), same pows.
    -> (pows, hashes computed)."""
    p = _params(0, challenge8, node_id, difficulty, key)
    pows = np.zeros(max(n_groups, 1), dtype=np.uint64)
    done = ctypes.c_uint64(0)
    cptr = ctypes.addressof(cancel) if cancel is not None else None
    if providers is not None:
        arr = (ctypes.c_uint32 * len(providers))(*providers)
        _check(_bind().b200post_k2pow_search_groups_multi(arr if len(providers) else None, len(providers), ctypes.byref(p),
                                                          n_groups, max_nonces_per_group, pows.ctypes.data, ctypes.byref(done),
                                                          cptr))
    else:
        _check(_bind().b200post_k2pow_search_groups(provider, ctypes.byref(p), n_groups, max_nonces_per_group,
                                                    pows.ctypes.data, ctypes.byref(done), cptr))
    pows = pows[:n_groups]
    return [None if int(v) == NOT_FOUND else int(v) for v in pows], done.value


def search_group_range(challenge8: bytes, node_id: bytes, difficulty: bytes, first_group: int, n_groups: int,
                       max_nonces_per_group: int = 0, *, key: bytes | None = None, provider: int = 0,
                       providers: list[int] | None = None, cancel=None):
    """search_groups for the groups first_group .. first_group + n_groups - 1 (first_group + n_groups <= 256): the pows
    of a pass of nonce windows.  -> (pows, hashes computed), pows[i] being group first_group + i's."""
    p = _params(0, challenge8, node_id, difficulty, key)
    pows = np.zeros(max(n_groups, 1), dtype=np.uint64)
    done = ctypes.c_uint64(0)
    cptr = ctypes.addressof(cancel) if cancel is not None else None
    if providers is not None:
        arr = (ctypes.c_uint32 * len(providers))(*providers)
        _check(_bind().b200post_k2pow_search_group_range_multi(arr if len(providers) else None, len(providers), ctypes.byref(p),
                                                               first_group, n_groups, max_nonces_per_group, pows.ctypes.data,
                                                               ctypes.byref(done), cptr))
    else:
        _check(_bind().b200post_k2pow_search_group_range(provider, ctypes.byref(p), first_group, n_groups, max_nonces_per_group,
                                                         pows.ctypes.data, ctypes.byref(done), cptr))
    return [None if int(v) == NOT_FOUND else int(v) for v in pows[:n_groups]], done.value


def search_jobs(jobs, max_nonces_per_job: int = 0, *, key: bytes | None = None, providers=(0,), cancel=None):
    """Several identities' k2pows in one search sharing device batches (b200post_k2pow_search_jobs).  jobs: a list of
    (node_id, challenge8, nonce_group, difficulty) with the difficulty already scaled by the identity's num_units.
    -> (pows, hashes computed), pows[j] being job j's smallest valid pow below max_nonces_per_job (0 = the whole nonce
    space) or None."""
    arr = (_Job * max(len(jobs), 1))()
    for a, (node_id, challenge8, group, difficulty) in zip(arr, jobs):
        a.node_id = (ctypes.c_uint8 * 32)(*node_id)
        a.challenge8 = (ctypes.c_uint8 * 8)(*challenge8[:8])
        a.nonce_group = group
        a.difficulty = (ctypes.c_uint8 * 32)(*difficulty)
    pows = np.zeros(max(len(jobs), 1), dtype=np.uint64)
    done = ctypes.c_uint64(0)
    provs = (ctypes.c_uint32 * max(len(providers), 1))(*providers)
    _check(_bind().b200post_k2pow_search_jobs(provs if len(providers) else None, len(providers), key, len(key) if key is not None else 0,
                                              len(jobs), arr, max_nonces_per_job, pows.ctypes.data, ctypes.byref(done),
                                              ctypes.addressof(cancel) if cancel is not None else None))
    return [None if int(v) == NOT_FOUND else int(v) for v in pows[:len(jobs)]], done.value


def dataset(first: int, count: int, key: bytes | None = None, *, provider: int = 0) -> np.ndarray:
    """RandomX dataset items first..first+count-1 of `key` as resident on the device: (count, 8) uint64."""
    out = np.zeros((count, 8), dtype=np.uint64)
    _check(_bind().b200post_randomx_dataset_read(provider, key, len(key) if key is not None else 0, first, count,
                                                 out.ctypes.data))
    return out


def verify(pow_: int, nonce_group: int, challenge8: bytes, node_id: bytes, difficulty: bytes, *, key: bytes | None = None,
           provider: int = 0) -> bool:
    p = _params(nonce_group, challenge8, node_id, difficulty, key)
    ok = ctypes.c_int(0)
    _check(_bind().b200post_k2pow_verify(provider, ctypes.byref(p), pow_, ctypes.byref(ok)))
    return bool(ok.value)


def last_timing(provider: int = 0) -> dict:
    t, v = ctypes.c_double(0), ctypes.c_double(0)
    h, l = ctypes.c_uint64(0), ctypes.c_uint64(0)
    _check(_bind().b200post_randomx_last_timing(provider, ctypes.byref(t), ctypes.byref(v), ctypes.byref(h), ctypes.byref(l)))
    return {"total_ms": t.value, "vm_kernel_ms": v.value, "hashes": h.value, "vm_launches": l.value}


def batch_size(provider: int = 0) -> int:
    v = ctypes.c_uint64(0)
    _check(_bind().b200post_randomx_batch_size(provider, ctypes.byref(v)))
    return v.value
