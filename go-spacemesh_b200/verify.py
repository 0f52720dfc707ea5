"""PostVerifier over libb200post.so — host-side mirror of activation.PostVerifier
(activation/interface.go:26-29, activation/post_verifier.go) for tests and bench.py.

`Verify` is blocking and safe for concurrent use; concurrent calls are coalesced into one GPU batch by the
library's dispatcher.  Errors keep the reference's meaning: `ErrInvalidIndex` (verifying.ErrInvalidIndex,
activation/handler_v1.go:228), "verifier is closed" (post_verifier_test.go:61), "proof indices are empty"
(e2e/validation_test.go:102).  Conventions outside label recomputation are ASSUMED (include/b200post_verify.h).
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass, field

from . import B200PostError, ERR_CLOSED, ERR_EMPTY_PROOF, ERR_INVALID_PROOF, OK, lib

MODE_ALL, MODE_SUBSET, MODE_SELECTED_INDEX = 0, 1, 2


class _Proof(ctypes.Structure):
    _fields_ = [("nonce", ctypes.c_uint32), ("indices", ctypes.c_char_p), ("indices_len", ctypes.c_size_t),
                ("pow", ctypes.c_uint64)]


class _Meta(ctypes.Structure):
    _fields_ = [("node_id", ctypes.c_uint8 * 32), ("commitment_atx_id", ctypes.c_uint8 * 32),
                ("challenge", ctypes.c_uint8 * 32), ("num_units", ctypes.c_uint32), ("labels_per_unit", ctypes.c_uint64)]


class _Params(ctypes.Structure):
    _fields_ = [("k1", ctypes.c_uint32), ("k2", ctypes.c_uint32), ("pow_difficulty", ctypes.c_uint8 * 32),
                ("scrypt_n", ctypes.c_uint64)]


class _Options(ctypes.Structure):
    _fields_ = [("mode", ctypes.c_uint32), ("k3", ctypes.c_uint32), ("seed", ctypes.c_char_p),
                ("seed_len", ctypes.c_size_t), ("selected_index", ctypes.c_uint32), ("prioritized", ctypes.c_uint32)]


POW_VERIFY_FN = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint8,
                                 ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_uint8),
                                 ctypes.POINTER(ctypes.c_uint8))


class _VerifierOpts(ctypes.Structure):
    _fields_ = [("pow_verify", POW_VERIFY_FN), ("pow_ctx", ctypes.c_void_p), ("max_batch_proofs", ctypes.c_uint32),
                ("pow_mode", ctypes.c_uint32), ("pow_cache_key", ctypes.c_char_p), ("pow_cache_key_len", ctypes.c_size_t)]


POW_BUILTIN, POW_CALLBACK, POW_SKIP = 0, 1, 2
POW_INVALID = 2**64 - 1     # invalid_index value when the k2pow, not a label, is what failed


def _verifier_opts(pow, max_batch_proofs: int = 0, pow_cache_key: bytes | None = None):
    """pow: "builtin" (RandomX on the device, the library default), "skip" (explicit opt-out) or a callable
    (pow, nonce_group, challenge8, difficulty32, node_id32) -> 0 if valid."""
    if callable(pow):
        cb = POW_VERIFY_FN(pow)
        return _VerifierOpts(cb, None, max_batch_proofs, POW_CALLBACK, None, 0), cb
    mode = {"builtin": POW_BUILTIN, "skip": POW_SKIP, "callback-missing": POW_CALLBACK}[pow]
    return _VerifierOpts(ctypes.cast(None, POW_VERIFY_FN), None, max_batch_proofs, mode, pow_cache_key,
                         len(pow_cache_key) if pow_cache_key else 0), None


class ErrInvalidIndex(Exception):
    """verifying.ErrInvalidIndex{Index}: Index = position in the proof's K2 index list (POW_INVALID: the k2pow failed)."""
    def __init__(self, index: int):
        super().__init__(f"invalid index: {index}")
        self.index = index


class ErrVerifierClosed(Exception):
    def __init__(self):
        super().__init__("verifier is closed")


class ErrEmptyProof(Exception):
    def __init__(self):
        super().__init__("proof indices are empty")


@dataclass
class Proof:                 # shared.Proof
    nonce: int
    indices: bytes
    pow: int = 0


@dataclass
class ProofMetadata:         # shared.ProofMetadata (activation/validation.go:193-199)
    node_id: bytes
    commitment_atx_id: bytes
    challenge: bytes
    num_units: int
    labels_per_unit: int


@dataclass
class VerifyParams:          # PostConfig.ToConfig() + Scrypt (activation/post.go:40-49,59)
    k1: int
    k2: int
    scrypt_n: int = 8192
    pow_difficulty: bytes = field(default_factory=lambda: b"\xff" * 32)


def _bind():
    L = lib()
    if getattr(L, "_verify_bound", False):
        return L
    vp = ctypes.c_void_p
    L.b200post_verifier_new.argtypes = [ctypes.c_uint32, ctypes.POINTER(_VerifierOpts), ctypes.POINTER(vp)]
    L.b200post_verifier_new_multi.argtypes = [ctypes.POINTER(ctypes.c_uint32), ctypes.c_int, ctypes.POINTER(_VerifierOpts), ctypes.POINTER(vp)]
    L.b200post_verifier_verify.argtypes = [vp, ctypes.POINTER(_Proof), ctypes.POINTER(_Meta), ctypes.POINTER(_Params),
                                           ctypes.POINTER(_Options), ctypes.POINTER(ctypes.c_uint64)]
    L.b200post_verifier_close.argtypes = [vp]
    L.b200post_verifier_free.argtypes = [vp]
    L.b200post_verifier_free.restype = None
    L.b200post_verifier_stats.argtypes = [vp, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint64)]
    L.b200post_verify_batch.argtypes = [ctypes.c_uint32, ctypes.c_size_t, ctypes.POINTER(_Proof), ctypes.POINTER(_Meta),
                                        ctypes.POINTER(_Params), ctypes.POINTER(_Options), ctypes.POINTER(_VerifierOpts),
                                        ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_uint64)]
    L.b200post_verify_batch_multi.argtypes = [ctypes.POINTER(ctypes.c_uint32), ctypes.c_int] + L.b200post_verify_batch.argtypes[1:]
    L.b200post_bits_per_index.argtypes = [ctypes.c_uint64]
    L.b200post_bits_per_index.restype = ctypes.c_uint32
    L.b200post_proving_difficulty.argtypes = [ctypes.c_uint32, ctypes.c_uint64]
    L.b200post_proving_difficulty.restype = ctypes.c_uint64
    L.b200post_pack_indices.argtypes = [ctypes.POINTER(ctypes.c_uint64), ctypes.c_size_t, ctypes.c_uint32, vp, ctypes.c_size_t]
    L.b200post_pack_indices.restype = ctypes.c_size_t
    L.b200post_unpack_indices.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_uint32, ctypes.POINTER(ctypes.c_uint64), ctypes.c_size_t]
    L.b200post_unpack_indices.restype = ctypes.c_size_t
    L._verify_bound = True
    return L


def bits_per_index(num_labels: int) -> int:
    return int(_bind().b200post_bits_per_index(num_labels))


def proving_difficulty(k1: int, num_labels: int) -> int:
    return int(_bind().b200post_proving_difficulty(k1, num_labels))


def pack_indices(indices, bits: int) -> bytes:
    arr = (ctypes.c_uint64 * len(indices))(*[int(v) for v in indices])
    out = ctypes.create_string_buffer((len(indices) * bits + 7) // 8 or 1)
    n = _bind().b200post_pack_indices(arr, len(indices), bits, out, len(out))
    return out.raw[:n]


def unpack_indices(packed: bytes, bits: int, count: int) -> list[int]:
    arr = (ctypes.c_uint64 * max(count, 1))()
    n = _bind().b200post_unpack_indices(packed, len(packed), bits, arr, count)
    return [int(v) for v in arr[:n]]


def _c_proof(p: Proof) -> _Proof:
    return _Proof(p.nonce, p.indices if p.indices else None, len(p.indices), p.pow)


def _c_meta(m: ProofMetadata) -> _Meta:
    c = _Meta()
    ctypes.memmove(c.node_id, m.node_id, 32)
    ctypes.memmove(c.commitment_atx_id, m.commitment_atx_id, 32)
    ctypes.memmove(c.challenge, m.challenge, 32)
    c.num_units, c.labels_per_unit = m.num_units, m.labels_per_unit
    return c


def _c_params(q: VerifyParams) -> _Params:
    c = _Params(k1=q.k1, k2=q.k2, scrypt_n=q.scrypt_n)
    ctypes.memmove(c.pow_difficulty, q.pow_difficulty, 32)
    return c


def _c_options(mode=MODE_ALL, k3=0, seed=b"", selected_index=0, prioritized=False) -> _Options:
    return _Options(mode, k3, seed if seed else None, len(seed), selected_index, int(prioritized))


def _raise(rc: int, bad: int):
    if rc == OK:
        return
    if rc == ERR_INVALID_PROOF:
        raise ErrInvalidIndex(bad)
    if rc == ERR_CLOSED:
        raise ErrVerifierClosed()
    if rc == ERR_EMPTY_PROOF:
        raise ErrEmptyProof()
    raise B200PostError(rc, lib().b200post_last_error().decode(errors="replace"))


class PostVerifier:
    """activation.PostVerifier: Verify(ctx, proof, metadata, opts...) error; Close() error."""

    def __init__(self, provider: int = 0, pow="builtin", max_batch_proofs: int = 0, providers: list[int] | None = None,
                 pow_cache_key: bytes | None = None):
        L = _bind()
        opts, self._cb = _verifier_opts(pow, max_batch_proofs, pow_cache_key)
        self._h = ctypes.c_void_p()
        if providers:     # one dispatcher, a worker per device
            ids = (ctypes.c_uint32 * len(providers))(*providers)
            rc = L.b200post_verifier_new_multi(ids, len(providers), ctypes.byref(opts), ctypes.byref(self._h))
        else:
            rc = L.b200post_verifier_new(provider, ctypes.byref(opts), ctypes.byref(self._h))
        if rc != OK:
            raise B200PostError(rc, L.b200post_last_error().decode(errors="replace"))

    def verify(self, proof: Proof, meta: ProofMetadata, params: VerifyParams, *, mode=MODE_ALL, k3=0, seed=b"",
               selected_index=0, prioritized=False) -> None:
        cp, cm, cq = _c_proof(proof), _c_meta(meta), _c_params(params)
        co = _c_options(mode, k3, seed, selected_index, prioritized)
        bad = ctypes.c_uint64(0)
        rc = _bind().b200post_verifier_verify(self._h, ctypes.byref(cp), ctypes.byref(cm), ctypes.byref(cq),
                                              ctypes.byref(co), ctypes.byref(bad))
        _raise(rc, bad.value)

    def stats(self) -> tuple[int, int]:
        b, p = ctypes.c_uint64(0), ctypes.c_uint64(0)
        _bind().b200post_verifier_stats(self._h, ctypes.byref(b), ctypes.byref(p))
        return int(b.value), int(p.value)

    def close(self) -> None:
        _bind().b200post_verifier_close(self._h)

    def __del__(self):
        try:
            if self._h:
                _bind().b200post_verifier_free(self._h)
                self._h = None
        except Exception:  # noqa: BLE001
            pass


class PreparedBatch:
    """The C structs of a batch, marshalled once (what a Go/C caller holds natively)."""

    def __init__(self, proofs: list[Proof], metas: list[ProofMetadata], params: VerifyParams, options: list[dict] | None = None):
        n = self.n = len(proofs)
        self._keep = proofs                      # the packed index bytes are referenced, not copied
        self.cps = (_Proof * max(n, 1))(*[_c_proof(p) for p in proofs])
        self.cms = (_Meta * max(n, 1))(*[_c_meta(m) for m in metas])
        self.cq = _c_params(params)
        self.cos = (_Options * n)(*[_c_options(**o) for o in options]) if options else None
        self.st = (ctypes.c_int * max(n, 1))()
        self.bad = (ctypes.c_uint64 * max(n, 1))()

    def run(self, provider: int = 0, pow="builtin"):
        opts, _cb = _verifier_opts(pow)
        rc = _bind().b200post_verify_batch(provider, self.n, self.cps, self.cms, ctypes.byref(self.cq), self.cos, ctypes.byref(opts),
                                           self.st, self.bad)
        if rc != OK:
            raise B200PostError(rc, lib().b200post_last_error().decode(errors="replace"))
        return list(self.st[:self.n]), list(self.bad[:self.n])

    def run_multi(self, providers: list[int], pow="builtin"):
        """The batch split over several GPUs (contiguous runs of proofs, one host thread per device)."""
        ids = (ctypes.c_uint32 * len(providers))(*providers)
        opts, _cb = _verifier_opts(pow)
        rc = _bind().b200post_verify_batch_multi(ids, len(providers), self.n, self.cps, self.cms, ctypes.byref(self.cq),
                                                 self.cos, ctypes.byref(opts), self.st, self.bad)
        if rc != OK:
            raise B200PostError(rc, lib().b200post_last_error().decode(errors="replace"))
        return list(self.st[:self.n]), list(self.bad[:self.n])


def verify_batch(proofs: list[Proof], metas: list[ProofMetadata], params: VerifyParams, *, provider: int = 0,
                 providers: list[int] | None = None, options: list[dict] | None = None, pow="builtin"):
    """One synchronous GPU batch (BASELINE.json configs[2]).  Returns (statuses, invalid_indices).  With
    `providers` the batch is split over those devices."""
    batch = PreparedBatch(proofs, metas, params, options)
    return batch.run_multi(providers, pow) if providers else batch.run(provider, pow)
