"""Proof generation over libb200post.so — the AES-scan half of activation.PostClient.Proof
(activation/interface.go:204-207; api/grpcserver/post_client.go:69-143 polls the external post-service for it).

`generate_proof(data_dir, challenge, cfg)` returns (verify.Proof, verify.ProofMetadata) ready for
PostVerifier.verify.  The k2pow (RandomX upstream) is a caller-supplied hook; conventions are ASSUMED
(include/b200post_prove.h)."""
from __future__ import annotations

import ctypes
from dataclasses import dataclass, field

import numpy as np

from . import B200PostError, ERR_NO_DEVICE, OK, lib, providers as _providers
from .setup import PostConfig, _PostConfig, _SumsBlock, _bind as _bind_setup
from .verify import Proof, ProofMetadata, _Meta

POW_PROVE_FN = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_uint8, ctypes.POINTER(ctypes.c_uint8),
                                ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_uint64))


ALL_WINDOWS = 2**32 - 1   # B200POST_PROVE_ALL_WINDOWS: every nonce window below nonce 4096


class _ProveOpts(ctypes.Structure):
    _fields_ = [("provider", ctypes.c_uint32), ("nonces", ctypes.c_uint32), ("chunk_labels", ctypes.c_uint64),
                ("pow_prove", POW_PROVE_FN), ("pow_ctx", ctypes.c_void_p), ("pow_mode", ctypes.c_uint32),
                ("pow_cache_key", ctypes.c_char_p), ("pow_cache_key_len", ctypes.c_size_t),
                ("max_windows", ctypes.c_uint32), ("windows_per_pass", ctypes.c_uint32)]


class _ProofOut(ctypes.Structure):
    _fields_ = [("nonce", ctypes.c_uint32), ("pow", ctypes.c_uint64), ("indices_len", ctypes.c_size_t),
                ("indices", ctypes.c_uint8 * 800), ("labels_scanned", ctypes.c_uint64)]


class _ProveCheck(ctypes.Structure):
    _fields_ = [("labels_rechecked", ctypes.c_uint64), ("damaged", ctypes.c_uint64), ("n_reported", ctypes.c_uint32),
                ("damaged_index", ctypes.c_uint64 * 64), ("proof_verified", ctypes.c_uint32), ("rounds", ctypes.c_uint32)]


@dataclass
class ProveCheck:
    """What generate_proof_checked found: hits rechecked against their recomputed labels, the distinct damaged label
    indices among them (a lower bound on the POST's damage), the lowest 64 of those ascending, whether the proof passed
    the library's verifier, and the recheck rounds run."""
    labels_rechecked: int
    damaged: int
    damaged_index: list = field(default_factory=list)
    proof_verified: bool = False
    rounds: int = 0


class _ProveSumsOpts(ctypes.Structure):
    _fields_ = [("max_heal_blocks", ctypes.c_uint32)]


class _SumsReport(ctypes.Structure):
    _fields_ = [("blocks_checked", ctypes.c_uint64), ("labels_verified", ctypes.c_uint64), ("labels_uncovered", ctypes.c_uint64),
                ("bad_blocks", ctypes.c_uint64), ("healed_blocks", ctypes.c_uint64), ("sidecar_only", ctypes.c_uint64),
                ("n_reported", ctypes.c_uint32), ("reserved", ctypes.c_uint32), ("bad", _SumsBlock * 64)]


@dataclass
class SumsReport:
    """What generate_proof_sums found in the block checksums: digest ranges hashed and compared, labels in ranges that
    matched, labels read without a usable sidecar (all three summed over passes), the distinct bad ranges, those healed
    (recomputed and scanned from the recomputation), the bad ranges whose stored bytes were right (only the sidecar's
    digest was wrong), and the lowest 64 bad ranges as (first label, labels), ascending."""
    blocks_checked: int
    labels_verified: int
    labels_uncovered: int
    bad_blocks: int
    healed_blocks: int
    sidecar_only: int
    bad: list = field(default_factory=list)


class _ProveItem(ctypes.Structure):
    _fields_ = [("data_dir", ctypes.c_char_p), ("challenge", ctypes.c_uint8 * 32), ("status", ctypes.c_int32),
                ("error", ctypes.c_char * 256), ("proof", _ProofOut), ("meta", _Meta), ("check", _ProveCheck)]


@dataclass
class ItemResult:
    """One identity's outcome in generate_proofs: status and error are what the one-identity call returns and sets
    (OK and "" on success); proof, metadata, labels scanned and (checked) the report are set when status is OK, and the
    report also when a checked proof failed later."""
    status: int
    error: str
    proof: Proof | None
    meta: ProofMetadata | None
    labels_scanned: int
    check: ProveCheck | None


def _bind():
    L = lib()
    if getattr(L, "_prove_bound", False):
        return L
    L.b200post_generate_proof.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.POINTER(_PostConfig), ctypes.POINTER(_ProveOpts),
                                          ctypes.POINTER(_ProofOut), ctypes.POINTER(_Meta), ctypes.c_void_p]
    L.b200post_generate_proof_multi.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.POINTER(_PostConfig), ctypes.POINTER(_ProveOpts),
                                                ctypes.POINTER(ctypes.c_uint32), ctypes.c_int, ctypes.POINTER(_ProofOut),
                                                ctypes.POINTER(_Meta), ctypes.c_void_p]
    L.b200post_prove_scan.argtypes = [ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_uint32,
                                      ctypes.POINTER(ctypes.c_uint64), ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint64, ctypes.POINTER(_ProofOut)]
    L.b200post_generate_proof_checked.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.POINTER(_PostConfig), ctypes.POINTER(_ProveOpts),
                                                  ctypes.POINTER(ctypes.c_uint32), ctypes.c_int, ctypes.POINTER(_ProofOut),
                                                  ctypes.POINTER(_Meta), ctypes.POINTER(_ProveCheck), ctypes.c_void_p]
    L.b200post_generate_proof_sums.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.POINTER(_PostConfig), ctypes.POINTER(_ProveOpts),
                                               ctypes.POINTER(ctypes.c_uint32), ctypes.c_int, ctypes.POINTER(_ProveSumsOpts),
                                               ctypes.POINTER(_ProofOut), ctypes.POINTER(_Meta), ctypes.POINTER(_ProveCheck),
                                               ctypes.POINTER(_SumsReport), ctypes.c_void_p]
    L.b200post_generate_proofs.argtypes = [ctypes.POINTER(_ProveItem), ctypes.c_size_t, ctypes.POINTER(_PostConfig),
                                           ctypes.POINTER(_ProveOpts), ctypes.POINTER(ctypes.c_uint32), ctypes.c_int, ctypes.c_uint32,
                                           ctypes.c_uint32, ctypes.c_void_p]
    L._prove_bound = True
    return L


def _c_cfg(cfg: PostConfig) -> _PostConfig:
    c = _PostConfig()
    _bind_setup().b200post_default_post_config(ctypes.byref(c))
    c.min_num_units, c.max_num_units, c.labels_per_unit = cfg.min_num_units, cfg.max_num_units, cfg.labels_per_unit
    c.k1, c.k2, c.k3 = cfg.k1, cfg.k2, cfg.k3
    if getattr(cfg, "pow_difficulty", None) is not None:
        ctypes.memmove(c.pow_difficulty, cfg.pow_difficulty, 32)
    return c


def _err(rc):
    if rc != OK:
        raise B200PostError(rc, lib().b200post_last_error().decode(errors="replace"))


def _opts(provider, providers, nonces, chunk_labels, pow, max_windows=1, windows_per_pass=1):
    if provider is not None and providers is not None:
        raise ValueError("give `provider` or `providers`, not both")
    if isinstance(providers, str):
        if providers != "all":
            raise ValueError(f"providers must be a list of device ids or 'all', not {providers!r}")
        providers = [p["id"] for p in _providers()]
        if not providers:
            raise B200PostError(ERR_NO_DEVICE, "providers='all': libb200post reports no CUDA device")
    if callable(pow):
        cb, mode = POW_PROVE_FN(pow), 1
    else:
        cb, mode = ctypes.cast(None, POW_PROVE_FN), {"builtin": 0, "skip": 2, "callback-missing": 1}[pow]
    if isinstance(max_windows, str):
        if max_windows != "all":
            raise ValueError(f"max_windows must be a count or 'all', not {max_windows!r}")
        max_windows = ALL_WINDOWS
    return _ProveOpts(provider or 0, nonces, chunk_labels, cb, None, mode, None, 0, max_windows, windows_per_pass), providers


def _results(out, meta):
    proof = Proof(int(out.nonce), bytes(out.indices[: out.indices_len]), int(out.pow))
    pm = ProofMetadata(bytes(meta.node_id), bytes(meta.commitment_atx_id), bytes(meta.challenge), int(meta.num_units),
                       int(meta.labels_per_unit))
    return proof, pm, int(out.labels_scanned)


def _report(chk) -> ProveCheck:
    return ProveCheck(int(chk.labels_rechecked), int(chk.damaged), [int(v) for v in chk.damaged_index[: chk.n_reported]],
                      bool(chk.proof_verified), int(chk.rounds))


def generate_proofs(items, cfg: PostConfig, *, providers=(0,), checked: bool = True, parallel_scans: int = 0,
                    nonces: int = 16, chunk_labels: int = 0, pow="builtin", cancel=None, max_windows=1,
                    windows_per_pass: int = 1):
    """Proofs of several identities' POSTs in one call (b200post_generate_proofs): items is a list of (data_dir,
    challenge).  Their k2pow searches share device batches and one identity's scan overlaps the others' searches; each
    result equals generate_proof_checked (checked) or generate_proof(providers=...) for that item alone.
    -> (the call's status, [ItemResult]).  The call's status is OK unless the arguments, the pow mode or the device
    list are refused, or `cancel` was set; an item's own failure is its ItemResult's, not an exception."""
    L = _bind()
    opts, providers = _opts(None, list(providers) if not isinstance(providers, str) else providers, nonces, chunk_labels, pow,
                            max_windows, windows_per_pass)
    arr = (_ProveItem * max(len(items), 1))()
    dirs = [d.encode() if d is not None else None for d, _ in items]   # kept alive for the call
    for a, d, (_, ch) in zip(arr, dirs, items):
        a.data_dir = d
        a.challenge = (ctypes.c_uint8 * 32)(*ch)
    c = _c_cfg(cfg)
    provs = (ctypes.c_uint32 * max(len(providers), 1))(*providers)
    cptr = ctypes.addressof(cancel) if cancel is not None else None
    rc = L.b200post_generate_proofs(arr, len(items), ctypes.byref(c), ctypes.byref(opts), provs if len(providers) else None,
                                    len(providers), int(checked), parallel_scans, cptr)
    out = []
    for a in arr[: len(items)]:
        ok = a.status == OK
        proof, meta, scanned = _results(a.proof, a.meta) if ok else (None, None, 0)
        out.append(ItemResult(int(a.status), a.error.decode(errors="replace"), proof, meta, scanned,
                              _report(a.check) if checked else None))
    return rc, out


def generate_proof_checked(data_dir: str, challenge: bytes, cfg: PostConfig, *, providers=(0,), nonces: int = 16,
                           chunk_labels: int = 0, pow="builtin", cancel=None, max_windows=1, windows_per_pass: int = 1):
    """generate_proof over stored data that may be damaged (b200post_generate_proof_checked): a stored label is a hit
    only when it also equals its recomputed label, so a damaged label never enters the proof, and the proof passes the
    library's verifier before it is returned.  On undamaged data the proof equals generate_proof's.
    Returns (Proof, ProofMetadata, labels scanned, ProveCheck).  A non-empty report is damage in the stored POST data:
    run `b200postcli -verify -fraction 100` to find all of it.  providers: a list of device ids or "all".
    max_windows / windows_per_pass: as for generate_proof; the report covers every pass."""
    L = _bind()
    opts, providers = _opts(None, list(providers) if not isinstance(providers, str) else providers, nonces, chunk_labels, pow,
                            max_windows, windows_per_pass)
    out, meta, chk, c = _ProofOut(), _Meta(), _ProveCheck(), _c_cfg(cfg)
    cptr = ctypes.addressof(cancel) if cancel is not None else None
    arr = (ctypes.c_uint32 * len(providers))(*providers)
    _err(L.b200post_generate_proof_checked(data_dir.encode(), challenge, ctypes.byref(c), ctypes.byref(opts),
                                           arr if len(providers) else None, len(providers), ctypes.byref(out),
                                           ctypes.byref(meta), ctypes.byref(chk), cptr))
    report = ProveCheck(int(chk.labels_rechecked), int(chk.damaged), [int(v) for v in chk.damaged_index[: chk.n_reported]],
                        bool(chk.proof_verified), int(chk.rounds))
    return (*_results(out, meta), report)


def generate_proof_sums(data_dir: str, challenge: bytes, cfg: PostConfig, *, providers=(0,), nonces: int = 16,
                        chunk_labels: int = 0, pow="builtin", cancel=None, max_windows=1, windows_per_pass: int = 1,
                        max_heal_blocks: int = 0):
    """generate_proof_checked with the POST's block checksums (postdata_<N>.sum) in the loop
    (b200post_generate_proof_sums): every covered block the scan reads is hashed on the GPU and compared with its
    checksum; a matching block's hits are usable at once, a damaged block is recomputed and scanned from the
    recomputation, and labels without a usable checksum follow generate_proof_checked's rule.  Where every label read is
    covered the proof is the undamaged POST's.  Nothing in data_dir is written: repair with check_sums(repair=True).
    max_heal_blocks: bad blocks the call may recompute (0 = 1024); past it the call raises ERR_LABEL_MISMATCH.
    Returns (Proof, ProofMetadata, ProveCheck, SumsReport).  A raised B200PostError carries the report as `.sums`."""
    L = _bind()
    opts, providers = _opts(None, list(providers) if not isinstance(providers, str) else providers, nonces, chunk_labels, pow,
                            max_windows, windows_per_pass)
    out, meta, chk, rep, c = _ProofOut(), _Meta(), _ProveCheck(), _SumsReport(), _c_cfg(cfg)
    sopts = _ProveSumsOpts(max_heal_blocks)
    cptr = ctypes.addressof(cancel) if cancel is not None else None
    arr = (ctypes.c_uint32 * max(len(providers), 1))(*providers)
    rc = L.b200post_generate_proof_sums(data_dir.encode(), challenge, ctypes.byref(c), ctypes.byref(opts), arr if len(providers) else None,
                                        len(providers), ctypes.byref(sopts), ctypes.byref(out), ctypes.byref(meta), ctypes.byref(chk),
                                        ctypes.byref(rep), cptr)
    report = SumsReport(int(rep.blocks_checked), int(rep.labels_verified), int(rep.labels_uncovered), int(rep.bad_blocks),
                        int(rep.healed_blocks), int(rep.sidecar_only),
                        [(int(b.first_label), int(b.count)) for b in rep.bad[: rep.n_reported]])
    if rc != OK:
        e = B200PostError(rc, L.b200post_last_error().decode(errors="replace"))
        e.sums = report
        raise e
    proof, pm, _ = _results(out, meta)
    return proof, pm, _report(chk), report


def generate_proof(data_dir: str, challenge: bytes, cfg: PostConfig, *, provider: int | None = None, nonces: int = 16,
                   chunk_labels: int = 0, pow="builtin", providers=None, cancel=None, max_windows=1, windows_per_pass: int = 1):
    """PostClient.Proof(ctx, challenge) -> (Post, PostInfo-like metadata); also returns labels scanned.
    pow: "builtin" (k2pow search on the device, the library default), "skip" (pow = 0, explicit) or a callable
    (ctx, nonce_group, challenge8, difficulty32, node_id32, pow_out) -> 0.
    providers: a list of device ids (repeats allowed) or "all" proves on several devices with the one-device result;
    it replaces `provider` (default 0), and giving both is an error.  cancel: an optional ctypes.c_int, polled per
    chunk.
    max_windows: how many nonce windows [w*nonces, (w+1)*nonces) to try when the first holds no proof (1, a count, or
    "all" = every window below nonce 4096, libpost's loop); windows_per_pass: windows scanned per read of the data.
    The proof is the lowest window's that has one, whatever windows_per_pass; labels scanned adds up over the reads."""
    L = _bind()
    opts, providers = _opts(provider, providers, nonces, chunk_labels, pow, max_windows, windows_per_pass)
    out, meta, c = _ProofOut(), _Meta(), _c_cfg(cfg)
    cptr = ctypes.addressof(cancel) if cancel is not None else None
    if providers is None:
        _err(L.b200post_generate_proof(data_dir.encode(), challenge, ctypes.byref(c), ctypes.byref(opts), ctypes.byref(out),
                                       ctypes.byref(meta), cptr))
    else:
        arr = (ctypes.c_uint32 * len(providers))(*providers)
        _err(L.b200post_generate_proof_multi(data_dir.encode(), challenge, ctypes.byref(c), ctypes.byref(opts),
                                             arr if len(providers) else None, len(providers), ctypes.byref(out),
                                             ctypes.byref(meta), cptr))
    return _results(out, meta)


def prove_scan(labels: np.ndarray, challenge: bytes, nonces: int, pows, k1: int, k2: int, num_labels: int, *,
               first_index: int = 0, provider: int = 0):
    """The scan alone over labels in host memory (uint8[n,16])."""
    labels = np.ascontiguousarray(labels, dtype=np.uint8).reshape(-1, 16)
    arr = (ctypes.c_uint64 * len(pows))(*[int(p) for p in pows])
    out = _ProofOut()
    _err(_bind().b200post_prove_scan(provider, labels.ctypes.data, first_index, labels.shape[0], challenge, nonces, arr, k1, k2,
                                     num_labels, ctypes.byref(out)))
    return int(out.nonce), bytes(out.indices[: out.indices_len]), int(out.pow), int(out.labels_scanned)
