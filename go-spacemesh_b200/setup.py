"""PostSetupManager over libb200post.so — host-side mirror of activation.PostSetupManager
(activation/post.go:185-449; interface postSetupProvider, activation/interface.go:114-119) for tests/tools.

Method names and the state machine are the reference's: prepare_initializer / start_session / status / reset,
states NotStarted(1) .. Error(6).  The state machine itself lives in C++ (csrc/setup.cu); this is ctypes glue.
"""
from __future__ import annotations

import ctypes
import functools
from dataclasses import dataclass

from . import B200PostError, ERR_CANCELLED, OK, VrfNonce, lib

(STATE_NOT_STARTED, STATE_PREPARED, STATE_IN_PROGRESS, STATE_STOPPED, STATE_COMPLETE, STATE_ERROR) = range(1, 7)
ERR_STATE, ERR_NO_PROVIDER, ERR_IO, ERR_LABEL_MISMATCH, ERR_CONFIG_MISMATCH = 10, 11, 12, 13, 14
PROVIDER_UNSET, PROVIDER_ALL = -1, -2


class _PostConfig(ctypes.Structure):
    _fields_ = [("min_num_units", ctypes.c_uint32), ("max_num_units", ctypes.c_uint32), ("labels_per_unit", ctypes.c_uint64),
                ("k1", ctypes.c_uint32), ("k2", ctypes.c_uint32), ("k3", ctypes.c_uint32), ("pow_difficulty", ctypes.c_uint8 * 32)]


class _SetupOpts(ctypes.Structure):
    _fields_ = [("data_dir", ctypes.c_char_p), ("num_units", ctypes.c_uint32), ("max_file_size", ctypes.c_uint64),
                ("provider_id", ctypes.c_int64), ("scrypt_n", ctypes.c_uint64), ("scrypt_r", ctypes.c_uint64),
                ("scrypt_p", ctypes.c_uint64), ("compute_batch_size", ctypes.c_uint64), ("self_check_every", ctypes.c_uint32)]


class _Status(ctypes.Structure):
    _fields_ = [("state", ctypes.c_int32), ("num_labels_written", ctypes.c_uint64)]


class _Metadata(ctypes.Structure):
    _fields_ = [("node_id", ctypes.c_uint8 * 32), ("commitment_atx_id", ctypes.c_uint8 * 32), ("labels_per_unit", ctypes.c_uint64),
                ("num_units", ctypes.c_uint32), ("max_file_size", ctypes.c_uint64), ("scrypt_n", ctypes.c_uint64),
                ("scrypt_r", ctypes.c_uint64), ("scrypt_p", ctypes.c_uint64), ("has_nonce", ctypes.c_uint32),
                ("nonce", ctypes.c_uint64), ("nonce_value", ctypes.c_uint8 * 32), ("last_position", ctypes.c_uint64),
                ("vrf_scan_pending", ctypes.c_uint32)]


class _VerifyPosOpts(ctypes.Structure):
    _fields_ = [("provider_id", ctypes.c_int64), ("fraction", ctypes.c_double), ("from_file", ctypes.c_uint64),
                ("to_file", ctypes.c_int64), ("seed", ctypes.c_uint64), ("progress", ctypes.c_void_p)]


class _VerifyPosResult(ctypes.Structure):
    _fields_ = [("files_checked", ctypes.c_uint64), ("labels_checked", ctypes.c_uint64), ("mismatches", ctypes.c_uint64),
                ("seed", ctypes.c_uint64), ("nonce_ok", ctypes.c_uint32), ("argmin_checked", ctypes.c_uint32),
                ("argmin_ok", ctypes.c_uint32), ("n_reported", ctypes.c_uint32), ("bad_index", ctypes.c_uint64 * 64)]


class _VrfSearchOpts(ctypes.Structure):
    _fields_ = [("provider_id", ctypes.c_int64), ("compute_batch_size", ctypes.c_uint64), ("chunk_labels", ctypes.c_uint64),
                ("progress", ctypes.c_void_p)]


class _SumsOpts(ctypes.Structure):
    _fields_ = [("provider_id", ctypes.c_int64), ("from_file", ctypes.c_uint64), ("to_file", ctypes.c_int64),
                ("progress", ctypes.c_void_p), ("repair", ctypes.c_uint32)]


class _SumsBlock(ctypes.Structure):
    _fields_ = [("first_label", ctypes.c_uint64), ("count", ctypes.c_uint64)]


class _SumsResult(ctypes.Structure):
    _fields_ = [("files_checked", ctypes.c_uint64), ("files_unchecked", ctypes.c_uint64), ("labels_checked", ctypes.c_uint64),
                ("labels_unchecked", ctypes.c_uint64), ("bytes_read", ctypes.c_uint64), ("blocks_checked", ctypes.c_uint64),
                ("bad_blocks", ctypes.c_uint64), ("repaired_blocks", ctypes.c_uint64), ("n_reported", ctypes.c_uint32),
                ("reserved", ctypes.c_uint32), ("bad", _SumsBlock * 64)]


class _MergeOpts(ctypes.Structure):
    _fields_ = [("provider_id", ctypes.c_int64), ("compute_batch_size", ctypes.c_uint64)]


@functools.lru_cache(maxsize=None)
def _merge_result_type():
    from . import prove   # imports this module: the proof struct is bound on first use
    return type("_MergeResult", (ctypes.Structure,), {"_fields_": [
        ("ranges", ctypes.c_uint32), ("nonce", VrfNonce), ("past_end", ctypes.c_uint32), ("proof_rc", ctypes.c_int32),
        ("proof_reason", ctypes.c_char * 256), ("proof", prove._ProofOut)]})


@dataclass
class MergeResult:           # b200post_merge_result
    ranges: int              # records merged
    nonce: int               # the VRF nonce the metadata now holds
    nonce_value: bytes       # its label32
    past_end: bool           # no label was below the threshold: the past-the-end search found the nonce
    proof_rc: int            # OK: initial_post.json written; ERR_INVALID_PROOF or ERR_STATE: no initial proof
    proof_reason: str        # why there is none
    proof: object = None     # the Proof written to initial_post.json, or None


@dataclass
class VerifyPosResult:       # b200post_verify_pos_result; `code` is the call's status (OK, ERR_LABEL_MISMATCH, ERR_CANCELLED)
    code: int
    files_checked: int
    labels_checked: int
    mismatches: int
    seed: int
    nonce_ok: bool
    argmin_checked: bool
    argmin_ok: bool
    bad_index: list[int]


@dataclass
class SumsResult:            # b200post_sums_result; `code` is the call's status (OK, ERR_LABEL_MISMATCH, ERR_STATE, ERR_CANCELLED)
    code: int
    files_checked: int       # check: files with a usable sidecar; write_sums: files given one
    files_unchecked: int     # check: files without one; write_sums: files with a mismatch (no sidecar)
    labels_checked: int
    labels_unchecked: int
    bytes_read: int
    blocks_checked: int
    bad_blocks: int
    repaired_blocks: int
    bad: list[tuple[int, int]]   # the lowest bad blocks: (first global label, label count), ascending


SUM_BLOCK_LABELS = 1 << 16   # labels per checksummed block (1 MiB)


@dataclass
class PostConfig:            # activation/post.go:27-38
    min_num_units: int = 1
    max_num_units: int = 10
    labels_per_unit: int = 512
    k1: int = 26
    k2: int = 37
    k3: int = 37
    pow_difficulty: bytes | None = None   # None = the library default (config/mainnet.go:41's prefix)


@dataclass
class PostSetupOpts:         # activation/post.go:53-61
    data_dir: str = ""
    num_units: int = 2
    max_file_size: int = 4 << 30
    provider_id: int | None = None
    scrypt_n: int = 8192
    scrypt_r: int = 1
    scrypt_p: int = 1
    compute_batch_size: int = 1 << 20
    self_check_every: int = 16


@dataclass
class PostSetupStatus:       # activation/post.go:121-125
    state: int
    num_labels_written: int


def _bind():
    L = lib()
    if getattr(L, "_setup_bound", False):
        return L
    vp = ctypes.c_void_p
    L.b200post_setup_manager_new.argtypes = [ctypes.POINTER(_PostConfig), ctypes.POINTER(vp)]
    L.b200post_setup_manager_free.argtypes = [vp]
    L.b200post_setup_manager_free.restype = None
    L.b200post_setup_prepare_initializer.argtypes = [vp, ctypes.POINTER(_SetupOpts), ctypes.c_char_p, ctypes.c_char_p]
    L.b200post_setup_start_session.argtypes = [vp, vp]
    L.b200post_setup_get_status.argtypes = [vp, ctypes.POINTER(_Status)]
    L.b200post_setup_reset.argtypes = [vp]
    L.b200post_setup_commitment_atx.argtypes = [vp, vp]
    L.b200post_load_metadata.argtypes = [ctypes.c_char_p, ctypes.POINTER(_Metadata)]
    L.b200post_default_post_config.argtypes = [ctypes.POINTER(_PostConfig)]
    L.b200post_default_post_config.restype = None
    L.b200post_verify_pos.argtypes = [ctypes.c_char_p, ctypes.POINTER(_VerifyPosOpts), ctypes.POINTER(_VerifyPosResult), vp]
    L.b200post_verify_pos_sample.argtypes = [ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_double, vp,
                                             ctypes.c_uint64, ctypes.POINTER(ctypes.c_uint64)]
    L.b200post_setup_prepare_files.argtypes = [vp, ctypes.POINTER(_SetupOpts), ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint64,
                                               ctypes.c_int64]
    L.b200post_search_vrf_nonce.argtypes = [ctypes.c_char_p, ctypes.POINTER(_VrfSearchOpts), ctypes.POINTER(VrfNonce), vp]
    L.b200post_setup_request_initial_proof.argtypes = [vp, vp]
    L.b200post_setup_initial_proof.argtypes = [vp, vp, vp]
    L.b200post_load_initial_proof.argtypes = [ctypes.c_char_p, ctypes.POINTER(_PostConfig), ctypes.c_uint32, vp, vp]
    L.b200post_setup_request_range_record.argtypes = [vp, vp]
    L.b200post_merge_range_records.argtypes = [ctypes.c_char_p, vp, ctypes.POINTER(_MergeOpts), vp, vp]
    L.b200post_label_block_digests.argtypes = [ctypes.c_uint32, vp, ctypes.c_uint64, vp]
    L.b200post_setup_request_checksums.argtypes = [vp]
    L.b200post_check_sums.argtypes = [ctypes.c_char_p, ctypes.POINTER(_SumsOpts), ctypes.POINTER(_SumsResult), vp]
    L.b200post_write_sums.argtypes = [ctypes.c_char_p, ctypes.POINTER(_SumsOpts), ctypes.POINTER(_SumsResult), vp]
    L._setup_bound = True
    return L


def _err(rc: int):
    if rc != OK:
        raise B200PostError(rc, lib().b200post_last_error().decode(errors="replace"))


def load_metadata(data_dir: str) -> dict:
    """initialization.LoadMetadata."""
    m = _Metadata()
    _err(_bind().b200post_load_metadata(data_dir.encode(), ctypes.byref(m)))
    return dict(node_id=bytes(m.node_id), commitment_atx_id=bytes(m.commitment_atx_id), labels_per_unit=m.labels_per_unit,
                num_units=m.num_units, max_file_size=m.max_file_size, scrypt_n=m.scrypt_n,
                nonce=int(m.nonce) if m.has_nonce else None, nonce_value=bytes(m.nonce_value) if m.has_nonce else None,
                last_position=m.last_position, vrf_scan_pending=m.vrf_scan_pending)


def search_vrf_nonce(data_dir: str, *, provider_id: int = 0, compute_batch_size: int = 0, chunk_labels: int = 0,
                     progress: ctypes.c_uint64 | None = None, cancel: ctypes.c_int | None = None) -> tuple[int, bytes]:
    """postcli -searchForNonce: the VRF nonce of the complete POST in data_dir from its stored labels, written to the
    metadata as a single uninterrupted init would have written it.  Returns (nonce, label32); raises B200PostError
    (ERR_LABEL_MISMATCH for damaged data, the index in its text; ERR_IO for missing data; ERR_CANCELLED)."""
    o = _VrfSearchOpts(provider_id, compute_batch_size, chunk_labels, ctypes.addressof(progress) if progress is not None else None)
    out = VrfNonce()
    _err(_bind().b200post_search_vrf_nonce(data_dir.encode(), ctypes.byref(o), ctypes.byref(out),
                                           ctypes.addressof(cancel) if cancel is not None else None))
    return int(out.index), bytes(out.label32)


def verify_pos(data_dir: str, *, fraction: float = 0.2, provider_id: int = 0, from_file: int = 0, to_file: int = -1,
               seed: int = 0, progress: ctypes.c_uint64 | None = None, cancel: ctypes.c_int | None = None) -> VerifyPosResult:
    """postcli -verify: recompute `fraction` percent of each file's labels on the GPU and compare them with the stored
    bytes.  Returns the result for OK, ERR_LABEL_MISMATCH (data invalid), ERR_STATE (labels fine, but the metadata has no
    VRF nonce: initialisation has not finished) and ERR_CANCELLED; raises on other errors."""
    o = _VerifyPosOpts(provider_id, fraction, from_file, to_file, seed,
                       ctypes.addressof(progress) if progress is not None else None)
    r = _VerifyPosResult()
    rc = _bind().b200post_verify_pos(data_dir.encode(), ctypes.byref(o), ctypes.byref(r),
                                     ctypes.addressof(cancel) if cancel is not None else None)
    if rc not in (OK, ERR_LABEL_MISMATCH, ERR_STATE, ERR_CANCELLED):
        _err(rc)
    return VerifyPosResult(rc, r.files_checked, r.labels_checked, r.mismatches, r.seed, bool(r.nonce_ok), bool(r.argmin_checked),
                           bool(r.argmin_ok), [int(r.bad_index[i]) for i in range(r.n_reported)])


def label_block_digests(labels, provider_id: int = 0):
    """BLAKE3 digests of labels (bytes or a uint8 array of n x 16 bytes) in blocks of SUM_BLOCK_LABELS from the first,
    the last one possibly short, hashed on CUDA ordinal provider_id: an (ceil(n / 2^16), 32) uint8 array."""
    import numpy as np
    a = np.ascontiguousarray(np.frombuffer(labels, dtype=np.uint8) if isinstance(labels, (bytes, bytearray)) else labels, dtype=np.uint8).reshape(-1)
    if a.size % 16:
        raise ValueError("labels are 16 bytes each")
    n = a.size // 16
    out = np.empty(((n + SUM_BLOCK_LABELS - 1) // SUM_BLOCK_LABELS, 32), dtype=np.uint8)
    _err(_bind().b200post_label_block_digests(provider_id, a.ctypes.data, n, out.ctypes.data))
    return out


def _sums_call(fn, data_dir, provider_id, from_file, to_file, repair, progress, cancel) -> SumsResult:
    o = _SumsOpts(provider_id, from_file, to_file, ctypes.addressof(progress) if progress is not None else None, int(repair))
    r = _SumsResult()
    rc = fn(data_dir.encode(), ctypes.byref(o), ctypes.byref(r), ctypes.addressof(cancel) if cancel is not None else None)
    if rc not in (OK, ERR_LABEL_MISMATCH, ERR_STATE, ERR_CANCELLED) or (rc == ERR_STATE and r.labels_checked == 0):
        _err(rc)
    return SumsResult(rc, r.files_checked, r.files_unchecked, r.labels_checked, r.labels_unchecked, r.bytes_read, r.blocks_checked,
                      r.bad_blocks, r.repaired_blocks, [(int(r.bad[i].first_label), int(r.bad[i].count)) for i in range(r.n_reported)])


def check_sums(data_dir: str, *, provider_id: int = 0, from_file: int = 0, to_file: int = -1, repair: bool = False,
               progress: ctypes.c_uint64 | None = None, cancel: ctypes.c_int | None = None) -> SumsResult:
    """b200postcli -checkSums: read the covered labels of files [from_file, to_file], hash them on the GPU and compare
    every 1 MiB block with its postdata_<N>.sum.  repair=True rewrites each bad block from its recomputation once that
    matches the checksum.  Returns the result for OK, ERR_LABEL_MISMATCH (bad blocks left), ERR_STATE (labels without a
    checksum) and ERR_CANCELLED; raises on other errors, and on ERR_STATE "no checksums" when nothing is covered."""
    return _sums_call(_bind().b200post_check_sums, data_dir, provider_id, from_file, to_file, repair, progress, cancel)


def write_sums(data_dir: str, *, provider_id: int = 0, from_file: int = 0, to_file: int = -1,
               progress: ctypes.c_uint64 | None = None, cancel: ctypes.c_int | None = None) -> SumsResult:
    """b200postcli -verify -fraction 100 -writeSums: the full check of verify_pos over files [from_file, to_file]; every
    file whose labels all match gets its postdata_<N>.sum from the verified bytes.  Returns the result for OK,
    ERR_LABEL_MISMATCH (files with a mismatch got none) and ERR_CANCELLED; raises on other errors."""
    return _sums_call(_bind().b200post_write_sums, data_dir, provider_id, from_file, to_file, False, progress, cancel)


def load_initial_proof(data_dir: str, cfg: PostConfig, nonces: int = 16):
    """The post-service side of the initial proof: the proof a setup session stored in data_dir/initial_post.json, if
    it answers the zero challenge for this POST, cfg (K1, K2, pow difficulty) and nonce count.  Returns
    (Proof, ProofMetadata, labels scanned) as prove.generate_proof does; raises B200PostError ERR_IO ("no initial proof")
    when it is absent or stale, and the caller then proves from the stored data."""
    from . import prove
    from .verify import _Meta
    out, meta = prove._ProofOut(), _Meta()
    _err(_bind().b200post_load_initial_proof(data_dir.encode(), ctypes.byref(prove._c_cfg(cfg)), nonces, ctypes.byref(out),
                                             ctypes.byref(meta)))
    return prove._results(out, meta)


def merge_range_records(data_dir: str, cfg: PostConfig, *, provider_id: int = 0, compute_batch_size: int = 0,
                        cancel: ctypes.c_int | None = None) -> MergeResult:
    """b200postcli -mergeRanges: the VRF nonce and initial proof of a POST whose files were written by range sessions
    with records (request_range_record), from the range_*.rec files in data_dir and without reading a stored label.
    The nonce is written to the metadata and the proof (when every record carries a common proof scan and it yields one)
    to initial_post.json, as one full session with the initial proof would have written them.  cfg gives K1, K2 and the
    pow difficulty; compute_batch_size the past-the-end batch (0 = 2^20).  Raises B200PostError when the records do not
    tile the POST, are damaged or foreign, or the data is incomplete (the metadata is then untouched)."""
    from . import prove
    o = _MergeOpts(provider_id, compute_batch_size)
    r = _merge_result_type()()
    _err(_bind().b200post_merge_range_records(data_dir.encode(), ctypes.byref(prove._c_cfg(cfg)), ctypes.byref(o), ctypes.byref(r),
                                              ctypes.addressof(cancel) if cancel is not None else None))
    proof = prove._results(r.proof, _zero_meta())[0] if r.proof_rc == OK else None
    return MergeResult(int(r.ranges), int(r.nonce.index), bytes(r.nonce.label32), bool(r.past_end), int(r.proof_rc),
                       r.proof_reason.decode(errors="replace"), proof)


def _zero_meta():
    from .verify import _Meta
    return _Meta()


def verify_pos_sample(seed: int, file: int, labels_in_file: int, fraction: float):
    """The positions (within the file, ascending, numpy uint64) that verify_pos checks for this seed and file."""
    import numpy as np
    L = _bind()
    n = ctypes.c_uint64()
    _err(L.b200post_verify_pos_sample(seed, file, labels_in_file, fraction, None, 0, ctypes.byref(n)))
    out = np.empty(n.value, dtype=np.uint64)
    _err(L.b200post_verify_pos_sample(seed, file, labels_in_file, fraction, out.ctypes.data, n.value, ctypes.byref(n)))
    return out


def _c_opts(opts: PostSetupOpts) -> _SetupOpts:
    return _SetupOpts(opts.data_dir.encode(), opts.num_units, opts.max_file_size,
                      PROVIDER_UNSET if opts.provider_id is None else opts.provider_id,
                      opts.scrypt_n, opts.scrypt_r, opts.scrypt_p, opts.compute_batch_size, opts.self_check_every)


class PostSetupManager:
    def __init__(self, cfg: PostConfig | None = None):
        L = _bind()
        cfg = cfg or PostConfig()
        c = _PostConfig()
        L.b200post_default_post_config(ctypes.byref(c))
        c.min_num_units, c.max_num_units, c.labels_per_unit = cfg.min_num_units, cfg.max_num_units, cfg.labels_per_unit
        c.k1, c.k2, c.k3 = cfg.k1, cfg.k2, cfg.k3
        if cfg.pow_difficulty is not None:   # the initial proof's k2pow difficulty
            ctypes.memmove(c.pow_difficulty, cfg.pow_difficulty, 32)
        self.cfg = cfg
        self._initial_opts = None
        self._h = ctypes.c_void_p()
        _err(L.b200post_setup_manager_new(ctypes.byref(c), ctypes.byref(self._h)))

    def prepare_initializer(self, opts: PostSetupOpts, node_id: bytes, commitment_atx_id: bytes) -> None:
        _err(_bind().b200post_setup_prepare_initializer(self._h, ctypes.byref(_c_opts(opts)), node_id, commitment_atx_id))

    def prepare_files(self, opts: PostSetupOpts, node_id: bytes, commitment_atx_id: bytes, from_file: int, to_file: int = -1) -> None:
        """PrepareInitializer restricted to postdata files [from_file, to_file] (-1 = the last file): postcli -fromFile/-toFile."""
        _err(_bind().b200post_setup_prepare_files(self._h, ctypes.byref(_c_opts(opts)), node_id, commitment_atx_id, from_file,
                                                  to_file))

    def start_session(self, cancel: ctypes.c_int | None = None) -> None:
        """Blocking.  `cancel` = a ctypes.c_int another thread sets to 1 (ctx cancel); raises code ERR_CANCELLED."""
        _err(_bind().b200post_setup_start_session(self._h, ctypes.addressof(cancel) if cancel is not None else None))

    def request_initial_proof(self, *, nonces: int = 16, pow="builtin", pow_cache_key: bytes | None = None,
                              windows_per_pass: int = 1) -> None:
        """Ask the prepared (whole-POST) session for the initial proof: the proof for the zero challenge, computed from
        the labels as start_session writes them and stored in initial_post.json.  pow as in prove.generate_proof:
        "builtin", "skip" or a callable.  windows_per_pass: the nonce windows the session scans (its proof is
        prove.generate_proof's with max_windows = that count).  Call between prepare_initializer and start_session."""
        from . import prove
        opts, _ = prove._opts(None, None, nonces, 0, pow, 1, windows_per_pass)
        if pow_cache_key is not None:
            opts.pow_cache_key, opts.pow_cache_key_len = pow_cache_key, len(pow_cache_key)
        self._initial_opts = opts   # keeps a pow callback alive for the session
        _err(_bind().b200post_setup_request_initial_proof(self._h, ctypes.byref(opts)))

    def request_range_record(self, *, initial_proof: bool = False, nonces: int = 16, pow="builtin",
                             pow_cache_key: bytes | None = None, windows_per_pass: int = 1) -> None:
        """Ask the prepared file-range session (prepare_files, metadata without a nonce) to keep a record of its range in
        range_<from>_<to>.rec: the range's VRF candidate, and with initial_proof=True also the initial-proof scan of its
        labels (nonces, pow, pow_cache_key and windows_per_pass as in request_initial_proof).  merge_range_records turns
        the records of every range into the POST's nonce and initial proof.  Call between prepare_files and start_session."""
        if not initial_proof:
            self._initial_opts = None
            _err(_bind().b200post_setup_request_range_record(self._h, None))
            return
        from . import prove
        opts, _ = prove._opts(None, None, nonces, 0, pow, 1, windows_per_pass)
        if pow_cache_key is not None:
            opts.pow_cache_key, opts.pow_cache_key_len = pow_cache_key, len(pow_cache_key)
        self._initial_opts = opts   # keeps a pow callback alive for the session
        _err(_bind().b200post_setup_request_range_record(self._h, ctypes.byref(opts)))

    def request_checksums(self) -> None:
        """Ask the prepared session to write postdata_<N>.sum (block checksums) for every file it writes, from the
        labels it computes; labels already on disk are recomputed for them, not read back.  Call between prepare and
        start_session."""
        _err(_bind().b200post_setup_request_checksums(self._h))

    def initial_proof(self):
        """After a completed session that asked for it: (Proof, ProofMetadata, labels scanned).  Raises ERR_INVALID_PROOF
        with the reason when no nonce reached K2 or the verifier refused the proof, ERR_STATE before completion."""
        from . import prove
        from .verify import _Meta
        out, meta = prove._ProofOut(), _Meta()
        _err(_bind().b200post_setup_initial_proof(self._h, ctypes.byref(out), ctypes.byref(meta)))
        return prove._results(out, meta)

    def status(self) -> PostSetupStatus:
        s = _Status()
        _err(_bind().b200post_setup_get_status(self._h, ctypes.byref(s)))
        return PostSetupStatus(int(s.state), int(s.num_labels_written))

    def reset(self) -> None:
        _err(_bind().b200post_setup_reset(self._h))

    def commitment_atx(self) -> bytes:
        out = ctypes.create_string_buffer(32)
        _err(_bind().b200post_setup_commitment_atx(self._h, out))
        return out.raw

    def __del__(self):
        try:
            if self._h:
                _bind().b200post_setup_manager_free(self._h)
                self._h = None
        except Exception:  # noqa: BLE001
            pass
