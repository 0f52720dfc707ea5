"""go-spacemesh_b200 — GPU-native POST label engine (host bindings over the C ABI).

The product is ``libb200post.so`` (hand-written sm_90a CUDA + a C++ host runtime, built from
``csrc/``); this module is the thin ctypes layer the tests, ``bench.py`` and ``__graft_entry__`` use,
named after the reference interfaces it stands behind (activation/post.go, post_verifier.go).

There is deliberately NO fallback: if the shared library is missing, or no CUDA device is usable,
every compute call raises.  Nothing here imports ``oracle/``.

The directory name contains a hyphen, so import it with
``importlib.import_module("go-spacemesh_b200")`` (``__graft_entry__.load_package()`` does that).
"""
from __future__ import annotations

import ctypes
import subprocess
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
import os as _os

# B200POST_LIB=<path> loads an alternative build of the library (kernel experiments); default = in-tree build
LIB_PATH = Path(_os.environ["B200POST_LIB"]) if _os.environ.get("B200POST_LIB") else _HERE / "libb200post.so"

CPU_PROVIDER_ID = 0xFFFFFFFF  # systest/cluster/nodes.go:997 — refused by this library (no CPU path)

(OK, ERR_INVALID_ARGUMENT, ERR_NO_DEVICE, ERR_CUDA, ERR_OUT_OF_MEMORY, ERR_CANCELLED, ERR_CLOSED,
 ERR_INVALID_PROOF, ERR_EMPTY_PROOF, ERR_UNSUPPORTED) = range(10)


class B200PostError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"b200post error {code}: {msg}")
        self.code = code


class Provider(ctypes.Structure):
    """PostSetupProvider{ID, Model, DeviceType} (activation/post.go:24)."""
    _fields_ = [("id", ctypes.c_uint32), ("device_class", ctypes.c_uint32), ("model", ctypes.c_char * 64),
                ("hbm_bytes", ctypes.c_uint64), ("sm_count", ctypes.c_uint32), ("cc_major", ctypes.c_uint32),
                ("cc_minor", ctypes.c_uint32)]


class VrfNonce(ctypes.Structure):
    _fields_ = [("found", ctypes.c_uint32), ("reserved", ctypes.c_uint32), ("index", ctypes.c_uint64),
                ("label32", ctypes.c_uint8 * 32)]


def build(verbose: bool = False) -> Path:
    """Compile libb200post.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
    cmd = ["make", "-C", str(_HERE / "csrc"), "-j4"]
    res = subprocess.run(cmd, capture_output=not verbose, text=True)
    if res.returncode != 0:
        raise RuntimeError("building libb200post.so failed:\n" + (res.stdout or "") + (res.stderr or ""))
    return LIB_PATH


_lib = None


def lib() -> ctypes.CDLL:
    """Load the C-ABI library; raises (never falls back) if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise FileNotFoundError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                                "(there is no CPU fallback in this package)")
    L = ctypes.CDLL(str(LIB_PATH))
    u8p, u64, u32, vp = ctypes.c_char_p, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_void_p
    L.b200post_providers.argtypes = [ctypes.POINTER(Provider), ctypes.c_int]
    L.b200post_providers.restype = ctypes.c_int
    L.b200post_last_error.restype = ctypes.c_char_p
    L.b200post_set_option.argtypes = [u8p, ctypes.c_int64]
    L.b200post_get_option.argtypes = [u8p]
    L.b200post_get_option.restype = ctypes.c_int64
    L.b200post_labels_range.argtypes = [u32, u8p, u64, u64, u64, vp, vp, ctypes.POINTER(VrfNonce), vp]
    L.b200post_labels_range_dev.argtypes = [u32, u8p, u64, u64, u64, vp, vp, ctypes.POINTER(VrfNonce), vp]
    L.b200post_labels_range_multi.argtypes = [ctypes.POINTER(u32), ctypes.c_int, u8p, u64, u64, u64, vp, vp,
                                              ctypes.POINTER(VrfNonce), vp]
    L.b200post_labels_gather.argtypes = [u32, ctypes.c_size_t, vp, vp, u64, vp]
    L.b200post_labels_gather_indexed.argtypes = [u32, ctypes.c_size_t, ctypes.c_size_t, vp, vp, vp, u64, vp]
    L.b200post_commitment.argtypes = [u8p, u8p, vp]
    L.b200post_commitment.restype = None
    L.b200post_vrf_difficulty.argtypes = [u64, vp]
    L.b200post_vrf_difficulty.restype = None
    L.b200post_verify_vrf_nonce.argtypes = [u32, u64, u8p, u8p, u32, u64, u64, ctypes.POINTER(ctypes.c_int)]
    L.b200post_benchmark.argtypes = [u32, u64, ctypes.c_double, ctypes.POINTER(ctypes.c_double)]
    L.b200post_launch_count.restype = ctypes.c_uint64
    L.b200post_romix_time.argtypes = [u32, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(u64),
                                      ctypes.POINTER(ctypes.c_double), ctypes.c_int]
    L.b200post_last_call_ms.argtypes = [u32]
    L.b200post_last_call_ms.restype = ctypes.c_double
    L.b200post_wave_slots.argtypes = [u32, u64, ctypes.POINTER(u64)]
    L.b200post_timer_mark.argtypes = [u32, ctypes.c_int]
    L.b200post_timer_elapsed_ms.argtypes = [u32]
    L.b200post_timer_elapsed_ms.restype = ctypes.c_double
    L.b200post_shutdown.restype = None
    _lib = L
    return L


def _check(rc: int) -> None:
    if rc != OK:
        raise B200PostError(rc, lib().b200post_last_error().decode(errors="replace"))


def _opt_bytes(b: bytes | None):
    return ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p) if b is not None else None


# ------------------------------------------------------------------------------------------ providers
def providers() -> list[dict]:
    """PostSupervisor.Providers() analogue (activation/post_supervisor.go:105-117)."""
    n = lib().b200post_providers(None, 0)
    arr = (Provider * max(n, 1))()
    n = lib().b200post_providers(arr, n)
    return [dict(id=p.id, model=p.model.decode(), device_class=p.device_class, hbm_bytes=p.hbm_bytes,
                 sm_count=p.sm_count, cc=(p.cc_major, p.cc_minor)) for p in arr[:n]]


def set_option(key: str, value: int) -> None:
    _check(lib().b200post_set_option(key.encode(), int(value)))


def get_option(key: str) -> int:
    return int(lib().b200post_get_option(key.encode()))


# ------------------------------------------------------------------------------------------ label path
def commitment(node_id: bytes, commitment_atx_id: bytes) -> bytes:
    out = ctypes.create_string_buffer(32)
    lib().b200post_commitment(node_id, commitment_atx_id, out)
    return out.raw


def vrf_difficulty(num_labels: int) -> bytes:
    out = ctypes.create_string_buffer(32)
    lib().b200post_vrf_difficulty(num_labels, out)
    return out.raw


def _nonce_tuple(nonce):
    if nonce is None or not nonce.found:
        return None
    return int(nonce.index), bytes(nonce.label32)


def labels_range(commitment_: bytes, n: int, start: int, count: int, *, provider: int = 0,
                 vrf_difficulty_: bytes | None = None, discard: bool = False, cancel=None):
    """Initializer.Initialize over [start, start+count) (activation/post.go:295).

    Returns (labels uint8[count,16] or None when discard, vrf) with vrf = (index, label32) or None."""
    assert len(commitment_) == 32
    out = None if discard else np.empty((count, 16), dtype=np.uint8)
    nonce = VrfNonce() if vrf_difficulty_ is not None else None
    rc = lib().b200post_labels_range(provider, commitment_, n, start, count,
                                     out.ctypes.data if out is not None and count else None,
                                     _opt_bytes(vrf_difficulty_),
                                     ctypes.byref(nonce) if nonce is not None else None,
                                     ctypes.addressof(cancel) if cancel is not None else None)
    _check(rc)
    return out, _nonce_tuple(nonce)


def labels_range_dev(commitment_: bytes, n: int, start: int, count: int, d_out_ptr, *, provider: int = 0,
                     vrf_difficulty_: bytes | None = None):
    """Same with the 16-byte labels written to a device buffer (e.g. a torch.uint8 tensor's data_ptr())."""
    nonce = VrfNonce() if vrf_difficulty_ is not None else None
    rc = lib().b200post_labels_range_dev(provider, commitment_, n, start, count, d_out_ptr,
                                         _opt_bytes(vrf_difficulty_),
                                         ctypes.byref(nonce) if nonce is not None else None, None)
    _check(rc)
    return _nonce_tuple(nonce)


def labels_range_multi(providers_: list[int], commitment_: bytes, n: int, start: int, count: int, *,
                       vrf_difficulty_: bytes | None = None, discard: bool = False):
    out = None if discard else np.empty((count, 16), dtype=np.uint8)
    nonce = VrfNonce() if vrf_difficulty_ is not None else None
    arr = (ctypes.c_uint32 * len(providers_))(*providers_)
    rc = lib().b200post_labels_range_multi(arr, len(providers_), commitment_, n, start, count,
                                           out.ctypes.data if out is not None and count else None,
                                           _opt_bytes(vrf_difficulty_),
                                           ctypes.byref(nonce) if nonce is not None else None, None)
    _check(rc)
    return out, _nonce_tuple(nonce)


def labels_gather(commitments: np.ndarray, indices: np.ndarray, n: int, *, provider: int = 0) -> np.ndarray:
    """Labels at scattered (commitment, index) pairs — the recomputation inside ProofVerifier.Verify
    (activation/post_verifier.go:159)."""
    commitments = np.ascontiguousarray(commitments, dtype=np.uint8).reshape(-1, 32)
    indices = np.ascontiguousarray(indices, dtype=np.uint64)
    if commitments.shape[0] != indices.shape[0]:
        raise ValueError("commitments and indices differ in length")
    out = np.empty((indices.shape[0], 16), dtype=np.uint8)
    _check(lib().b200post_labels_gather(provider, indices.shape[0], commitments.ctypes.data, indices.ctypes.data, n,
                                        out.ctypes.data))
    return out


def labels_gather_indexed(commitments: np.ndarray, commitment_index: np.ndarray, indices: np.ndarray, n: int, *,
                          provider: int = 0) -> np.ndarray:
    """labels_gather for items sharing few commitments: item i uses commitments[commitment_index[i]]."""
    commitments = np.ascontiguousarray(commitments, dtype=np.uint8).reshape(-1, 32)
    commitment_index = np.ascontiguousarray(commitment_index, dtype=np.uint32)
    indices = np.ascontiguousarray(indices, dtype=np.uint64)
    if commitment_index.shape[0] != indices.shape[0]:
        raise ValueError("commitment_index and indices differ in length")
    out = np.empty((indices.shape[0], 16), dtype=np.uint8)
    _check(lib().b200post_labels_gather_indexed(provider, indices.shape[0], commitments.shape[0], commitments.ctypes.data,
                                                commitment_index.ctypes.data, indices.ctypes.data, n, out.ctypes.data))
    return out


def verify_vrf_nonce(nonce: int, node_id: bytes, commitment_atx_id: bytes, num_units: int, labels_per_unit: int,
                     n: int, *, provider: int = 0) -> bool:
    """verifying.VerifyVRFNonce (activation/validation.go:261-282)."""
    valid = ctypes.c_int(0)
    _check(lib().b200post_verify_vrf_nonce(provider, nonce, node_id, commitment_atx_id, num_units, labels_per_unit, n,
                                           ctypes.byref(valid)))
    return bool(valid.value)


def vrf_nonce_label(nonce: int, node_id: bytes, commitment_atx_id: bytes, n: int, *, provider: int = 0) -> bytes:
    """label32 at index `nonce` of the identity's POST — the policy-free half of VerifyVRFNonce."""
    out = ctypes.create_string_buffer(32)
    L = lib()
    L.b200post_vrf_nonce_label.argtypes = [ctypes.c_uint32, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_void_p]
    _check(L.b200post_vrf_nonce_label(provider, nonce, node_id, commitment_atx_id, n, out))
    return out.raw


def reference_label(commitment_: bytes, index: int, n: int) -> bytes:
    """The fault detector's independent checker: one label32 on the host CPU (NOT a compute path)."""
    out = ctypes.create_string_buffer(32)
    L = lib()
    L.b200post_reference_label.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_void_p]
    _check(L.b200post_reference_label(commitment_, index, n, out))
    return out.raw


def benchmark(n: int = 8192, seconds: float = 2.0, *, provider: int = 0) -> float:
    """PostSupervisor.Benchmark (activation/post_supervisor.go:120-127): labels ("hashes") per second."""
    v = ctypes.c_double(0)
    _check(lib().b200post_benchmark(provider, n, seconds, ctypes.byref(v)))
    return v.value


def launch_count() -> int:
    return int(lib().b200post_launch_count())


def romix_time(provider: int = 0, reset: bool = False) -> tuple[float, int, float]:
    """(device ms, launches, label-equivalents) accumulated by the ROMix kernel since the last reset."""
    ms, k, lab = ctypes.c_double(0), ctypes.c_uint64(0), ctypes.c_double(0)
    _check(lib().b200post_romix_time(provider, ctypes.byref(ms), ctypes.byref(k), ctypes.byref(lab), int(reset)))
    return ms.value, int(k.value), lab.value


def last_call_ms(provider: int = 0) -> float:
    """Device time (CUDA events on the engine's stream) of the last labels_* call on `provider`."""
    return float(lib().b200post_last_call_ms(provider))


def timer_mark(which: int, provider: int = 0) -> None:
    """Record a CUDA event on the engine's launching stream (0 = start, 1 = stop)."""
    _check(lib().b200post_timer_mark(provider, which))


def timer_elapsed_ms(provider: int = 0) -> float:
    return float(lib().b200post_timer_elapsed_ms(provider))


def wave_slots(n: int = 8192, provider: int = 0) -> int:
    """Labels one wave holds (= ROMix scratchpads resident at once) for scrypt-N."""
    v = ctypes.c_uint64(0)
    _check(lib().b200post_wave_slots(provider, n, ctypes.byref(v)))
    return int(v.value)


def metrics_text() -> str:
    """Counters of the engine in the Prometheus text format (activation/metrics/metrics.go analogue)."""
    L = lib()
    L.b200post_metrics_text.argtypes = [ctypes.c_char_p, ctypes.c_size_t]
    L.b200post_metrics_text.restype = ctypes.c_size_t
    n = L.b200post_metrics_text(None, 0)
    buf = ctypes.create_string_buffer(n + 1)
    L.b200post_metrics_text(buf, n + 1)
    return buf.value.decode()


def shutdown() -> None:
    lib().b200post_shutdown()
