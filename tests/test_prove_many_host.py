"""CPU tier: several identities in one call (b200post_generate_proofs, b200post_k2pow_search_jobs) without touching a
device, and the job search's schedule (csrc/k2pow_jobs.cpp) driven through tests/k2pow_jobs_emul.cpp.

* Argument validation: the call's INVALID_ARGUMENT leaves every item untouched.
* Item errors stay with the item: a missing directory gets the single call's IO and text, while the call answers for
  the device list (NO_DEVICE on a machine without one, UNSUPPORTED for the CPU id) and the other items with it.
* b200post_k2pow_search_jobs answers as the group search does for the same provider list.
* The schedule: with 1, 2 and 3 simulated devices finishing windows in random order, every job's pow is its smallest
  valid pow below the cap, it is final exactly when announced, the batches tile at most `batch` VMs, and one device
  computes the hashes of the group search's round schedule."""
import ctypes
import importlib
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
POST_FILES = ROOT / "tests" / "golden" / "post_files"
CPU = 0xFFFFFFFF
LPU, UNITS, PER_FILE, K1, K2 = 2048, 2, 1024, 300, 12
U64P = ctypes.POINTER(ctypes.c_uint64)
ERR_IO = 12                 # B200POST_ERR_IO (include/b200post_setup.h)


def _mod(name):
    if str(ROOT) not in sys.path:
        sys.path.insert(0, str(ROOT))
    return importlib.import_module("go-spacemesh_b200" + name)


def _post_dir(d: Path) -> str:
    d.mkdir(parents=True)
    for p in (POST_FILES / "full_w1").iterdir():
        shutil.copy(p, d / p.name)
    for f in range(LPU * UNITS // PER_FILE):
        (d / f"postdata_{f}.bin").write_bytes(bytes(16 * PER_FILE))
    return str(d)


@pytest.fixture(scope="module")
def api(b2):
    su, pv, k2 = _mod(".setup"), _mod(".prove"), _mod(".k2pow")
    C = ctypes.CDLL(str(b2.LIB_PATH))
    C.b200post_last_error.restype = ctypes.c_char_p
    cfg = pv._c_cfg(su.PostConfig(labels_per_unit=LPU, k1=K1, k2=K2, k3=K2, max_num_units=8))
    return C, pv, k2, cfg


def _items(pv, specs):
    arr = (pv._ProveItem * max(len(specs), 1))()
    for a, (d, ch) in zip(arr, specs):
        a.data_dir = d.encode() if d is not None else None
        a.challenge = (ctypes.c_uint8 * 32)(*ch)
        a.status = 12345
    return arr


def _call(C, pv, cfg, arr, n, providers, pow_="skip", checked=1, use_cfg=True):
    opts, _ = pv._opts(None, None, 16, 0, pow_)
    ids = None if providers is None else (ctypes.c_uint32 * max(len(providers), 1))(*providers)
    rc = C.b200post_generate_proofs(arr, ctypes.c_size_t(n), ctypes.byref(cfg) if use_cfg else None, ctypes.byref(opts), ids,
                                    len(providers) if providers is not None else 0, ctypes.c_uint32(checked), ctypes.c_uint32(0), None)
    return rc, C.b200post_last_error().decode()


def test_argument_validation_touches_no_item(api, b2, tmp_path):
    C, pv, _, cfg = api
    good = _post_dir(tmp_path / "p")
    for specs, n, providers, use_cfg, what in (
            ([(good, bytes(32))], 0, [0], True, "n = 0"),
            ([(good, bytes(32))], 1, None, True, "no providers"),
            ([(good, bytes(32))], 1, [], True, "n_providers = 0"),
            ([(good, bytes(32))], 1, [0], False, "cfg NULL"),
            ([(good, bytes(32)), (None, bytes(32))], 2, [0], True, "item without data_dir")):
        arr = _items(pv, specs)
        rc, err = _call(C, pv, cfg, arr, n, providers, use_cfg=use_cfg)
        assert rc == b2.ERR_INVALID_ARGUMENT, what
        assert err.startswith("invalid argument"), what
        assert all(a.status == 12345 for a in arr[:len(specs)]), what
    rc, _ = _call(C, pv, cfg, None, 1, [0])
    assert rc == b2.ERR_INVALID_ARGUMENT


def _single(C, pv, cfg, d, providers, pow_="skip"):
    opts, _ = pv._opts(None, None, 16, 0, pow_)
    ids = (ctypes.c_uint32 * len(providers))(*providers)
    rc = C.b200post_generate_proof_checked(d.encode(), bytes(32), ctypes.byref(cfg), ctypes.byref(opts), ids, len(providers),
                                           ctypes.byref(pv._ProofOut()), None, ctypes.byref(pv._ProveCheck()), None)
    return rc, C.b200post_last_error().decode()


@pytest.mark.parametrize("pow_", ("skip", "builtin"))
def test_item_errors_stay_with_the_item(api, b2, tmp_path, pow_):
    """Missing directory + a good POST: the missing item gets the single call's IO and text; the call and the good item
    answer for the device list as the single call does (CPU id: UNSUPPORTED anywhere; no device: NO_DEVICE)."""
    C, pv, _, cfg = api
    good, missing = _post_dir(tmp_path / "p"), str(tmp_path / "missing")
    lists = [[CPU], [CPU, 0]] + ([] if b2.providers() else [[0]])
    for providers in lists:
        arr = _items(pv, [(missing, bytes(32)), (good, bytes(32))])
        rc, err = _call(C, pv, cfg, arr, 2, providers, pow_)
        alone = [_single(C, pv, cfg, d, providers, pow_) for d in (missing, good)]
        assert alone[0][0] == ERR_IO
        assert alone[1][0] in (b2.ERR_NO_DEVICE, b2.ERR_UNSUPPORTED)
        assert (rc, err) == alone[1], providers
        assert [(a.status, a.error.decode()) for a in arr[:2]] == alone, providers
        assert all(a.proof.indices_len == 0 for a in arr[:2])


def test_pow_mode_is_the_calls_answer(api, b2, tmp_path):
    C, pv, _, cfg = api
    good, missing = _post_dir(tmp_path / "p"), str(tmp_path / "missing")
    arr = _items(pv, [(missing, bytes(32)), (good, bytes(32))])
    rc, err = _call(C, pv, cfg, arr, 2, [0], "callback-missing")
    alone = [_single(C, pv, cfg, d, [0], "callback-missing") for d in (missing, good)]
    assert alone[1][0] == b2.ERR_UNSUPPORTED and (rc, err) == alone[1]
    assert [(a.status, a.error.decode()) for a in arr[:2]] == alone


def test_search_jobs_answers_as_the_group_search(api, b2):
    C, _, k2, _ = api
    u32, u64 = ctypes.c_uint32, ctypes.c_uint64
    job = k2._Job()
    kp = k2._params(0, bytes(8), bytes(32), b"\x00" * 31 + b"\x01", None)

    def jobs(ps, n=1, with_jobs=True, with_pows=True):
        ids = None if ps is None else (u32 * max(len(ps), 1))(*ps)
        rc = C.b200post_k2pow_search_jobs(ids, len(ps) if ps is not None else 2, None, ctypes.c_size_t(0), ctypes.c_size_t(n),
                                          ctypes.byref(job) if with_jobs else None, u64(1), (u64 * 1)() if with_pows else None,
                                          ctypes.byref(u64()), None)
        return rc, C.b200post_last_error().decode()

    def groups(ps):
        ids = None if ps is None else (u32 * max(len(ps), 1))(*ps)
        rc = C.b200post_k2pow_search_group_range_multi(ids, len(ps) if ps is not None else 2, ctypes.byref(kp), u32(0), u32(1), u64(1),
                                                       (u64 * 1)(), ctypes.byref(u64()), None)
        return rc, C.b200post_last_error().decode()

    for bad in (jobs(None), jobs([]), jobs([0], n=0), jobs([0], with_jobs=False), jobs([0], with_pows=False)):
        assert bad == (b2.ERR_INVALID_ARGUMENT, "invalid argument")
    lists = [[CPU], [CPU, 0], [0xFFFFFFFE]] + ([] if b2.providers() else [[0], [0, CPU]])
    for ps in lists:
        assert jobs(ps) == groups(ps), ps
        assert jobs(ps)[0] in (b2.ERR_NO_DEVICE, b2.ERR_UNSUPPORTED)


# ------------------------------------------------------------------------------------------------- the schedule
@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = tmp_path_factory.mktemp("k2pow_jobs") / "k2pow_jobs_emul.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", str(out), str(ROOT / "tests" / "k2pow_jobs_emul.cpp"),
                    str(ROOT / "go-spacemesh_b200" / "csrc" / "k2pow_jobs.cpp")], check=True)
    L = ctypes.CDLL(str(out))
    L.emul_search.argtypes = [ctypes.c_uint32, U64P, ctypes.POINTER(ctypes.c_uint32), ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint32,
                              ctypes.c_uint32, U64P, U64P, U64P, U64P]
    return L


def _hashes_done(batch, n_jobs, cap, pows):
    """The group search's round schedule: every pending job tries `per` more nonces per round."""
    pending, nxt, total = list(range(n_jobs)), 0, 0
    while pending and nxt < cap:
        per = min(max(1, batch // len(pending)), cap - nxt)
        total += len(pending) * per
        pending = [j for j in pending if pows[j] is None or pows[j] >= nxt + per]
        nxt += per
    return total


CASES = [   # (jobs, 1 / pass rate, cap, batch)
    (1, 16, 10_000, 64),
    (18, 16, 10_000, 64),       # the pending list shrinks over the rounds
    (150, 4, 10_000, 64),       # more jobs than a batch: one nonce each, windows of several batches
    (7, 50, 40, 16),            # the cap ends the search with jobs still pending
    (40, 30, 10_000, 1000),
]


@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}jobs-1in{c[1]}-cap{c[2]}-batch{c[3]}" for c in CASES])
@pytest.mark.parametrize("devices", (1, 2, 3))
def test_schedule_gives_the_smallest_pow_and_announces_it_once(emul, case, devices):
    n_jobs, rate, cap, batch = case
    rng = np.random.default_rng(n_jobs * 1000 + rate)
    valid = [np.flatnonzero(rng.random(cap + 500) < 1 / rate).astype(np.uint64) for _ in range(n_jobs)]
    flat = np.concatenate(valid + [np.zeros(1, np.uint64)]).astype(np.uint64)
    first = np.cumsum([0] + [len(v) for v in valid]).astype(np.uint32)
    want = [int(v[0]) if len(v) and v[0] < cap else None for v in valid]
    assert any(w is not None for w in want)
    for seed in range(4):
        pows, final, hashes, batches = (np.zeros(n_jobs, np.uint64), np.zeros(n_jobs, np.uint64), ctypes.c_uint64(),
                                        ctypes.c_uint64())
        rc = emul.emul_search(n_jobs, flat.ctypes.data_as(U64P), first.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), cap, batch,
                              devices, seed, pows.ctypes.data_as(U64P), final.ctypes.data_as(U64P), ctypes.byref(hashes),
                              ctypes.byref(batches))
        assert rc == 0, {1: "a job announced final twice", 2: "segments do not tile a batch", 3: "a batch over `batch` VMs"}[rc]
        got = [None if int(p) == 2**64 - 1 else int(p) for p in pows]
        assert got == want, seed
        # the pow announced at finality is the final pow: nothing ever lowered it afterwards
        assert [None if int(p) == 2**64 - 1 else int(p) for p in final] == want, seed
        if devices == 1:
            assert hashes.value == _hashes_done(batch, n_jobs, cap, want)
