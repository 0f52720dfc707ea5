"""GPU tier: the initial proof of a setup session (b200post_setup_request_initial_proof).

The session scans every label batch as it writes it and proves for the zero challenge without reading the data back.
Its proof must be the prover's over the written files (b200post_generate_proof with the same config, nonces and pows),
its files and metadata those of a session without the request, and a stopped session must resume to the same proof
whatever became of its scan state."""
import ctypes
import importlib
import json
import shutil
import struct
import subprocess
import sys
import threading
from pathlib import Path

import pytest

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
NODE, ATX = bytes(range(7, 39)), bytes(range(100, 132))
ZERO = bytes(32)
# (N, LabelsPerUnit, units, K1, K2, nonces, batch, labels per file)
PARITY = [(2, 2048, 2, 300, 12, 64, 1 << 10, 1024), (8192, 1024, 2, 200, 10, 16, 1 << 10, 512)]
# K1 below K2: a nonce expects fewer hits than it needs, so the winner's K2-th hit lies deep in the POST and the proof
# depends on many batches, file boundaries and (when resumed) on the state, the rescanned gap and the labels after it.
# With these identities the CPU oracle puts the winner's last index at 8600 (pow 0) and 10718 (pow 1000 + group) of
# 16384 in LATE, and the winner's indices of RESUME at 294 .. 9971 of 16384.
LATE = (2, 8192, 2, 10, 12, 64, 1 << 10, 4096)
RESUME = (8192, 8192, 2, 10, 12, 32, 512, 4096)
# one batch larger than a scan chunk (2^22 labels): the session computes it into its own buffer and scans it in pieces
BIG = (2, (1 << 22) + (1 << 21), 1, 10, 12, 16, (1 << 22) + (1 << 21), (1 << 22) + (1 << 21))


@pytest.fixture(scope="module")
def mods(b2, gpu_ready):
    return (importlib.import_module("go-spacemesh_b200.setup"), importlib.import_module("go-spacemesh_b200.prove"),
            importlib.import_module("go-spacemesh_b200.verify"), importlib.import_module("go-spacemesh_b200.k2pow"))


def _cfg(su, case, k2=None, pow_difficulty=None):
    n, lpu, units, k1, k2_, nonces, batch, per_file = case
    k2 = k2 or k2_
    return su.PostConfig(labels_per_unit=lpu, k1=k1, k2=k2, k3=k2, max_num_units=8, pow_difficulty=pow_difficulty)


def _opts(su, d, case, provider_id=0, units=None):
    n, lpu, units_, k1, k2, nonces, batch, per_file = case
    return su.PostSetupOpts(data_dir=str(d), num_units=units or units_, max_file_size=16 * per_file, provider_id=provider_id,
                            scrypt_n=n, compute_batch_size=batch)


def _callback_pow(calls=None):
    def pow_(ctx, group, ch, diff, node, out):
        if calls is not None:
            calls.append(group)
        out[0] = 1000 + group
        return 0
    return pow_


def _session(su, d, case, request=None, cancel_at=None, provider_id=0, cfg=None, units=None):
    """prepare (+ request) + start; cancel_at: a status-polling thread sets the cancel flag once that many labels are
    written.  Returns the manager."""
    mgr = su.PostSetupManager(cfg or _cfg(su, case))
    mgr.prepare_initializer(_opts(su, d, case, provider_id, units), NODE, ATX)
    if request is not None:
        mgr.request_initial_proof(**request)
    cancel = ctypes.c_int(0)
    if cancel_at is None:
        mgr.start_session()
        return mgr
    done = threading.Event()

    def poll():
        while not done.is_set():
            if mgr.status().num_labels_written >= cancel_at:
                cancel.value = 1
                return

    t = threading.Thread(target=poll)
    t.start()
    try:
        with pytest.raises(Exception) as e:
            mgr.start_session(cancel)
        assert e.value.code == 5   # ERR_CANCELLED
    finally:
        done.set()
        t.join()
    return mgr


def _files(d: Path) -> dict:
    return {p.name: p.read_bytes() for p in sorted(d.iterdir()) if p.name.startswith("postdata_")}


def _triple(proof):
    return proof.nonce, proof.indices, proof.pow


def _indices(vf, proof, case):
    n, lpu, units, k1, k2, nonces, batch, per_file = case
    return vf.unpack_indices(proof.indices, vf.bits_per_index(lpu * units), k2)


def _upto(state: bytes, nonces: int) -> int:
    """The end of the scanned prefix in initial_post.scan: after the 180-byte header (no cache key) and the pows."""
    return struct.unpack_from("<Q", state, 180 + 8 * (nonces // 16))[0]


@pytest.mark.parametrize("case", PARITY + [LATE], ids=["N2", "N8192", "N2-late"])
@pytest.mark.parametrize("pow_", ["skip", "callback"])
def test_parity_with_the_prover(mods, orc, tmp_path, case, pow_):
    su, pr, vf, _ = mods
    n, lpu, units, k1, k2, nonces, batch, per_file = case
    powarg = "skip" if pow_ == "skip" else _callback_pow()
    plain, req = tmp_path / "plain", tmp_path / "req"
    assert _session(su, plain, case).status().state == su.STATE_COMPLETE
    mgr = _session(su, req, case, request=dict(nonces=nonces, pow=powarg))
    assert mgr.status().state == su.STATE_COMPLETE
    assert _files(plain) == _files(req)                      # the labels and the metadata are untouched by the request
    proof, meta, scanned = mgr.initial_proof()
    assert scanned == units * lpu
    assert (meta.node_id, meta.commitment_atx_id, meta.challenge, meta.num_units, meta.labels_per_unit) == (NODE, ATX, ZERO, units, lpu)
    ref, ref_meta, _ = pr.generate_proof(str(plain), ZERO, _cfg(su, case), nonces=nonces, pow=powarg)
    assert _triple(proof) == _triple(ref)
    if pow_ == "callback":
        assert proof.pow == 1000 + proof.nonce // 16
    if case == LATE:   # decided by labels of later batches, past the first file boundary
        assert _indices(vf, proof, case)[-1] >= per_file
    assert orc.py_verify(proof.nonce, proof.indices, proof.pow, NODE, ATX, ZERO, units, lpu, k1, k2, n) == (True, None)
    v = vf.PostVerifier(pow="skip")
    try:
        v.verify(proof, meta, vf.VerifyParams(k1=k1, k2=k2, scrypt_n=n))
    finally:
        v.close()
    loaded, loaded_meta, _ = su.load_initial_proof(str(req), _cfg(su, case), nonces)
    assert _triple(loaded) == _triple(proof) and loaded_meta == meta
    doc = json.loads((req / "initial_post.json").read_text())
    assert (doc["Nonce"], doc["Pow"], doc["K1"], doc["K2"], doc["Nonces"]) == (proof.nonce, proof.pow, k1, k2, nonces)


def test_resume_after_cancel(mods, tmp_path):
    """(a) the state as left, (b) deleted, (c) one byte flipped, (d) an older state from the first file boundary.
    The winner has indices below the older state's prefix, inside the gap between the two states, and past the
    point where the session stopped, so a wrong restore, rescan or later scan changes the proof."""
    su, pr, vf, _ = mods
    n, lpu, units, k1, k2, nonces, batch, per_file = RESUME
    num = lpu * units
    ref = _session(su, tmp_path / "ref", RESUME, request=dict(nonces=nonces, pow=_callback_pow())).initial_proof()[0]
    assert _triple(ref) == _triple(pr.generate_proof(str(tmp_path / "ref"), ZERO, _cfg(su, RESUME), nonces=nonces,
                                                     pow=_callback_pow())[0])
    half = tmp_path / "half"
    calls = []
    _session(su, half, RESUME, request=dict(nonces=nonces, pow=_callback_pow(calls)), cancel_at=per_file)
    assert calls == list(range(nonces // 16))
    older = (half / "initial_post.scan").read_bytes()          # saved at the stop, one file in
    mgr = _session(su, half, RESUME, request=dict(nonces=nonces, pow=_callback_pow(calls)), cancel_at=num // 2)
    stopped = mgr.status().num_labels_written
    assert mgr.status().state == su.STATE_STOPPED and num // 2 <= stopped < num
    assert calls == list(range(nonces // 16))                   # the stored pows were used
    state = (half / "initial_post.scan").read_bytes()
    older_upto, upto = _upto(older, nonces), _upto(state, nonces)
    assert per_file <= older_upto < upto == stopped
    idx = _indices(vf, ref, RESUME)
    assert idx[0] < older_upto                                  # from the restored hit lists
    assert any(older_upto <= i < upto for i in idx)             # from the gap, rescanned from disk under (d)
    assert idx[-1] >= stopped                                   # from labels computed after the resume
    for variant in "abcd":
        d = tmp_path / variant
        shutil.copytree(half, d)
        state = d / "initial_post.scan"
        if variant == "b":
            state.unlink()
        elif variant == "c":
            raw = bytearray(state.read_bytes())
            raw[len(raw) // 2] ^= 0x10
            state.write_bytes(bytes(raw))
        elif variant == "d":
            state.write_bytes(older)
        vcalls = []
        mgr = _session(su, d, RESUME, request=dict(nonces=nonces, pow=_callback_pow(vcalls)))
        assert mgr.status().state == su.STATE_COMPLETE
        assert _triple(mgr.initial_proof()[0]) == _triple(ref), variant
        assert vcalls == ([] if variant in "ad" else list(range(nonces // 16))), variant
        assert _files(d) == _files(tmp_path / "ref"), variant


def test_batches_larger_than_a_scan_chunk(mods, tmp_path):
    """One batch of 1.5 x 2^22 labels is scanned in two pieces; the winner has hits in both."""
    su, pr, vf, _ = mods
    n, lpu, units, k1, k2, nonces, batch, per_file = BIG
    plain, req = tmp_path / "plain", tmp_path / "req"
    _session(su, plain, BIG)
    proof = _session(su, req, BIG, request=dict(nonces=nonces, pow="skip")).initial_proof()[0]
    assert _files(plain) == _files(req)
    assert _triple(proof) == _triple(pr.generate_proof(str(plain), ZERO, _cfg(su, BIG), nonces=nonces, pow="skip")[0])
    idx = _indices(vf, proof, BIG)
    assert idx[0] < 1 << 22 <= idx[-1]


def test_all_providers_give_the_same_proof(mods, tmp_path):
    su, _, _, _ = mods
    case = PARITY[0]
    a = _session(su, tmp_path / "one", case, request=dict(nonces=case[5], pow="skip")).initial_proof()[0]
    b = _session(su, tmp_path / "all", case, request=dict(nonces=case[5], pow="skip"), provider_id=su.PROVIDER_ALL).initial_proof()[0]
    assert _triple(a) == _triple(b)


EASY = b"\x0f" + b"\xff" * 31


def test_builtin_pow(mods, tmp_path):
    su, pr, _, k2 = mods
    case = PARITY[0]
    n, lpu, units, k1, k2_, nonces, batch, per_file = case
    cfg = _cfg(su, case, pow_difficulty=EASY)
    mgr = _session(su, tmp_path / "p", case, request=dict(nonces=nonces, pow="builtin"), cfg=cfg)
    proof, meta, _ = mgr.initial_proof()                        # the gate passed, k2pow included
    pows, _ = k2.search_groups(ZERO[:8], NODE, k2.scale_difficulty(EASY, units), nonces // 16)
    assert proof.pow == pows[proof.nonce // 16]
    ref = pr.generate_proof(str(tmp_path / "p"), ZERO, cfg, nonces=nonces, pow="builtin")[0]
    assert _triple(proof) == _triple(ref)


_SLOTS = r"""
import importlib, sys, threading, tempfile
sys.path.insert(0, sys.argv[1])
b2 = importlib.import_module("go-spacemesh_b200")
su = importlib.import_module("go-spacemesh_b200.setup")
k2 = importlib.import_module("go-spacemesh_b200.k2pow")
mode, easy = sys.argv[2], bytes.fromhex(sys.argv[3])
if mode == "resident":
    k2.search_groups(bytes(8), bytes(32), easy, 2)
    print(b2.wave_slots(8192)); sys.exit(0)
cfg = su.PostConfig(labels_per_unit=1 << 14, k1=200, k2=10, k3=10, pow_difficulty=easy)
mgr = su.PostSetupManager(cfg)
d = tempfile.mkdtemp()
mgr.prepare_initializer(su.PostSetupOpts(data_dir=d, num_units=2, max_file_size=16 << 14, provider_id=0, scrypt_n=8192,
                                         compute_batch_size=4096), bytes(range(32)), bytes(32))
if mode == "request":
    mgr.request_initial_proof(nonces=32, pow="builtin")
out = []
def watch():
    while mgr.status().num_labels_written < 4096:
        pass
    out.append(b2.wave_slots(8192))
t = threading.Thread(target=watch); t.start()
mgr.start_session(); t.join()
print(out[0])
"""


def test_randomx_memory_is_released_before_the_labels(b2, mods, tmp_path):
    """In fresh processes: the label layer of a session with a BUILTIN request has the slots of one without, and fewer
    slots while a RandomX dataset is resident (so the comparison can see the difference)."""
    b2.shutdown()   # this process's engines give their HBM back: the subprocesses see the same free memory
    slots = {}
    for mode in ("plain", "request", "resident"):
        r = subprocess.run([sys.executable, "-c", _SLOTS, str(ROOT), mode, EASY.hex()], capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr
        slots[mode] = int(r.stdout.split()[-1])
    assert slots["request"] == slots["plain"], slots
    assert slots["resident"] < slots["plain"], slots


def test_no_proof_reset_and_load(mods, tmp_path):
    su, _, _, _ = mods
    case = PARITY[0]
    n, lpu, units, k1, k2, nonces, batch, per_file = case
    # no nonce reaches K2: the session still completes, without a proof file
    d = tmp_path / "none"
    mgr = _session(su, d, case, request=dict(nonces=nonces, pow="skip"), cfg=_cfg(su, case, k2=4000))
    assert mgr.status().state == su.STATE_COMPLETE
    with pytest.raises(Exception) as e:
        mgr.initial_proof()
    assert e.value.code == 7 and "no proof found" in str(e.value)   # ERR_INVALID_PROOF
    assert not (d / "initial_post.json").exists() and (d / "initial_post.scan").exists()
    # the outcome belongs to that session: re-prepared and run without a request, the getter has nothing to give
    mgr.prepare_initializer(_opts(su, d, case), NODE, ATX)
    mgr.start_session()
    with pytest.raises(Exception) as e:
        mgr.initial_proof()
    assert e.value.code == su.ERR_STATE
    mgr.reset()
    assert not (d / "initial_post.scan").exists() and not any(d.iterdir())
    # load_initial_proof answers from the file, and refuses it once the metadata grows or K2 differs
    d = tmp_path / "ok"
    proof = _session(su, d, case, request=dict(nonces=nonces, pow="skip")).initial_proof()[0]
    assert _triple(su.load_initial_proof(str(d), _cfg(su, case), nonces)[0]) == _triple(proof)
    with pytest.raises(Exception) as e:
        su.load_initial_proof(str(d), _cfg(su, case, k2=k2 + 1), nonces)
    assert e.value.code == su.ERR_IO and "no initial proof" in str(e.value)
    su.PostSetupManager(_cfg(su, case)).prepare_initializer(_opts(su, d, case, units=units + 1), NODE, ATX)
    with pytest.raises(Exception) as e:
        su.load_initial_proof(str(d), _cfg(su, case), nonces)
    assert e.value.code == su.ERR_IO and "no initial proof" in str(e.value)
    # re-preparing with more units ignores the old state: the written labels are rescanned from disk
    mgr = _session(su, d, case, request=dict(nonces=nonces, pow="skip"), units=units + 1)
    grown = mgr.initial_proof()[0]
    assert _triple(su.load_initial_proof(str(d), _cfg(su, case), nonces)[0]) == _triple(grown)
