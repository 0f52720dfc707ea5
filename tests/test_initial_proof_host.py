"""CPU tier: the host checks of the setup session's initial proof: when it may be requested, argument errors, no CPU
path without a device, and b200post_load_initial_proof on hand-written files."""
import base64
import ctypes
import importlib
import json

import pytest

NODE, ATX = bytes(range(32)), bytes(range(32, 64))
LPU, UNITS, K1, K2, NONCES = 512, 2, 26, 12, 32


@pytest.fixture()
def mods(b2):
    return importlib.import_module("go-spacemesh_b200.setup"), importlib.import_module("go-spacemesh_b200.prove")


def _cfg(su, k2=K2):
    return su.PostConfig(labels_per_unit=LPU, k1=K1, k2=k2, k3=k2)


def _prepared(su, d, provider_id=0, **kw):
    mgr = su.PostSetupManager(_cfg(su))
    o = su.PostSetupOpts(data_dir=str(d), num_units=UNITS, max_file_size=4096, provider_id=provider_id, scrypt_n=2)
    if kw:
        mgr.prepare_files(o, NODE, ATX, **kw)
    else:
        mgr.prepare_initializer(o, NODE, ATX)
    return mgr


def _raises(b2, fn, *a, **kw) -> int:
    with pytest.raises(b2.B200PostError) as e:
        fn(*a, **kw)
    return e.value.code


def test_request_needs_a_prepared_whole_post_session(b2, mods, tmp_path):
    su, _ = mods
    mgr = su.PostSetupManager(_cfg(su))
    assert _raises(b2, mgr.request_initial_proof, nonces=NONCES, pow="skip") == su.ERR_STATE   # never prepared
    rng = _prepared(su, tmp_path / "r", from_file=0, to_file=0)
    assert _raises(b2, rng.request_initial_proof, nonces=NONCES, pow="skip") == su.ERR_STATE   # a file range
    mgr = _prepared(su, tmp_path / "w")
    mgr.request_initial_proof(nonces=NONCES, pow="skip")
    mgr.request_initial_proof(nonces=NONCES, pow="skip")                                       # a new call replaces it


def test_request_argument_errors(b2, mods, tmp_path):
    su, pr = mods
    mgr = _prepared(su, tmp_path / "p")
    for bad in (8, 17, 4112):
        assert _raises(b2, mgr.request_initial_proof, nonces=bad, pow="skip") == b2.ERR_INVALID_ARGUMENT, bad
    assert _raises(b2, mgr.request_initial_proof, nonces=NONCES, pow="callback-missing") == b2.ERR_UNSUPPORTED
    L = su._bind()
    assert L.b200post_setup_request_initial_proof(mgr._h, None) == b2.ERR_INVALID_ARGUMENT
    opts, _ = pr._opts(None, None, NONCES, 0, "skip")
    opts.pow_mode = 7
    assert L.b200post_setup_request_initial_proof(mgr._h, ctypes.byref(opts)) == b2.ERR_UNSUPPORTED


def test_getter_before_completion(b2, mods, tmp_path):
    su, _ = mods
    mgr = su.PostSetupManager(_cfg(su))
    assert _raises(b2, mgr.initial_proof) == su.ERR_STATE
    mgr = _prepared(su, tmp_path / "p")
    mgr.request_initial_proof(nonces=NONCES, pow="skip")
    assert _raises(b2, mgr.initial_proof) == su.ERR_STATE


def test_start_with_a_request_and_no_device(b2, mods, tmp_path):
    su, _ = mods
    if b2.providers():
        pytest.skip("a CUDA device is present: the no-device contract is covered on CPU-only boxes")
    for pid in (0, su.PROVIDER_ALL):
        d = tmp_path / f"p{pid}"
        mgr = _prepared(su, d, provider_id=pid)
        mgr.request_initial_proof(nonces=NONCES, pow="skip")
        assert _raises(b2, mgr.start_session) == b2.ERR_NO_DEVICE
        assert not (d / "initial_post.scan").exists() and not (d / "initial_post.json").exists()
        assert mgr.status().state == su.STATE_ERROR


def _proof_file(d, **over):
    bits = (LPU * UNITS).bit_length()
    doc = {"NodeId": base64.b64encode(NODE).decode(), "CommitmentAtxId": base64.b64encode(ATX).decode(), "NumUnits": UNITS,
           "LabelsPerUnit": LPU, "K1": K1, "K2": K2, "Nonces": NONCES, "PowDifficulty": None,
           "Challenge": base64.b64encode(bytes(32)).decode(), "Nonce": 5,
           "Indices": base64.b64encode(bytes(range((K2 * bits + 7) // 8))).decode(), "Pow": 77}
    doc.update(over)
    (d / "initial_post.json").write_text(json.dumps(doc, indent=1))


def test_load_initial_proof_from_hand_written_files(b2, mods, tmp_path):
    su, pr = mods
    d = tmp_path / "p"
    _prepared(su, d)                                   # writes the metadata only
    cfg = _cfg(su)
    diff = bytes(pr._c_cfg(cfg).pow_difficulty).hex()
    # absent
    e = pytest.raises(b2.B200PostError, su.load_initial_proof, str(d), cfg, NONCES)
    assert e.value.code == su.ERR_IO and "no initial proof" in str(e.value)
    # a well-formed file loads
    _proof_file(d, PowDifficulty=diff)
    proof, meta, scanned = su.load_initial_proof(str(d), cfg, NONCES)
    assert (proof.nonce, proof.pow, scanned) == (5, 77, LPU * UNITS)
    assert proof.indices == bytes(range(len(proof.indices)))
    assert (meta.node_id, meta.commitment_atx_id, meta.challenge, meta.num_units) == (NODE, ATX, bytes(32), UNITS)
    # truncated
    text = (d / "initial_post.json").read_text()
    (d / "initial_post.json").write_text(text[: len(text) // 2])
    assert _raises(b2, su.load_initial_proof, str(d), cfg, NONCES) == su.ERR_IO
    # stale or foreign: identity, K2, NumUnits, nonce count, challenge, pow difficulty
    for over in ({"NodeId": base64.b64encode(bytes(32)).decode()}, {"K2": K2 + 1}, {"NumUnits": UNITS + 1},
                 {"Nonces": NONCES + 16}, {"Challenge": base64.b64encode(b"\x01" * 32).decode()}, {"PowDifficulty": "00" * 32}):
        _proof_file(d, **{"PowDifficulty": diff, **over})
        e = pytest.raises(b2.B200PostError, su.load_initial_proof, str(d), cfg, NONCES)
        assert e.value.code == su.ERR_IO and "no initial proof" in str(e.value), over
    _proof_file(d, PowDifficulty=diff)
    assert _raises(b2, su.load_initial_proof, str(d), _cfg(su, k2=K2 + 1), NONCES) == su.ERR_IO
    assert _raises(b2, su.load_initial_proof, str(d), cfg, NONCES + 16) == su.ERR_IO
    # the metadata grew (re-prepared with more units): the stored proof no longer applies
    mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=LPU, k1=K1, k2=K2, k3=K2))
    mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=UNITS + 1, max_file_size=4096, provider_id=0, scrypt_n=2),
                            NODE, ATX)
    assert _raises(b2, su.load_initial_proof, str(d), cfg, NONCES) == su.ERR_IO
    # no metadata at all
    (tmp_path / "empty").mkdir()
    assert _raises(b2, su.load_initial_proof, str(tmp_path / "empty"), cfg, NONCES) == su.ERR_IO


def test_reset_removes_the_initial_proof_files(b2, mods, tmp_path):
    su, _ = mods
    d = tmp_path / "p"
    mgr = _prepared(su, d)
    (d / "initial_post.json").write_text("{}")
    (d / "initial_post.scan").write_bytes(b"x" * 64)
    (d / "keep.txt").write_text("not ours")
    mgr.reset()
    assert not (d / "initial_post.json").exists() and not (d / "initial_post.scan").exists()
    assert (d / "keep.txt").exists()
