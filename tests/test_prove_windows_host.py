"""CPU tier: proving over further nonce windows (b200post_prove_opts.max_windows / windows_per_pass).

* The windowed oracle (tests/window_oracle.py) against the scalar oracle, and its window 0 against np_prove_hits.
* The pass rule: scanning m windows per read gives the proof sequential windows give, and never reads more labels.
* The host checks: option mirroring and clamping, the k2pow group range's arguments, no CPU path, no device."""
import ctypes
import importlib
import random

import numpy as np
import pytest

import window_oracle as wo

NODE, ATX = bytes(range(32)), bytes(range(32, 64))
EASY = b"\x0f" + b"\xff" * 31


@pytest.fixture()
def mods(b2):
    return (importlib.import_module("go-spacemesh_b200.setup"), importlib.import_module("go-spacemesh_b200.prove"),
            importlib.import_module("go-spacemesh_b200.k2pow"))


# ------------------------------------------------------------------------------------------------------------ oracle
def test_window_hits_match_the_scalar_oracle(orc):
    rng = np.random.default_rng(5)
    labels = rng.integers(0, 256, (600, 16), dtype=np.uint8)
    ch, num, k1 = bytes(range(9, 41)), 600, 60           # about one label in ten passes a nonce
    pows = [11, 22]
    hits = wo.window_hits(orc, labels, ch, 32, 32, pows, k1, 600, num)   # window 1 of 32 nonces: groups 2 and 3
    assert sorted(hits) == list(range(32, 64))
    diff = orc.py_proving_difficulty(k1, num)
    for nonce in (32, 40, 47, 48, 63):
        want = [i for i in range(len(labels)) if orc.py_label_passes(labels[i].tobytes(), ch, nonce, pows[(nonce - 32) // 16], diff)]
        assert [int(i) for i in hits[nonce]] == want, nonce
    # window 0 is np_prove_hits
    zero = wo.window_hits(orc, labels, ch, 0, 32, [3, 4], k1, 5, num)
    ref = orc.np_prove_hits(labels, ch, 32, [3, 4], k1, 5, num)
    assert sorted(zero) == sorted(ref) and all(list(zero[n]) == list(ref[n]) for n in ref)


def test_windowed_proof_is_the_first_window_with_one(orc):
    """K2 set so that window 0 rarely has a proof: the oracle's answer is the first window whose own proof exists."""
    rng = np.random.default_rng(6)
    labels = rng.integers(0, 256, (4000, 16), dtype=np.uint8)
    ch, num, k1, k2, n = bytes(range(50, 82)), 4000, 20, 31, 16
    got = wo.windowed_proof(orc, labels, ch, n, lambda g: 7 * g, k1, k2, num, 256 // 16 * 16)
    assert got is not None
    w = got[0]
    for v in range(w):
        assert wo.pick(wo.window_hits(orc, labels, ch, v * n, n, [7 * v], k1, k2, num), k2) is None
    assert wo.pick(wo.window_hits(orc, labels, ch, w * n, n, [7 * w], k1, k2, num), k2) == got[1:]


def test_passes_equal_sequential_windows():
    """Random hit patterns: every windows-per-pass and chunk size gives the sequential proof, and reads no more."""
    r = random.Random(3)
    for trial in range(300):
        n, windows, k2 = 16 * r.choice((1, 2)), r.randint(1, 9), r.randint(1, 4)
        n_labels, chunk = r.randint(20, 300), r.randint(1, 64)
        rate = r.uniform(0.002, 0.03)
        hits = {x: sorted(r.sample(range(n_labels), min(n_labels, int(rate * n_labels) + r.randint(0, 2))))
                for x in range(n * windows)}
        seq, seq_read = None, 0
        for w in range(windows):
            proof, read = wo.pass_model(hits, n_labels, chunk, w, n, 1, k2)
            seq_read += read
            if proof:
                seq = (w, proof)
                break
        for m in (1, 2, 3, windows, windows + 1):
            got, read, a = None, 0, 0
            while a < windows and got is None:
                mm = min(m, windows - a)
                proof, rd = wo.pass_model(hits, n_labels, chunk, a, n, mm, k2)
                read += rd
                if proof:
                    got = (proof[0] // n, proof)
                a += mm
            assert got == seq, (trial, m)
            assert read <= seq_read, (trial, m)


# ------------------------------------------------------------------------------------------------------ host checks
def _post(su, d):
    o = su.PostSetupOpts(data_dir=str(d), num_units=2, max_file_size=4096, provider_id=0, scrypt_n=2)
    su.PostSetupManager().prepare_initializer(o, NODE, ATX)
    return o.data_dir


def test_options_mirror_the_c_struct(mods):
    _, pr, _ = mods
    old = pr._ProveOpts(3, 32, 7, ctypes.cast(None, pr.POW_PROVE_FN), None, 2, None, 0)   # positional, as before windows
    assert (old.provider, old.nonces, old.chunk_labels, old.max_windows, old.windows_per_pass) == (3, 32, 7, 0, 0)
    o, _ = pr._opts(None, [0], 16, 0, "skip", "all", 4)
    assert (o.max_windows, o.windows_per_pass) == (pr.ALL_WINDOWS, 4) and pr.ALL_WINDOWS == 2**32 - 1
    o, _ = pr._opts(None, None, 16, 0, "skip")
    assert (o.max_windows, o.windows_per_pass) == (1, 1)
    with pytest.raises(ValueError):
        pr._opts(None, None, 16, 0, "skip", "every")
    assert ctypes.sizeof(pr._ProveOpts) == 64


def test_group_range_arguments(b2, mods):
    _, _, k2 = mods
    for first, n in ((250, 7), (256, 1), (0, 257), (5, 0), (2**32 - 1, 2)):
        for provs in (None, [0], [0, 0]):
            with pytest.raises(b2.B200PostError) as e:
                k2.search_group_range(bytes(8), bytes(32), EASY, first, n, providers=provs)
            assert e.value.code == b2.ERR_INVALID_ARGUMENT, (first, n, provs)
    for provs in (None, [b2.CPU_PROVIDER_ID], [b2.CPU_PROVIDER_ID, 0]):
        with pytest.raises(b2.B200PostError) as e:
            k2.search_group_range(bytes(8), bytes(32), EASY, 5, 3, provider=b2.CPU_PROVIDER_ID if provs is None else 0, providers=provs)
        assert e.value.code == b2.ERR_UNSUPPORTED, provs


def test_cpu_provider_refused_with_windows(b2, mods, tmp_path):
    su, pr, _ = mods
    d = _post(su, tmp_path / "p")
    for pow_ in ("skip", "builtin"):
        for kw in (dict(max_windows="all"), dict(max_windows=5, windows_per_pass=3), dict(max_windows=2**31, windows_per_pass=2**31)):
            with pytest.raises(b2.B200PostError) as e:
                pr.generate_proof(d, bytes(32), su.PostConfig(), provider=b2.CPU_PROVIDER_ID, pow=pow_, **kw)
            assert e.value.code == b2.ERR_UNSUPPORTED, (pow_, kw)
            with pytest.raises(b2.B200PostError) as e:
                pr.generate_proof_checked(d, bytes(32), su.PostConfig(), providers=[b2.CPU_PROVIDER_ID] * 2, pow=pow_, **kw)
            assert e.value.code == b2.ERR_UNSUPPORTED, (pow_, kw)


def test_no_device_with_windows(b2, mods, tmp_path):
    su, pr, k2 = mods
    if b2.providers():
        pytest.skip("a CUDA device is present: the no-device contract is covered on CPU-only boxes")
    d = _post(su, tmp_path / "p")
    for pow_ in ("skip", "builtin"):
        for kw in (dict(max_windows="all"), dict(max_windows=3, windows_per_pass=2)):
            for call, extra in ((pr.generate_proof, {}), (pr.generate_proof, dict(providers=[0, 0])),
                                (pr.generate_proof_checked, dict(providers=[0, 1]))):
                with pytest.raises(b2.B200PostError) as e:
                    call(d, bytes(32), su.PostConfig(), pow=pow_, **kw, **extra)
                assert e.value.code == b2.ERR_NO_DEVICE, (pow_, kw, call)
    for provs in (None, [0, 0]):
        with pytest.raises(b2.B200PostError) as e:
            k2.search_group_range(bytes(8), bytes(32), EASY, 5, 3, providers=provs)
        assert e.value.code == b2.ERR_NO_DEVICE


def test_initial_proof_request_takes_any_window_count(b2, mods, tmp_path):
    """windows_per_pass is clamped to the windows below nonce 4096, never refused; max_windows is ignored."""
    su, pr, _ = mods
    mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=512, k1=26, k2=12, k3=12))
    mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(tmp_path / "p"), num_units=2, max_file_size=4096, provider_id=0,
                                             scrypt_n=2), NODE, ATX)
    for w in (0, 1, 3, 256, 2**32 - 1):
        mgr.request_initial_proof(nonces=32, pow="skip", windows_per_pass=w)
    opts, _ = pr._opts(None, None, 16, 0, "skip", "all", 2)
    assert su._bind().b200post_setup_request_initial_proof(mgr._h, ctypes.byref(opts)) == 0


def test_load_initial_proof_with_windows(b2, mods, tmp_path):
    """A file from a session that scanned W windows says so ("Windows": W, only when W > 1) and may hold any nonce below
    nonces * W; without the field the nonce must be below nonces, as before windows."""
    import base64
    import json
    su, pr, _ = mods
    d = tmp_path / "p"
    lpu, units, k1, k2, nonces = 512, 2, 26, 12, 32
    cfg = su.PostConfig(labels_per_unit=lpu, k1=k1, k2=k2, k3=k2)
    su.PostSetupManager(cfg).prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=units, max_file_size=4096,
                                                                  provider_id=0, scrypt_n=2), NODE, ATX)
    bits = (lpu * units).bit_length()

    def write(**over):
        doc = {"NodeId": base64.b64encode(NODE).decode(), "CommitmentAtxId": base64.b64encode(ATX).decode(), "NumUnits": units,
               "LabelsPerUnit": lpu, "K1": k1, "K2": k2, "Nonces": nonces, "PowDifficulty": bytes(pr._c_cfg(cfg).pow_difficulty).hex(),
               "Challenge": base64.b64encode(bytes(32)).decode(), "Nonce": 5,
               "Indices": base64.b64encode(bytes(range((k2 * bits + 7) // 8))).decode(), "Pow": 77}
        doc.update(over)
        (d / "initial_post.json").write_text(json.dumps(doc, indent=1))

    def code(**over):
        write(**over)
        try:
            return su.load_initial_proof(str(d), cfg, nonces)[0].nonce
        except b2.B200PostError as e:
            assert "no initial proof" in str(e)
            return e.code

    assert code(Nonce=31) == 31 and code(Nonce=32) == su.ERR_IO
    assert code(Nonce=95, Windows=3) == 95 and code(Nonce=96, Windows=3) == su.ERR_IO
    assert code(Nonce=4095, Windows=128) == 4095
    for bad in (0, 1, 129, "x"):
        assert code(Nonce=5, Windows=bad) == su.ERR_IO, bad
