"""GPU tier: proving over further nonce windows (b200post_prove_opts.max_windows / windows_per_pass).

POSTs are written by setup sessions (N = 2, one case at N = 8192).  Challenges come from a seeded RNG, chosen with the
windowed oracle (tests/window_oracle.py) so that windows 0 .. k-1 hold no proof and window k does.  The proof must be
the oracle's from window k for every windows_per_pass, device list and chunk size; the pow that of its nonce group."""
import ctypes
import importlib
import json
import re
import shutil
from pathlib import Path

import numpy as np
import pytest

import window_oracle as wo

pytestmark = pytest.mark.gpu

NODE, ATX = bytes(range(3, 35)), bytes(range(90, 122))
ZERO = bytes(32)
LPU, UNITS, PER_FILE = 1 << 14, 2, 10_007
NUM = LPU * UNITS
K1, K2, NONCES = 26, 37, 16                 # mainnet K1/K2, go-spacemesh's default nonce count
CHUNK = 4099
EASY = b"\x0f" + b"\xff" * 31


def _pow_of(g: int) -> int:
    return 1000 + g


def _callback(calls=None):
    def pow_(ctx, group, ch, diff, node, out):
        if calls is not None:
            calls.append(group)
        out[0] = _pow_of(group)
        return 0
    return pow_


@pytest.fixture(scope="module")
def mods(b2, gpu_ready):
    return (importlib.import_module("go-spacemesh_b200.setup"), importlib.import_module("go-spacemesh_b200.prove"),
            importlib.import_module("go-spacemesh_b200.verify"), importlib.import_module("go-spacemesh_b200.k2pow"))


def _cfg(su, lpu=LPU, **kw):
    return su.PostConfig(labels_per_unit=lpu, k1=K1, k2=K2, k3=K2, max_num_units=8, **kw)


def _write_setup(su, d: Path, n, lpu=LPU, units=UNITS, per_file=PER_FILE, node=NODE):
    o = su.PostSetupOpts(data_dir=str(d), num_units=units, max_file_size=16 * per_file, provider_id=0, scrypt_n=n,
                         compute_batch_size=1 << 12)
    mgr = su.PostSetupManager(_cfg(su, lpu))
    mgr.prepare_initializer(o, node, ATX)
    mgr.start_session()
    assert mgr.status().state == su.STATE_COMPLETE
    files = sorted(d.glob("postdata_*.bin"), key=lambda p: int(p.stem.split("_")[1]))
    return np.concatenate([np.fromfile(f, dtype=np.uint8) for f in files]).reshape(-1, 16)


def _pick_challenge(orc, labels, seed, pow_of=_pow_of, lo=2, hi=6, num=NUM):
    """A challenge whose first proof is in window k, lo <= k <= hi: (challenge, (k, nonce, indices))."""
    rng = np.random.default_rng(seed)
    for _ in range(400):
        ch = rng.bytes(32)
        got = wo.windowed_proof(orc, labels, ch, NONCES, pow_of, K1, K2, num, hi + 1)
        if got and got[0] >= lo:
            return ch, got
    raise AssertionError("no challenge found")


@pytest.fixture(scope="module")
def base(mods, orc, tmp_path_factory):
    """The N = 2 POST: (data dir, labels, challenge, (k, nonce, indices))."""
    su = mods[0]
    d = tmp_path_factory.mktemp("post")
    stored = _write_setup(su, d, 2)
    real, _, _, _ = orc.c_labels_range(orc.c_commitment(NODE, ATX), 2, 0, NUM)
    assert (stored == real).all()
    ch, want = _pick_challenge(orc, real, 11)
    return str(d), real, ch, want


def _counter(b2, name) -> int:
    return int(re.search(rf"^{name} (\S+)$", b2.metrics_text(), re.M).group(1))


def _unpack(vf, proof, num=NUM):
    return vf.unpack_indices(proof.indices, vf.bits_per_index(num), K2)


def _verify_both(orc, vf, proof, meta, challenge, n=2, lpu=LPU, **kw):
    assert orc.py_verify(proof.nonce, proof.indices, proof.pow, NODE, ATX, challenge, UNITS, lpu, K1, K2, n) == (True, None)
    v = vf.PostVerifier(pow=kw.pop("pow", "skip"))
    try:
        v.verify(proof, meta, vf.VerifyParams(k1=K1, k2=K2, scrypt_n=n, **kw))
    finally:
        v.close()


# ------------------------------------------------------------------------------------------------ the window rule
def test_all_windows_finds_the_first_window_with_a_proof(mods, b2, orc, base):
    su, pr, vf, _ = mods
    d, real, ch, (k, nonce, idx) = base
    calls = []
    proof, meta, _ = pr.generate_proof(d, ch, _cfg(su), nonces=NONCES, chunk_labels=CHUNK, pow=_callback(calls), max_windows="all")
    assert (proof.nonce, _unpack(vf, proof)) == (nonce, idx) and k * NONCES <= nonce < (k + 1) * NONCES
    assert proof.pow == _pow_of(nonce // 16)
    assert calls == list(range((k + 1) * NONCES // 16))          # one pow per group of every window tried
    _verify_both(orc, vf, proof, meta, ch)
    # k windows hold no proof
    with pytest.raises(b2.B200PostError) as e:
        pr.generate_proof(d, ch, _cfg(su), nonces=NONCES, chunk_labels=CHUNK, pow=_callback(), max_windows=k, windows_per_pass=2)
    assert e.value.code == b2.ERR_INVALID_PROOF and str(e.value).find("no proof found") >= 0
    assert f"windows 0..{k - 1}" in str(e.value)
    # one window: today's behaviour
    with pytest.raises(b2.B200PostError) as e:
        pr.generate_proof(d, ch, _cfg(su), nonces=NONCES, chunk_labels=CHUNK, pow=_callback())
    assert e.value.code == b2.ERR_INVALID_PROOF and "no proof found" in str(e.value)


@pytest.mark.parametrize("per_pass", ["1", "2", "k", "k+1", "64"])
def test_windows_per_pass_gives_the_same_proof(mods, b2, base, per_pass):
    su, pr, vf, _ = mods
    d, real, ch, (k, nonce, idx) = base
    m = {"1": 1, "2": 2, "k": k, "k+1": k + 1, "64": 64}[per_pass]
    ref, _, _ = pr.generate_proof(d, ch, _cfg(su), nonces=NONCES, chunk_labels=CHUNK, pow=_callback(), max_windows="all")
    before = _counter(b2, "b200post_prove_passes_total")
    proof, _, scanned = pr.generate_proof(d, ch, _cfg(su), nonces=NONCES, chunk_labels=CHUNK, pow=_callback(), max_windows="all",
                                          windows_per_pass=m)
    passes = _counter(b2, "b200post_prove_passes_total") - before
    assert proof == ref
    assert passes == k // m + 1
    last = scanned - (passes - 1) * NUM                          # the earlier passes read every label
    assert idx[-1] < last <= NUM
    if k % m:                                                    # window k is not its pass's lowest: no early stop
        assert last == NUM


@pytest.mark.parametrize("plist", ([0], [0, 0], [0, 0, 0]), ids=["x1", "x2", "x3"])
@pytest.mark.parametrize("chunk", [CHUNK, 1 << 14])
def test_device_lists_and_chunks_give_the_same_proof(mods, base, plist, chunk):
    su, pr, vf, _ = mods
    d, real, ch, (k, nonce, idx) = base
    for per_pass in (1, 3):
        proof, _, _ = pr.generate_proof(d, ch, _cfg(su), nonces=NONCES, chunk_labels=chunk, pow=_callback(), providers=plist,
                                        max_windows="all", windows_per_pass=per_pass)
        assert (proof.nonce, _unpack(vf, proof), proof.pow) == (nonce, idx, _pow_of(nonce // 16)), (plist, chunk, per_pass)
        proof, _, _, rep = pr.generate_proof_checked(d, ch, _cfg(su), nonces=NONCES, chunk_labels=chunk, pow=_callback(),
                                                     providers=plist, max_windows="all", windows_per_pass=per_pass)
        assert (proof.nonce, _unpack(vf, proof)) == (nonce, idx) and rep.proof_verified and rep.damaged == 0


# ------------------------------------------------------------------------------------------------ damaged data
def test_checked_drops_a_forged_window_zero_winner(mods, b2, orc, base, tmp_path):
    """K2 forged hits of a window-0 nonce at the lowest indices: the unchecked call proves with them in window 0; the
    checked call drops and reports them and proves from the first window with K2 usable hits."""
    su, pr, vf, _ = mods
    d0, real, ch, _ = base
    n = 7
    blocks = np.random.default_rng(77).integers(0, 256, (1_000_000, 16), dtype=np.uint8)
    fh = wo.window_hits(orc, blocks, ch, 0, NONCES, [_pow_of(0)], K1, K2, NUM)[n]
    assert len(fh) == K2
    d = tmp_path / "p"
    shutil.copytree(d0, d)
    stored = real.copy()
    stored[:K2] = blocks[fh]
    (d / "postdata_0.bin").write_bytes(stored[:PER_FILE].tobytes())
    ok = (stored == real).all(axis=1)
    want = wo.windowed_proof(orc, stored, ch, NONCES, _pow_of, K1, K2, NUM, 4096 // NONCES, usable=ok, k2_hits=4 * K2)
    assert want is not None and want[0] >= 1
    unchecked, meta, _ = pr.generate_proof(str(d), ch, _cfg(su), nonces=NONCES, chunk_labels=CHUNK, pow=_callback(), max_windows="all")
    assert (unchecked.nonce, _unpack(vf, unchecked)) == (n, list(range(K2)))
    for plist in ([0], [0, 0]):
        for per_pass in (1, 2, want[0] + 1):
            proof, meta, _, rep = pr.generate_proof_checked(str(d), ch, _cfg(su), nonces=NONCES, chunk_labels=CHUNK, pow=_callback(),
                                                            providers=plist, max_windows="all", windows_per_pass=per_pass)
            assert (proof.nonce, _unpack(vf, proof)) == want[1:], (plist, per_pass)
            assert rep.damaged_index == list(range(K2)) and rep.damaged == K2 and rep.proof_verified, (plist, per_pass)
    _verify_both(orc, vf, proof, meta, ch)


# ------------------------------------------------------------------------------------------------ k2pow
def test_group_range_equals_search_groups(mods):
    _, _, _, k2 = mods
    scaled = k2.scale_difficulty(EASY, UNITS)
    ch = bytes(range(200, 208))
    full, _ = k2.search_groups(ch, NODE, scaled, 8)
    for provs in (None, [0, 0]):
        part, done = k2.search_group_range(ch, NODE, scaled, 5, 3, providers=provs)
        assert part == full[5:8] and done > 0, provs
    top, _ = k2.search_group_range(ch, NODE, scaled, 250, 6)
    assert all(p is not None for p in top)
    for g, p in zip(range(250, 256), top):
        assert k2.verify(p, g, ch, NODE, scaled)


def test_builtin_pow_windowed_proof_passes_the_verifier(mods, orc, base):
    su, pr, vf, k2 = mods
    d, real, _, _ = base
    scaled = k2.scale_difficulty(EASY, UNITS)
    cfg = _cfg(su, pow_difficulty=EASY)
    rng = np.random.default_rng(5)
    for _ in range(40):
        ch = rng.bytes(32)
        pows, _ = k2.search_groups(ch[:8], NODE, scaled, 8)                # the groups of windows 0 .. 7
        got = wo.windowed_proof(orc, real, ch, NONCES, lambda g: pows[g], K1, K2, NUM, len(pows))
        if got and got[0] >= 1:
            break
    else:
        raise AssertionError("no challenge found")
    proof, meta, _ = pr.generate_proof(d, ch, cfg, nonces=NONCES, chunk_labels=CHUNK, max_windows="all", windows_per_pass=2)
    assert (proof.nonce, _unpack(vf, proof), proof.pow) == (got[1], got[2], pows[got[1] // 16])
    checked, _, _, rep = pr.generate_proof_checked(d, ch, cfg, nonces=NONCES, chunk_labels=CHUNK, max_windows="all", providers=[0, 0])
    assert checked == proof and rep.proof_verified
    _verify_both(orc, vf, proof, meta, ch, pow="builtin", pow_difficulty=EASY)


# ------------------------------------------------------------------------------------------------ N = 8192
def test_n8192_all_windows(mods, orc, tmp_path):
    su, pr, vf, _ = mods
    lpu = 1 << 13
    num = lpu * UNITS
    stored = _write_setup(su, tmp_path / "p", 8192, lpu=lpu, per_file=5003)
    sample = np.array([0, 1, 5002, 5003, num - 1], dtype=np.uint64)
    comm = np.tile(np.frombuffer(orc.c_commitment(NODE, ATX), dtype=np.uint8), (len(sample), 1))
    assert (orc.c_labels_gather(comm, sample, 8192) == stored[sample.astype(np.int64)]).all()
    ch, (k, nonce, idx) = _pick_challenge(orc, stored, 3, num=num, lo=1)
    for per_pass in (1, k + 1):
        proof, meta, _ = pr.generate_proof(str(tmp_path / "p"), ch, _cfg(su, lpu), nonces=NONCES, pow=_callback(), max_windows="all",
                                           windows_per_pass=per_pass)
        assert (proof.nonce, _unpack(vf, proof, num), proof.pow) == (nonce, idx, _pow_of(nonce // 16))
    _verify_both(orc, vf, proof, meta, ch, n=8192, lpu=lpu)


# ------------------------------------------------------------------------------------------------ initial proof
def _session(su, d, request, node, cancel=None):
    """prepare + request + start; with `cancel` (set by the request's pow hook) the session must stop."""
    mgr = su.PostSetupManager(_cfg(su))
    mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=UNITS, max_file_size=16 * LPU, provider_id=0, scrypt_n=2,
                                             compute_batch_size=1 << 12), node, ATX)
    mgr.request_initial_proof(**request)
    if cancel is None:
        mgr.start_session()
        return mgr
    with pytest.raises(Exception) as e:
        mgr.start_session(cancel)
    assert e.value.code == 5   # ERR_CANCELLED
    return mgr


def test_initial_proof_over_three_windows(mods, orc, tmp_path):
    su, pr, vf, _ = mods
    # an identity whose zero challenge has no proof in window 0 and one in window 1 or 2
    for s in range(64):
        node = bytes([s]) + NODE[1:]
        labels, _, _, _ = orc.c_labels_range(orc.c_commitment(node, ATX), 2, 0, NUM)
        got = wo.windowed_proof(orc, labels, ZERO, NONCES, _pow_of, K1, K2, NUM, 3)
        if got and got[0] >= 1:
            break
    else:
        raise AssertionError("no identity found")
    req = dict(nonces=NONCES, pow=_callback(), windows_per_pass=3)
    d = tmp_path / "w3"
    mgr = _session(su, d, req, node)
    proof, meta, _ = mgr.initial_proof()
    assert (proof.nonce, _unpack(vf, proof), proof.pow) == (got[1], got[2], _pow_of(got[1] // 16))
    ref, _, _ = pr.generate_proof(str(d), ZERO, _cfg(su), nonces=NONCES, pow=_callback(), max_windows=3)
    assert (proof.nonce, proof.indices, proof.pow) == (ref.nonce, ref.indices, ref.pow)
    loaded, _, _ = su.load_initial_proof(str(d), _cfg(su), NONCES)
    assert (loaded.nonce, loaded.indices, loaded.pow) == (proof.nonce, proof.indices, proof.pow)
    doc = json.loads((d / "initial_post.json").read_text())
    assert doc["Windows"] == 3 and doc["Nonce"] == proof.nonce
    # stopped right after the pows (the hook raises the cancel flag at the last group) and resumed: the state's pows
    # (the 3 windows' groups) are used, and the file is the same
    half, flag = tmp_path / "half", ctypes.c_int(0)

    def stopping(ctx, group, ch, diff, node_, out):
        out[0] = _pow_of(group)
        if group == 3 * NONCES // 16 - 1:
            flag.value = 1
        return 0

    _session(su, half, dict(req, pow=stopping), node, cancel=flag)
    assert (half / "initial_post.scan").exists() and not (half / "initial_post.json").exists()
    calls = []
    _session(su, half, dict(req, pow=_callback(calls)), node)
    assert calls == []
    assert (half / "initial_post.json").read_bytes() == (d / "initial_post.json").read_bytes()
    # one window: no proof for this identity, and no count in the state header
    one = tmp_path / "one"
    mgr = _session(su, one, dict(nonces=NONCES, pow=_callback(), windows_per_pass=1), node)
    with pytest.raises(Exception) as e:
        mgr.initial_proof()
    assert e.value.code == 7 and "no proof found" in str(e.value) and "windows" not in str(e.value)
    state3, state1 = (d / "initial_post.scan").read_bytes(), (one / "initial_post.scan").read_bytes()
    assert state3[:180] == state1[:180] and state3[180:184] == (3).to_bytes(4, "little")
