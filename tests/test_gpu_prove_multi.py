"""GPU tier: proving on several devices (b200post_k2pow_search_groups_multi and b200post_generate_proof_multi) must give
exactly the one-device answer.

Every case runs on one H100 through repeated provider lists ([0, 0], [0, 0, 0]: the shards, or k2pow windows, share the
device, each with its own buffers), and on the real device list when the box has more than one GPU.

* k2pow: the smallest valid pow of every nonce group, whatever the number of devices and the order windows finish in,
  against the single-device search and the RandomX oracle.
* The scan over the four-unit, five-file POST of test_gpu_prove_matrix.py in its three regimes, at chunk sizes that put
  shard boundaries inside files and across file seams, against the single-device call and np_prove_multi.
* Synthetic POSTs (label files written by the test, hit labels planted where a case needs them): a proof straddling a
  shard boundary, a tie across shards, a first shard without any hit (per-shard saturation stop).
* Builtin k2pow end to end, the early stop, cancel, and a truncated last file."""
import contextlib
import ctypes
import importlib
import re
import shutil
import time
from pathlib import Path

import numpy as np
import pytest

from oracle import pyrandomx as orx

pytestmark = pytest.mark.gpu

LISTS = {"x1": [0], "x2": [0, 0], "x3": [0, 0, 0], "devices": None}   # None = every device, when there are several


@pytest.fixture(params=list(LISTS), ids=list(LISTS))
def plist(request, gpu_ready):
    ids = LISTS[request.param]
    if ids is None:
        if len(gpu_ready) < 2:
            pytest.skip("one GPU: the real device list is the x1 case")
        ids = [p["id"] for p in gpu_ready]
    return ids


@pytest.fixture(scope="module")
def mods(b2, gpu_ready):
    return (importlib.import_module("go-spacemesh_b200.setup"), importlib.import_module("go-spacemesh_b200.prove"),
            importlib.import_module("go-spacemesh_b200.verify"), importlib.import_module("go-spacemesh_b200.k2pow"))


@contextlib.contextmanager
def options(b2, **values):
    before = {k: b2.get_option(k) for k in values}
    try:
        for k, v in values.items():
            b2.set_option(k, v)
        yield
    finally:
        for k, v in before.items():
            b2.set_option(k, v)


def _scanned_total(b2) -> int:
    return int(re.search(r"^b200post_prove_labels_scanned_total (\S+)$", b2.metrics_text(), re.M).group(1))


def _shards(total: int, chunk: int, n: int):
    """The documented split: contiguous shards of whole chunks in list order, the earlier shards taking the odd chunks."""
    chunks = -(-total // chunk)
    q, r = divmod(chunks, n)
    out, first = [], 0
    for s in range(n):
        end = first + q + (1 if s < r else 0)
        out.append((min(total, first * chunk), min(total, end * chunk)))
        first = end
    return out


# ------------------------------------------------------------------------------------------------ k2pow groups
@pytest.fixture(scope="module")
def rx_oracle():
    c = orx.Cache(orx.K2POW_CACHE_KEY)
    c.init_dataset()
    yield c
    c.close()


def _rate(r: int) -> bytes:
    return (2**256 // r).to_bytes(32, "big")


GROUP_CASES = [   # (groups, 1 / pass rate, max_nonces_per_group); one VM per SM, so each group spans several windows
    (1, 300, 0),
    (18, 24, 0),
    (256, 4, 0),      # more groups than a batch holds: windows of one nonce per group, two launches each
    (5, 64, 40),      # the cap ends the search with groups still pending
]


@pytest.fixture(scope="module")
def single_groups(mods, b2, rx_oracle):
    """case -> (pows, hashes) of the single-device search, each pow checked against the oracle once."""
    k2 = mods[3]
    cache = {}

    def get(case):
        if case not in cache:
            n_groups, rate, cap = case
            r = np.random.default_rng(60 + GROUP_CASES.index(case))
            ch, node = bytes(r.integers(0, 256, 8, dtype=np.uint8)), bytes(r.integers(0, 256, 32, dtype=np.uint8))
            with options(b2, rx_vms_per_sm=1):
                pows, done = k2.search_groups(ch, node, _rate(rate), n_groups, cap)
            for g, pw in enumerate(pows):
                _, found, _ = rx_oracle.k2pow_scan(g, ch, node, 0, cap if pw is None else pw + 1, _rate(rate), want_hashes=False)
                assert found == pw, f"group {g}: GPU pow {pw}, smallest valid pow {found}"
            cache[case] = (ch, node, pows, done)
        return cache[case]
    return get


@pytest.mark.parametrize("case", GROUP_CASES, ids=[f"{c[0]}groups-1in{c[1]}-cap{c[2]}" for c in GROUP_CASES])
def test_search_groups_multi_equals_one_device(mods, b2, single_groups, plist, case):
    k2 = mods[3]
    n_groups, rate, cap = case
    ch, node, want, single_done = single_groups(case)
    before = b2.get_option("rx_vms_per_sm")
    with options(b2, rx_vms_per_sm=1):
        pows, done = k2.search_groups(ch, node, _rate(rate), n_groups, cap, providers=plist)
    assert b2.get_option("rx_vms_per_sm") == before
    assert pows == want
    if cap:
        assert None in pows and any(p is not None for p in pows)
    assert done >= single_done if len(plist) > 1 else done == single_done


# ------------------------------------------------------------------------------- the scan over a real POST
NODE, ATX = bytes(range(50, 82)), bytes(range(150, 182))
UNITS, LPU = 4, 1 << 20
NUM_LABELS = UNITS * LPU
PER_FILE = 1_000_003
PROOF_REGIMES = {                            # regime: (k1, k2, nonces, challenge), as in test_gpu_prove_matrix.py
    "mainnet": (26, 37, 288, bytes(range(90, 122))),
    "round": (1 << 17, 200, 16, bytes(range(1, 33))),
    "mid": (100003, 200, 16, bytes(range(2, 34))),
}
CHUNKS = ((1 << 20) + 13, 4099)


def _pow_of(group: int) -> int:
    return 2**55 + 977 * group


def _pow_callback(ctx, nonce_group, challenge8, difficulty, node_id, pow_out):
    pow_out[0] = _pow_of(nonce_group)
    return 0


@pytest.fixture(scope="module")
def post(mods, tmp_path_factory):
    """4 units x 2^20 labels at N = 2, in five files; (data dir, the labels read back)."""
    su = mods[0]
    mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=LPU, k1=26, k2=37, k3=37, max_num_units=8))
    o = su.PostSetupOpts(data_dir=str(tmp_path_factory.mktemp("post")), num_units=UNITS, max_file_size=16 * PER_FILE,
                         provider_id=0, scrypt_n=2, compute_batch_size=1 << 20)
    mgr.prepare_initializer(o, NODE, ATX)
    mgr.start_session()
    assert mgr.status().state == su.STATE_COMPLETE
    files = [Path(o.data_dir) / f"postdata_{i}.bin" for i in range(5)]
    labels = np.concatenate([np.fromfile(f, dtype=np.uint8) for f in files]).reshape(-1, 16)
    assert labels.shape[0] == NUM_LABELS
    return o.data_dir, labels


def _cfg(su, k1, k2, lpu=LPU, **kw):
    return su.PostConfig(labels_per_unit=lpu, k1=k1, k2=k2, k3=k2, max_num_units=8, **kw)


@pytest.fixture(scope="module")
def real_proofs(mods, post, orc):
    """regime -> (oracle proof, oracle indices, single-device proof at the default chunk)."""
    su, pr, vf, _ = mods
    data_dir, labels = post
    cache = {}

    def get(regime):
        if regime not in cache:
            k1, k2, nonces, challenge = PROOF_REGIMES[regime]
            nonce, idx = orc.np_prove_multi(labels, challenge, nonces, [_pow_of(g) for g in range(nonces // 16)], k1, k2,
                                            NUM_LABELS)
            assert nonce is not None
            want = vf.Proof(nonce, vf.pack_indices(idx, vf.bits_per_index(NUM_LABELS)), _pow_of(nonce // 16))
            single, _, _ = pr.generate_proof(data_dir, challenge, _cfg(su, k1, k2), nonces=nonces, pow=_pow_callback)
            assert single == want
            cache[regime] = (want, idx)
        return cache[regime]
    return get


@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("regime", PROOF_REGIMES)
def test_generate_proof_multi_equals_one_device_and_oracle(mods, b2, post, real_proofs, plist, regime, chunk):
    su, pr, vf, _ = mods
    data_dir, _ = post
    k1, k2, nonces, challenge = PROOF_REGIMES[regime]
    want, idx = real_proofs(regime)
    single, _, single_scanned = pr.generate_proof(data_dir, challenge, _cfg(su, k1, k2), nonces=nonces, chunk_labels=chunk,
                                                  pow=_pow_callback)
    assert single == want
    before = _scanned_total(b2)
    proof, meta, scanned = pr.generate_proof(data_dir, challenge, _cfg(su, k1, k2), nonces=nonces, chunk_labels=chunk,
                                             pow=_pow_callback, providers=plist)
    assert _scanned_total(b2) - before == scanned
    assert proof == want
    assert idx[-1] < scanned <= NUM_LABELS
    if len(plist) == 1:
        assert scanned == single_scanned
    assert meta == vf.ProofMetadata(NODE, ATX, challenge, UNITS, LPU)
    v = vf.PostVerifier(pow="skip")
    try:
        v.verify(proof, meta, vf.VerifyParams(k1=k1, k2=k2, scrypt_n=2))
    finally:
        v.close()


def test_no_proof_from_either_call(mods, b2, post, orc):
    su, pr, _, _ = mods
    data_dir, labels = post
    k1, k2, nonces, challenge = 26, 278, 288, bytes(range(90, 122))
    assert orc.np_prove_multi(labels, challenge, nonces, [_pow_of(g) for g in range(nonces // 16)], k1, k2,
                              NUM_LABELS) == (None, None)
    for kw in ({}, {"providers": [0, 0]}, {"providers": [0, 0, 0]}):
        with pytest.raises(b2.B200PostError) as e:
            pr.generate_proof(data_dir, challenge, _cfg(su, k1, k2), nonces=nonces, chunk_labels=4099, pow=_pow_callback, **kw)
        assert e.value.code == b2.ERR_INVALID_PROOF and "no proof found" in str(e.value), kw


def test_early_decision_stops_every_shard(mods, post, orc):
    """Round difficulty (1 label in 32 passes per nonce), K2 = 20: shard 0 decides the proof in its first chunk, and
    the other shards stop within their first chunks (decided, or saturated on their own)."""
    su, pr, _, _ = mods
    data_dir, labels = post
    k1, k2, nonces, challenge, chunk = 1 << 17, 20, 16, bytes(range(5, 37)), 4099
    nonce, idx = orc.np_prove_multi(labels[:chunk], challenge, nonces, [_pow_of(0)], k1, k2, NUM_LABELS)
    assert nonce is not None
    single, _, _ = pr.generate_proof(data_dir, challenge, _cfg(su, k1, k2), nonces=nonces, chunk_labels=chunk, pow=_pow_callback)
    for plist in ([0, 0], [0, 0, 0]):
        proof, _, scanned = pr.generate_proof(data_dir, challenge, _cfg(su, k1, k2), nonces=nonces, chunk_labels=chunk,
                                              pow=_pow_callback, providers=plist)
        assert proof == single and proof.nonce == nonce
        assert idx[-1] < scanned <= 2 * chunk * len(plist) < NUM_LABELS // 100, (plist, scanned)


# ------------------------------------------------------------------------------------------- synthetic POSTs
LPU_S, UNITS_S, PER_FILE_S, CHUNK_S = 1 << 16, 3, 50_001, 4099
NUM_S = LPU_S * UNITS_S
ROUND_S = (NUM_S // 32, 16)                   # k1 for a round difficulty (MSB 0x08, lsb 0), nonces


def _write_post(su, d: Path, labels: np.ndarray) -> str:
    """Metadata of a 3 x 2^16-label POST, then label files holding exactly `labels` (the prover trusts stored bytes)."""
    assert labels.shape == (NUM_S, 16)
    o = su.PostSetupOpts(data_dir=str(d), num_units=UNITS_S, max_file_size=16 * PER_FILE_S, provider_id=0, scrypt_n=2)
    su.PostSetupManager(_cfg(su, 26, 37, LPU_S)).prepare_initializer(o, NODE, ATX)
    for f in range(-(-NUM_S // PER_FILE_S)):
        (d / f"postdata_{f}.bin").write_bytes(labels[f * PER_FILE_S:(f + 1) * PER_FILE_S].tobytes())
    return str(d)


@pytest.fixture(scope="module")
def pool(orc):
    """Random labels and, per label, the set of nonces it is a hit for at the round difficulty."""
    k1, nonces = ROUND_S
    labels = np.random.default_rng(77).integers(0, 256, (20000, 16), dtype=np.uint8)
    challenge = bytes(range(11, 43))
    hits = orc.np_prove_hits(labels, challenge, nonces, [_pow_of(0)], k1, len(labels), NUM_S)
    sets = [set() for _ in range(len(labels))]
    for n, pos in hits.items():
        for i in pos:
            sets[int(i)].add(n)
    filler = labels[next(i for i, s in enumerate(sets) if not s)]
    return labels, sets, filler, challenge


def _prove_both(pr, su, data_dir, challenge, k1, k2, plist, nonces=16):
    single = pr.generate_proof(data_dir, challenge, _cfg(su, k1, k2, LPU_S), nonces=nonces, chunk_labels=CHUNK_S,
                               pow=_pow_callback)
    multi = pr.generate_proof(data_dir, challenge, _cfg(su, k1, k2, LPU_S), nonces=nonces, chunk_labels=CHUNK_S,
                              pow=_pow_callback, providers=plist)
    return single, multi


@pytest.mark.parametrize("n", [2, 3])
def test_proof_straddles_a_shard_boundary(mods, orc, tmp_path, n):
    """Random labels at a MSB-0 difficulty.  The nonce with the most hits in shard 0 gets one of its hit labels copied
    just past the boundary, and K2 is one more than that count: the proof needs hits from both shards."""
    su, pr, vf, _ = mods
    k1, nonces = 100, 16
    challenge = bytes(range(20, 52))
    labels = np.random.default_rng(n).integers(0, 256, (NUM_S, 16), dtype=np.uint8)
    boundary = _shards(NUM_S, CHUNK_S, n)[0][1]
    first = orc.np_prove_hits(labels[:boundary], challenge, nonces, [_pow_of(0)], k1, boundary, NUM_S)
    lead = max(first, key=lambda m: len(first[m]))
    k2 = len(first[lead]) + 1
    labels[boundary + 5] = labels[first[lead][0]]
    nonce, idx = orc.np_prove_multi(labels, challenge, nonces, [_pow_of(0)], k1, k2, NUM_S)
    assert nonce is not None and idx[0] < boundary <= idx[-1]
    data_dir = _write_post(su, tmp_path, labels)
    (single, _, _), (proof, _, scanned) = _prove_both(pr, su, data_dir, challenge, k1, k2, [0] * n)
    assert (proof.nonce, vf.unpack_indices(proof.indices, vf.bits_per_index(NUM_S), k2)) == (nonce, idx)
    assert proof == single and idx[-1] < scanned <= NUM_S


@pytest.mark.parametrize("n", [2, 3])
def test_tie_across_shards_goes_to_the_lower_nonce(mods, orc, pool, tmp_path, n):
    """K2 = 2.  Nonce a's first hit is in shard 0, nonce b's (b > a) in shard 1, and one label later in shard 1 is the
    second hit of both: a tie at the K2-th index, which the lower nonce must win with its own two indices."""
    su, pr, vf, _ = mods
    k1, nonces = ROUND_S
    plabels, sets, filler, challenge = pool
    ab = next(i for i, s in enumerate(sets) if len(s) == 2)
    a, b = sorted(sets[ab])
    only_a = next(i for i, s in enumerate(sets) if s == {a})
    only_b = next(i for i, s in enumerate(sets) if s == {b})
    boundary = _shards(NUM_S, CHUNK_S, n)[1][0]
    labels = np.tile(filler, (NUM_S, 1))
    labels[10], labels[boundary + 10], labels[boundary + 20] = plabels[only_a], plabels[only_b], plabels[ab]
    nonce, idx = orc.np_prove_multi(labels, challenge, nonces, [_pow_of(0)], k1, 2, NUM_S)
    assert (nonce, idx) == (a, [10, boundary + 20])
    data_dir = _write_post(su, tmp_path, labels)
    (single, _, _), (proof, _, _) = _prove_both(pr, su, data_dir, challenge, k1, 2, [0] * n)
    assert (proof.nonce, vf.unpack_indices(proof.indices, vf.bits_per_index(NUM_S), 2)) == (a, [10, boundary + 20])
    assert proof == single


def test_saturated_shards_stop_on_their_own(mods, orc, pool, tmp_path):
    """Shard 0 holds no hit, so nothing is decided before it is scanned to its end.  Shards 1 and 2 hold random labels:
    every nonce reaches K2 hits early in each, and each must stop within two chunks of that point instead of scanning on
    until shard 0 is done."""
    su, pr, vf, _ = mods
    k1, nonces = ROUND_S
    _, _, filler, challenge = pool
    k2 = 4
    shards = _shards(NUM_S, CHUNK_S, 3)
    labels = np.random.default_rng(5).integers(0, 256, (NUM_S, 16), dtype=np.uint8)
    labels[:shards[0][1]] = filler
    bound = shards[0][1] - shards[0][0]
    for lo, hi in shards[1:]:
        hits = orc.np_prove_hits(labels[lo:hi], challenge, nonces, [_pow_of(0)], k1, k2, NUM_S)
        assert all(len(h) == k2 for h in hits.values())
        sat = max(int(h[-1]) for h in hits.values()) + 1          # labels of the shard up to its saturation point
        bound += min(hi - lo, sat + 2 * CHUNK_S)
        assert sat + 2 * CHUNK_S < (hi - lo) // 2
    nonce, idx = orc.np_prove_multi(labels, challenge, nonces, [_pow_of(0)], k1, k2, NUM_S)
    data_dir = _write_post(su, tmp_path, labels)
    (single, _, _), (proof, _, scanned) = _prove_both(pr, su, data_dir, challenge, k1, k2, [0, 0, 0])
    assert (proof.nonce, vf.unpack_indices(proof.indices, vf.bits_per_index(NUM_S), k2)) == (nonce, idx)
    assert proof == single
    assert shards[0][1] <= scanned <= bound, (scanned, bound)


# ------------------------------------------------------------------------------- builtin k2pow, cancel, errors
def test_builtin_pow_end_to_end(mods, b2, post):
    su, pr, vf, _ = mods
    data_dir, _ = post
    k1, k2, nonces, challenge = 100003, 200, 32, bytes(range(2, 34))
    pow_difficulty = bytes([0x30]) + bytes(range(101, 132))
    cfg = _cfg(su, k1, k2, pow_difficulty=pow_difficulty)
    with options(b2, rx_vms_per_sm=1):
        single, meta, _ = pr.generate_proof(data_dir, challenge, cfg, nonces=nonces, chunk_labels=4099)
        proof, _, _ = pr.generate_proof(data_dir, challenge, cfg, nonces=nonces, chunk_labels=4099, providers=[0, 0])
    assert proof == single
    v = vf.PostVerifier()
    try:
        v.verify(proof, meta, vf.VerifyParams(k1=k1, k2=k2, scrypt_n=2, pow_difficulty=pow_difficulty))
    finally:
        v.close()


def test_cancel_during_the_scan(mods, b2, post, real_proofs):
    """The pow hook raises the cancel flag after the last group, so the scan starts cancelled: every shard sees it at its
    first poll.  A following call on the same device succeeds."""
    su, pr, _, _ = mods
    data_dir, _ = post
    k1, k2, nonces, challenge = PROOF_REGIMES["mainnet"]
    flag = ctypes.c_int(0)

    def hook(ctx, nonce_group, challenge8, difficulty, node_id, pow_out):
        pow_out[0] = _pow_of(nonce_group)
        if nonce_group == nonces // 16 - 1:
            flag.value = 1
        return 0

    for plist in ([0, 0], [0, 0, 0]):
        flag.value = 0
        t0 = time.perf_counter()
        with pytest.raises(b2.B200PostError) as e:
            pr.generate_proof(data_dir, challenge, _cfg(su, k1, k2), nonces=nonces, chunk_labels=4099, pow=hook,
                              providers=plist, cancel=flag)
        assert e.value.code == b2.ERR_CANCELLED and flag.value == 1
        assert time.perf_counter() - t0 < 30
        proof, _, _ = pr.generate_proof(data_dir, challenge, _cfg(su, k1, k2), nonces=nonces, chunk_labels=4099,
                                        pow=_pow_callback, providers=[0])
        assert proof == real_proofs("mainnet")[0]


def test_truncated_last_file_fails_the_call(mods, b2, post, real_proofs, tmp_path):
    """No nonce reaches K2 = 278, so the last shard reaches the end of the last file, which is 1001 labels short: the
    call fails with ERR_IO once every shard has joined, and the device stays usable."""
    su, pr, _, _ = mods
    data_dir, _ = post
    d = tmp_path / "short"
    shutil.copytree(data_dir, d)
    last = d / "postdata_4.bin"
    last.write_bytes(last.read_bytes()[:-16 * 1001])
    k1, _, nonces, challenge = PROOF_REGIMES["mainnet"]
    for plist in ([0, 0], [0, 0, 0]):
        with pytest.raises(b2.B200PostError) as e:
            pr.generate_proof(str(d), challenge, _cfg(su, k1, 278), nonces=nonces, chunk_labels=4099, pow=_pow_callback,
                              providers=plist)
        assert e.value.code == su.ERR_IO and "short read" in str(e.value), plist
    k1, k2, nonces, challenge = PROOF_REGIMES["round"]
    proof, _, _ = pr.generate_proof(data_dir, challenge, _cfg(su, k1, k2), nonces=nonces, chunk_labels=4099,
                                    pow=_pow_callback, providers=[0, 0, 0])
    assert proof == real_proofs("round")[0]
