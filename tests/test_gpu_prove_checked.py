"""GPU tier: proving over damaged POST data (b200post_generate_proof_checked).

A usable hit is a stored label that passes a nonce's difficulty AND equals its real label.  The checked proof is the
selection rule over usable hits only, for every device list and chunk size; on clean data it is the unchecked proof.

POSTs are written by a setup session at N = 2 (one case at N = 8192); real labels come from the C oracle; damage is
planted by rewriting rows of postdata_N.bin.  A forged hit for nonce n is a random 16-byte block that passes n, found
among 10^6 random blocks (the pass rate is K1 / numLabels).  The expected proof comes from `_oracle_checked`:
np_prove_hits over the stored rows, restricted to rows equal to the real ones, under the same selection rule."""
import ctypes
import importlib
import re
import shutil
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NODE, ATX = bytes(range(60, 92)), bytes(range(160, 192))
LPU, UNITS, PER_FILE = 1 << 16, 3, 50_001
NUM = LPU * UNITS
K1, K2, NONCES = 100, 20, 32
CH = bytes(range(40, 72))
POWS = [0] * (NONCES // 16)
LISTS = ([0], [0, 0], [0, 0, 0])
CHUNKS = (4099, 1 << 16, 0)          # 0 = the default chunk (the whole POST here)


@pytest.fixture(scope="module")
def mods(b2, gpu_ready):
    return (importlib.import_module("go-spacemesh_b200.setup"), importlib.import_module("go-spacemesh_b200.prove"),
            importlib.import_module("go-spacemesh_b200.verify"))


def _cfg(su, k1=K1, k2=K2, lpu=LPU, **kw):
    return su.PostConfig(labels_per_unit=lpu, k1=k1, k2=k2, k3=k2, max_num_units=8, **kw)


def _write_setup(su, d: Path, units, lpu, per_file, n):
    o = su.PostSetupOpts(data_dir=str(d), num_units=units, max_file_size=16 * per_file, provider_id=0, scrypt_n=n,
                         compute_batch_size=1 << 16)
    mgr = su.PostSetupManager(_cfg(su, lpu=lpu))
    mgr.prepare_initializer(o, NODE, ATX)
    mgr.start_session()
    assert mgr.status().state == su.STATE_COMPLETE
    files = sorted(d.glob("postdata_*.bin"), key=lambda p: int(p.stem.split("_")[1]))
    return np.concatenate([np.fromfile(f, dtype=np.uint8) for f in files]).reshape(-1, 16)


@pytest.fixture(scope="module")
def base(mods, orc, tmp_path_factory):
    """The clean N = 2 POST: (data dir, real labels)."""
    su = mods[0]
    d = tmp_path_factory.mktemp("clean")
    stored = _write_setup(su, d, UNITS, LPU, PER_FILE, 2)
    real, _, _, _ = orc.c_labels_range(orc.c_commitment(NODE, ATX), 2, 0, NUM)
    assert (stored == real).all()
    return str(d), real


def _damage(base_dir: str, d: Path, real: np.ndarray, rows: dict, per_file=PER_FILE):
    """A copy of the POST with rows {index: 16 bytes} rewritten; returns (data dir, stored labels)."""
    shutil.copytree(base_dir, d)
    stored = real.copy()
    for i, v in rows.items():
        stored[i] = np.frombuffer(bytes(v), dtype=np.uint8)
    for f in sorted({i // per_file for i in rows}):
        (d / f"postdata_{f}.bin").write_bytes(stored[f * per_file:(f + 1) * per_file].tobytes())
    return str(d), stored


def _oracle_checked(orc, stored, real, nonces, pows, k1, k2, num, challenge=CH):
    """The selection rule over usable hits: (nonce, indices) or (None, None)."""
    ok = (stored == real).all(axis=1)
    best = None
    for n, hits in orc.np_prove_hits(stored, challenge, nonces, pows, k1, len(stored), num).items():
        usable = [int(i) for i in hits if ok[i]][:k2]
        if len(usable) == k2 and (best is None or usable[-1] < best[1][-1]):
            best = (n, usable)
    return best or (None, None)


@pytest.fixture(scope="module")
def forged(orc):
    """nonce -> random blocks that pass it (K1, NUM, CH, pow 0), and one block that passes no nonce."""
    blocks = np.random.default_rng(1234).integers(0, 256, (1_000_000, 16), dtype=np.uint8)
    hits = orc.np_prove_hits(blocks, CH, NONCES, POWS, K1, len(blocks), NUM)
    out = {n: blocks[h] for n, h in hits.items()}
    any_hit = np.zeros(len(blocks), bool)
    for h in hits.values():
        any_hit[h] = True
    out["none"] = blocks[np.flatnonzero(~any_hit)[0]]
    assert all(len(out[n]) >= 200 for n in range(NONCES))
    return out


def _unpack(vf, proof, k2, num=NUM):
    return proof.nonce, vf.unpack_indices(proof.indices, vf.bits_per_index(num), k2)


def _verify(vf, proof, meta, k1=K1, k2=K2, n=2, **kw):
    v = vf.PostVerifier(pow="skip")
    try:
        v.verify(proof, meta, vf.VerifyParams(k1=k1, k2=k2, scrypt_n=n, **kw))
    finally:
        v.close()


def _counter(b2, name) -> int:
    return int(re.search(rf"^{name} (\S+)$", b2.metrics_text(), re.M).group(1))


def _checked(pr, su, d, plist=(0,), chunk=4099, k1=K1, k2=K2, nonces=NONCES, lpu=LPU, **kw):
    return pr.generate_proof_checked(d, CH, _cfg(su, k1, k2, lpu), providers=list(plist), nonces=nonces, chunk_labels=chunk,
                                     pow=kw.pop("pow", "skip"), **kw)


# --------------------------------------------------------------------------------------------------- clean data
@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("plist", LISTS, ids=["x1", "x2", "x3"])
def test_clean_data_gives_the_unchecked_proof(mods, orc, base, plist, chunk):
    su, pr, vf = mods
    d, real = base
    unchecked, _, _ = pr.generate_proof(d, CH, _cfg(su), providers=plist, nonces=NONCES, chunk_labels=chunk, pow="skip")
    proof, meta, scanned, rep = _checked(pr, su, d, plist, chunk)
    assert proof == unchecked
    assert _unpack(vf, proof, K2) == orc.np_prove_multi(real, CH, NONCES, POWS, K1, K2, NUM)
    assert (rep.damaged, rep.damaged_index, rep.proof_verified) == (0, [], True)
    if len(plist) == 1:   # one round: the winner's K2 hits
        assert (rep.labels_rechecked, rep.rounds) == (K2, 1)
    assert 0 < rep.labels_rechecked <= NONCES * K2 * len(plist)
    assert meta == vf.ProofMetadata(NODE, ATX, CH, UNITS, LPU)
    _verify(vf, proof, meta)


# --------------------------------------------------------------------------------------------------- damage
def test_forged_winner(mods, b2, orc, base, forged, tmp_path):
    """K2 forged hits of one nonce at the lowest indices: the unchecked proof is made of them and the verifier rejects
    it at position 0; the checked proof drops and reports all of them and equals the oracle's."""
    su, pr, vf = mods
    n = 5
    d, stored = _damage(base[0], tmp_path / "p", base[1], {i: forged[n][i] for i in range(K2)})
    unchecked, meta, _ = pr.generate_proof(d, CH, _cfg(su), nonces=NONCES, chunk_labels=4099, pow="skip")
    assert _unpack(vf, unchecked, K2) == (n, list(range(K2)))
    with pytest.raises(vf.ErrInvalidIndex) as e:
        _verify(vf, unchecked, meta)
    assert e.value.index == 0
    want = _oracle_checked(orc, stored, base[1], NONCES, POWS, K1, K2, NUM)
    before = (_counter(b2, "b200post_prove_labels_rechecked_total"), _counter(b2, "b200post_prove_damaged_labels_total"))
    proof, meta, _, rep = _checked(pr, su, d)
    after = (_counter(b2, "b200post_prove_labels_rechecked_total"), _counter(b2, "b200post_prove_damaged_labels_total"))
    assert after[0] - before[0] == rep.labels_rechecked and after[1] - before[1] == rep.damaged
    assert _unpack(vf, proof, K2) == want
    assert rep.damaged_index == list(range(K2)) and rep.damaged == K2 and rep.proof_verified
    _verify(vf, proof, meta)


def _clean_winner(orc, real, k2=K2):
    return orc.np_prove_multi(real, CH, NONCES, POWS, K1, k2, NUM)


def test_altered_hit_that_still_passes_is_dropped(mods, orc, base, forged, tmp_path):
    su, pr, vf = mods
    w, idx = _clean_winner(orc, base[1])
    d, stored = _damage(base[0], tmp_path / "p", base[1], {idx[3]: forged[w][0]})
    want = _oracle_checked(orc, stored, base[1], NONCES, POWS, K1, K2, NUM)
    assert want != (w, idx)
    for plist in ([0], [0, 0, 0]):
        proof, meta, _, rep = _checked(pr, su, d, plist)
        assert _unpack(vf, proof, K2) == want
        assert rep.damaged_index == [idx[3]] and rep.damaged == 1
        _verify(vf, proof, meta)


def test_damage_that_makes_a_hit_fail_is_invisible(mods, orc, base, forged, tmp_path):
    su, pr, vf = mods
    w, idx = _clean_winner(orc, base[1])
    d, stored = _damage(base[0], tmp_path / "p", base[1], {idx[3]: forged["none"]})
    want = orc.np_prove_multi(stored, CH, NONCES, POWS, K1, K2, NUM)
    assert want == _oracle_checked(orc, stored, base[1], NONCES, POWS, K1, K2, NUM) and want != (w, idx)
    proof, meta, _, rep = _checked(pr, su, d)
    assert _unpack(vf, proof, K2) == want and rep.damaged == 0 and rep.damaged_index == []
    _verify(vf, proof, meta)


def test_damage_past_the_decision_point_is_not_seen(mods, orc, base, forged, tmp_path):
    su, pr, vf = mods
    w, idx = _clean_winner(orc, base[1])
    rows = {NUM - 1 - j: forged[j % NONCES][j] for j in range(100)}
    d, _ = _damage(base[0], tmp_path / "p", base[1], rows)
    proof, _, scanned, rep = _checked(pr, su, d)
    assert _unpack(vf, proof, K2) == (w, idx)
    assert scanned < NUM - 100 and rep.damaged == 0 and rep.damaged_index == []


def test_more_than_64_damaged_hits(mods, orc, base, forged, tmp_path):
    """80 forged hits of one nonce at the lowest indices and K2 = 70: the first round alone meets 70 mismatches, more than
    one compare reports, so the compare is repeated; the report is the lowest 64, ascending."""
    su, pr, vf = mods
    n, k2 = 9, 70
    planted = set(range(80))
    d, stored = _damage(base[0], tmp_path / "p", base[1], {i: forged[n][i] for i in planted})
    want = _oracle_checked(orc, stored, base[1], NONCES, POWS, K1, k2, NUM)
    assert want[0] is not None
    proof, meta, _, rep = _checked(pr, su, d, k2=k2)
    assert _unpack(vf, proof, k2) == want
    assert rep.damaged_index == list(range(64)) and 64 <= rep.damaged <= 80 and rep.proof_verified
    _verify(vf, proof, meta, k2=k2)


def _shards(total: int, chunk: int, n: int):
    chunks = -(-total // chunk)
    q, r = divmod(chunks, n)
    out, first = [], 0
    for s in range(n):
        end = first + q + (1 if s < r else 0)
        out.append((min(total, first * chunk), min(total, end * chunk)))
        first = end
    return out


def test_damage_around_shard_boundaries(mods, orc, base, forged, tmp_path):
    """K2 = 70 puts the decision past the shard boundaries of [0, 0] and [0, 0, 0]; forged hits of several nonces sit on
    both sides of each boundary.  Every list and chunk size gives the oracle's proof; every report names planted rows."""
    su, pr, vf = mods
    k2 = 70
    w, _ = _clean_winner(orc, base[1], k2)
    bounds = {b for chunk in (4099, 1 << 16) for n in (2, 3) for _, b in _shards(NUM, chunk, n)[:-1]}
    rows, j = {}, 0
    for b in sorted(bounds):
        for off in (-3, -2, -1, 0, 1, 2):
            nonce = (w, 1, 2, 3)[j % 4]
            rows[b + off] = forged[nonce][j]
            j += 1
    d, stored = _damage(base[0], tmp_path / "p", base[1], rows)
    want = _oracle_checked(orc, stored, base[1], NONCES, POWS, K1, k2, NUM)
    assert want[0] is not None and want[1][-1] > min(bounds)
    for chunk in (4099, 1 << 16):
        for plist in LISTS:
            proof, meta, _, rep = _checked(pr, su, d, plist, chunk, k2=k2)
            assert _unpack(vf, proof, k2) == want, (plist, chunk)
            assert set(rep.damaged_index) <= set(rows) and rep.damaged >= len(rep.damaged_index), (plist, chunk)
            assert rep.proof_verified
    _verify(vf, proof, meta, k2=k2)


def test_saturated_shards_stop_with_damage_inside(mods, orc, base, forged, tmp_path):
    """Round difficulty (1 label in 32 per nonce), K2 = 4, [0, 0, 0].  Shard 0 holds a block that passes nothing (damage
    no scan can see), so nothing is decided before it is scanned to its end.  Shards 1 and 2 hold real labels with forged
    hits early on: each must drop those and still stop within two chunks of the point where every nonce has K2 usable
    hits in it."""
    su, pr, vf = mods
    k1, k2, nonces, chunk = NUM // 32, 4, 16, 4099
    pows = [0]
    shards = _shards(NUM, chunk, 3)
    blocks = np.random.default_rng(99).integers(0, 256, (200_000, 16), dtype=np.uint8)
    hits = orc.np_prove_hits(blocks, CH, nonces, pows, k1, len(blocks), NUM)
    passing = np.zeros(len(blocks), bool)
    for h in hits.values():
        passing[h] = True
    rows = {i: blocks[np.flatnonzero(~passing)[0]] for i in range(shards[0][1])}
    planted = set()
    for lo, _ in shards[1:]:
        for j in range(8):
            rows[lo + 3 * j] = blocks[hits[j][0]]
            planted.add(lo + 3 * j)
    d, stored = _damage(base[0], tmp_path / "p", base[1], rows)
    ok = (stored == base[1]).all(axis=1)
    bound = shards[0][1]
    for lo, hi in shards[1:]:
        sh = orc.np_prove_hits(stored[lo:hi], CH, nonces, pows, k1, hi - lo, NUM)
        usable = {n: [int(i) for i in h if ok[lo + i]][:k2] for n, h in sh.items()}
        assert all(len(u) == k2 for u in usable.values())
        sat = max(u[-1] for u in usable.values()) + 1
        assert sat + 2 * chunk < (hi - lo) // 2
        bound += sat + 2 * chunk
    want = _oracle_checked(orc, stored, base[1], nonces, pows, k1, k2, NUM)
    proof, meta, scanned, rep = _checked(pr, su, d, [0, 0, 0], chunk, k1=k1, k2=k2, nonces=nonces)
    assert _unpack(vf, proof, k2) == want
    assert shards[0][1] <= scanned <= bound, (scanned, bound)
    assert set(rep.damaged_index) <= planted and rep.damaged > 0
    _verify(vf, proof, meta, k1=k1, k2=k2)


# ------------------------------------------------------------------------------------ pow, cancel, errors, N = 8192
def test_builtin_pow_end_to_end(mods, b2, orc, base, tmp_path):
    su, pr, vf = mods
    pow_difficulty = bytes([0x30]) + bytes(range(101, 132))
    cfg = _cfg(su, pow_difficulty=pow_difficulty)
    before = b2.get_option("rx_vms_per_sm")
    b2.set_option("rx_vms_per_sm", 1)
    try:
        unchecked, _, _ = pr.generate_proof(base[0], CH, cfg, nonces=NONCES, chunk_labels=4099)
        proof, meta, _, rep = pr.generate_proof_checked(base[0], CH, cfg, nonces=NONCES, chunk_labels=4099, providers=[0, 0])
    finally:
        b2.set_option("rx_vms_per_sm", before)
    assert proof == unchecked and rep.proof_verified and rep.damaged == 0
    v = vf.PostVerifier()
    try:
        v.verify(proof, meta, vf.VerifyParams(k1=K1, k2=K2, scrypt_n=2, pow_difficulty=pow_difficulty))
    finally:
        v.close()


def test_cancel_and_truncated_last_file_as_unchecked(mods, b2, base, tmp_path):
    su, pr, _ = mods
    flag = ctypes.c_int(0)

    def hook(ctx, nonce_group, challenge8, difficulty, node_id, pow_out):
        pow_out[0] = 0
        if nonce_group == NONCES // 16 - 1:
            flag.value = 1
        return 0

    for call in (pr.generate_proof, pr.generate_proof_checked):
        for plist in ([0], [0, 0]):
            flag.value = 0
            with pytest.raises(b2.B200PostError) as e:
                call(base[0], CH, _cfg(su), nonces=NONCES, chunk_labels=4099, pow=hook, providers=plist, cancel=flag)
            assert e.value.code == b2.ERR_CANCELLED
    d = tmp_path / "short"
    shutil.copytree(base[0], d)
    last = d / f"postdata_{(NUM - 1) // PER_FILE}.bin"
    last.write_bytes(last.read_bytes()[:-16 * 1001])
    for call in (pr.generate_proof, pr.generate_proof_checked):
        for plist in ([0], [0, 0, 0]):
            with pytest.raises(b2.B200PostError) as e:   # K2 = 500: no nonce reaches it, so the scan reaches the end
                call(str(d), CH, _cfg(su, k2=500), nonces=NONCES, chunk_labels=4099, pow="skip", providers=plist)
            assert e.value.code == su.ERR_IO and "short read" in str(e.value), (call, plist)
    proof, _, _, rep = _checked(pr, su, base[0])
    assert rep.proof_verified


def test_mainnet_shape_at_n8192_with_a_forged_winner(mods, orc, tmp_path):
    """N = 8192, 2^14 labels, 288 nonces, K1 = 26, K2 = 37: the recheck runs the low-latency ROMix path."""
    su, pr, vf = mods
    lpu, units, per_file, k1, k2, nonces = 1 << 13, 2, 10_007, 26, 37, 288
    num = lpu * units
    pows = [0] * (nonces // 16)
    d = tmp_path / "clean"
    real = _write_setup(su, d, units, lpu, per_file, 8192)
    sample = np.array([0, 1, 5000, num - 1], dtype=np.uint64)
    comm = np.tile(np.frombuffer(orc.c_commitment(NODE, ATX), dtype=np.uint8), (len(sample), 1))
    assert (orc.c_labels_gather(comm, sample, 8192) == real[sample.astype(np.int64)]).all()
    blocks = np.random.default_rng(8).integers(0, 256, (200_000, 16), dtype=np.uint8)
    n = 17
    fh = orc.np_prove_hits(blocks, CH, nonces, pows, k1, len(blocks), num)[n]
    assert len(fh) >= k2
    dd, stored = _damage(str(d), tmp_path / "p", real, {i: blocks[fh[i]] for i in range(k2)}, per_file)
    want = _oracle_checked(orc, stored, real, nonces, pows, k1, k2, num)
    assert want[0] is not None and want[0] != n
    unchecked, _, _ = pr.generate_proof(dd, CH, _cfg(su, k1, k2, lpu), nonces=nonces, pow="skip")
    assert _unpack(vf, unchecked, k2, num) == (n, list(range(k2)))
    proof, meta, _, rep = pr.generate_proof_checked(dd, CH, _cfg(su, k1, k2, lpu), nonces=nonces, pow="skip")
    assert _unpack(vf, proof, k2, num) == want
    assert rep.damaged_index == list(range(k2)) and rep.proof_verified
    _verify(vf, proof, meta, k1=k1, k2=k2, n=8192)
