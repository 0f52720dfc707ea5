"""GPU tier: proving over checksummed POST data (b200post_generate_proof_sums).

A covered label (one a usable postdata_<N>.sum describes) is scanned from stored bytes whose digest matched, or, in a
bad block, from its recomputation, so its hits are the real label's; an uncovered label follows the checked rule (a hit
only when the stored bytes equal the real label).  The expected proof is `_oracle_sums`: the selection rule over those
usable hits, with real labels from the C oracle.  Where every label is covered it is also generate_proof_multi's proof
over the pristine POST, whatever the damage.

POSTs are written by a setup session with checksums at N = 2 (one case at N = 8192).  Damage is planted by rewriting rows
of postdata_N.bin; crafted sidecars (partial `covered`, a wrong digest with a valid or a broken FNV-1a) are written here
with the `blake3` package.  Every call checks that the data dir's bytes and mtimes are unchanged and that the metrics
counters moved by the report's numbers."""
import ctypes
import importlib
import re
import shutil
import struct
from pathlib import Path

import blake3
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NODE, ATX = bytes(range(60, 92)), bytes(range(160, 192))
B = 1 << 16
LPU, UNITS = B, 3
NUM = LPU * UNITS
K1, K2, NONCES = 100, 20, 32
CH = bytes(range(40, 72))
POWS = [0] * (NONCES // 16)
LISTS = ([0], [0, 0], [0, 0, 0])
CHUNKS = (4099, B, 0)                  # 0 = the default chunk (the whole POST here)
PER_FILE = 50_001                      # files of 50001 labels: one short range each
PER_FILE_B = 2 * B + 5000              # two whole ranges and a short one per file
HEADER = 112


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
    mgr.request_checksums()
    mgr.start_session()
    assert mgr.status().state == su.STATE_COMPLETE
    files = sorted(d.glob("postdata_*.bin"), key=lambda p: int(p.stem.split("_")[1]))
    assert len(list(d.glob("postdata_*.sum"))) == len(files)
    return np.concatenate([np.fromfile(f, dtype=np.uint8) for f in files]).reshape(-1, 16)


@pytest.fixture(scope="module")
def real(orc):
    return orc.c_labels_range(orc.c_commitment(NODE, ATX), 2, 0, NUM)[0]


@pytest.fixture(scope="module")
def base(mods, real, tmp_path_factory):
    """The clean N = 2 POST in files of 50001 labels, with sidecars."""
    d = tmp_path_factory.mktemp("clean")
    assert (_write_setup(mods[0], d, UNITS, LPU, PER_FILE, 2) == real).all()
    return str(d)


@pytest.fixture(scope="module")
def base_b(mods, real, tmp_path_factory):
    """The same POST in files of 2 x 2^16 + 5000 labels."""
    d = tmp_path_factory.mktemp("clean_b")
    assert (_write_setup(mods[0], d, UNITS, LPU, PER_FILE_B, 2) == real).all()
    return str(d)


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


def _damage(base_dir: str, d: Path, real: np.ndarray, rows: dict, per_file=PER_FILE):
    """A copy of the POST with rows {index: 16 bytes} rewritten; returns (data dir, stored labels)."""
    shutil.copytree(base_dir, d)
    stored = real.copy()
    for i, v in rows.items():
        stored[i] = np.frombuffer(bytes(v), dtype=np.uint8)
    for f in sorted({i // per_file for i in rows}):
        (d / f"postdata_{f}.bin").write_bytes(stored[f * per_file:(f + 1) * per_file].tobytes())
    return str(d), stored


def _fnv(b: bytes) -> int:
    h = 0xcbf29ce484222325
    for c in b:
        h = ((h ^ c) * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
    return h


def _write_sidecar(d, f, labels_of_file: np.ndarray, covered, per_file, n=2):
    """postdata_<f>.sum covering the file's first `covered` labels, digests by the blake3 package (format restated)."""
    data = labels_of_file[:covered].tobytes()
    body = b"B2PSUMS1" + struct.pack("<II", 1, B) + NODE + ATX + struct.pack("<QQQQ", n, per_file, f, covered)
    body += b"".join(blake3.blake3(data[o:o + 16 * B]).digest() for o in range(0, len(data), 16 * B))
    Path(d, f"postdata_{f}.sum").write_bytes(body + struct.pack("<Q", _fnv(body)))


def _wrong_digest(d, f, rng, fix_fnv=True):
    """Flip one byte of digest `rng` of postdata_<f>.sum, with the FNV-1a rewritten (still usable) or not (unusable)."""
    p = Path(d, f"postdata_{f}.sum")
    raw = bytearray(p.read_bytes())
    raw[HEADER + 32 * rng + 3] ^= 0x40
    if fix_fnv:
        raw[-8:] = struct.pack("<Q", _fnv(bytes(raw[:-8])))
    p.write_bytes(bytes(raw))


def _covered_mask(d, per_file=PER_FILE):
    """Per label: whether a sidecar in d claims it (as the tests craft them: usable unless its FNV is broken)."""
    m = np.zeros(NUM, bool)
    for p in Path(d).glob("postdata_*.sum"):
        raw = p.read_bytes()
        if struct.unpack_from("<Q", raw, len(raw) - 8)[0] != _fnv(raw[:-8]):
            continue
        f = int(p.stem.split("_")[1])
        covered = struct.unpack_from("<Q", raw, 104)[0]
        m[f * per_file:f * per_file + covered] = True
    return m


def _oracle_sums(orc, stored, real, covered, k1=K1, k2=K2, nonces=NONCES, pows=POWS):
    """The selection rule over usable hits: covered rows scanned as their real label, uncovered rows as stored and usable
    only when equal to the real one.  -> (nonce, indices) or (None, None)."""
    eff = np.where(covered[:, None], real, stored)
    ok = covered | (stored == real).all(axis=1)
    best = None
    for n, hits in orc.np_prove_hits(eff, CH, nonces, pows, k1, len(eff), NUM).items():
        usable = [int(i) for i in hits if ok[i]][:k2]
        if len(usable) == k2 and (best is None or usable[-1] < best[1][-1]):
            best = (n, usable)
    return best or (None, None)


def _unpack(vf, proof, k2, num=NUM):
    return proof.nonce, vf.unpack_indices(proof.indices, vf.bits_per_index(num), k2)


def _counter(b2, name) -> int:
    return int(re.search(rf"^{name} (\S+)$", b2.metrics_text(), re.M).group(1))


COUNTERS = ("b200post_prove_sum_blocks_checked_total", "b200post_prove_sum_blocks_bad_total", "b200post_prove_sum_blocks_healed_total")


def _snapshot(d):
    return {p.name: (p.read_bytes(), p.stat().st_mtime_ns) for p in sorted(Path(d).iterdir())}


def _sums(b2, pr, su, d, plist=(0,), chunk=4099, k1=K1, k2=K2, nonces=NONCES, lpu=LPU, **kw):
    """generate_proof_sums, checking that the data dir is untouched and that the counters move by the report."""
    before, counts = _snapshot(d), [_counter(b2, c) for c in COUNTERS]
    err = None
    try:
        res = pr.generate_proof_sums(d, CH, _cfg(su, k1, k2, lpu, **kw.pop("cfg", {})), providers=list(plist), nonces=nonces,
                                     chunk_labels=chunk, pow=kw.pop("pow", "skip"), **kw)
        rep = res[3]
    except b2.B200PostError as e:
        err, rep = e, e.sums
    assert _snapshot(d) == before
    moved = [_counter(b2, c) - v for c, v in zip(COUNTERS, counts)]
    assert moved == [rep.blocks_checked, rep.bad_blocks, rep.healed_blocks]
    if err is not None:
        raise err
    return res


def _checked(pr, su, d, plist=(0,), chunk=4099, k2=K2, **kw):
    return pr.generate_proof_checked(d, CH, _cfg(su, k2=k2), providers=list(plist), nonces=NONCES, chunk_labels=chunk, pow="skip", **kw)


def _multi(pr, su, d, plist=(0,), chunk=4099, k2=K2, **kw):
    return pr.generate_proof(d, CH, _cfg(su, k2=k2), providers=list(plist), nonces=NONCES, chunk_labels=chunk, pow="skip", **kw)[0]


def _pristine(orc, real, k2=K2):
    return orc.np_prove_multi(real, CH, NONCES, POWS, K1, k2, NUM)


# --------------------------------------------------------------------------------------------------- clean data
@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("plist", LISTS, ids=["x1", "x2", "x3"])
@pytest.mark.parametrize("layout", ["short", "whole"])
def test_clean_covered_data(mods, b2, orc, real, base, base_b, layout, plist, chunk):
    su, pr, vf = mods
    d = base if layout == "short" else base_b
    proof, meta, chk, rep = _sums(b2, pr, su, d, plist, chunk)
    assert proof == _multi(pr, su, d, plist, chunk) == _checked(pr, su, d, plist, chunk)[0]
    assert _unpack(vf, proof, K2) == _pristine(orc, real)
    assert (rep.bad_blocks, rep.healed_blocks, rep.labels_uncovered, rep.bad) == (0, 0, 0, [])
    assert chk.labels_rechecked == 0 and chk.damaged == 0 and chk.proof_verified
    assert rep.blocks_checked > 0 and rep.labels_verified > 0
    assert meta == vf.ProofMetadata(NODE, ATX, CH, UNITS, LPU)


def test_clean_whole_read_counts_every_range(mods, b2, base, base_b):
    """K2 = 500: no nonce reaches it, so every label is read once: every range hashed and verified."""
    su, pr, _ = mods
    for d, ranges in ((base, 4), (base_b, 4)):   # 3 x 50001 + 46605; 2^16 + 2^16 + 5000 and 60536
        with pytest.raises(b2.B200PostError) as e:
            _sums(b2, pr, su, d, k2=500)
        assert e.value.code == b2.ERR_INVALID_PROOF
        assert (e.value.sums.blocks_checked, e.value.sums.labels_verified, e.value.sums.labels_uncovered) == (ranges, NUM, 0)


# --------------------------------------------------------------------------------------------------- damage
def test_forged_winner_is_healed(mods, b2, orc, real, base, forged, tmp_path):
    """K2 forged hits of nonce 5 at the lowest indices (covered): the unchecked proof is made of them; the sums proof is
    the pristine one, and the report names exactly file 0's range, healed, with the data (not the sidecar) damaged."""
    su, pr, vf = mods
    d, stored = _damage(base, tmp_path / "p", real, {i: forged[5][i] for i in range(K2)})
    assert _unpack(vf, _multi(pr, su, d), K2) == (5, list(range(K2)))
    for plist in LISTS:
        for chunk in CHUNKS:
            proof, _, chk, rep = _sums(b2, pr, su, d, plist, chunk)
            assert _unpack(vf, proof, K2) == _pristine(orc, real), (plist, chunk)
            assert rep.bad == [(0, PER_FILE)] and rep.bad_blocks == rep.healed_blocks == 1 and rep.sidecar_only == 0
            assert chk.labels_rechecked == 0 and chk.proof_verified


def test_damage_that_makes_a_hit_fail_is_seen(mods, b2, orc, real, base, forged, tmp_path):
    """A real hit of the pristine winner rewritten so that it passes nothing: the checked proof loses it (invisible
    damage); the sums proof is the pristine one."""
    su, pr, vf = mods
    w, idx = _pristine(orc, real)
    d, _ = _damage(base, tmp_path / "p", real, {idx[3]: forged["none"]})
    checked = _checked(pr, su, d)[0]
    assert _unpack(vf, checked, K2) != (w, idx)
    proof, _, _, rep = _sums(b2, pr, su, d)
    assert _unpack(vf, proof, K2) == (w, idx)
    r0 = idx[3] // PER_FILE * PER_FILE
    assert rep.bad == [(r0, min(PER_FILE, NUM - r0))] and rep.healed_blocks == 1


def test_wrong_digest_in_a_usable_sidecar(mods, b2, orc, real, base, forged, tmp_path):
    """A digest rewritten with a valid FNV: the block is recomputed, found right, and counted sidecar_only.  The same flip
    with a broken FNV makes the file's sidecar unusable: its labels follow the checked rule, which a failing hit there
    makes differ from the pristine proof."""
    su, pr, vf = mods
    w, idx = _pristine(orc, real)
    f = idx[3] // PER_FILE
    d = tmp_path / "fixed"
    shutil.copytree(base, d)
    _wrong_digest(d, f, 0)
    proof, _, _, rep = _sums(b2, pr, su, str(d))
    assert _unpack(vf, proof, K2) == (w, idx)
    assert rep.bad == [(f * PER_FILE, min(PER_FILE, NUM - f * PER_FILE))] and rep.sidecar_only == 1 and rep.healed_blocks == 1
    d2, stored = _damage(base, tmp_path / "broken", real, {idx[3]: forged["none"]})
    _wrong_digest(d2, f, 0, fix_fnv=False)
    cov = _covered_mask(d2)
    assert not cov[idx[3]]
    want = _oracle_sums(orc, stored, real, cov)
    assert want != (w, idx)
    checked = _checked(pr, su, d2)[0]
    proof, _, chk, rep = _sums(b2, pr, su, d2)
    assert proof == checked and _unpack(vf, proof, K2) == want
    assert rep.bad_blocks == 0 and rep.labels_uncovered > 0


def test_mixed_coverage(mods, b2, orc, real, base, forged, tmp_path):
    """File 3 has no sidecar and holds forged hits; file 1's sidecar covers its first 20000 labels only, with forged hits
    on both sides of that end; files 0 and 2 hold damage that their sidecars catch."""
    su, pr, vf = mods
    n = 7
    rows = {3 * PER_FILE + j: forged[n][j] for j in range(10)}
    rows.update({PER_FILE + 19_990 + j: forged[n][10 + j] for j in range(20)})
    rows.update({j: forged[n][40 + j] for j in range(5)})
    rows.update({2 * PER_FILE + 3 * j: forged[n][50 + j] for j in range(8)})
    d, stored = _damage(base, tmp_path / "p", real, rows)
    Path(d, "postdata_3.sum").unlink()
    _write_sidecar(d, 1, real[PER_FILE:2 * PER_FILE], 20_000, PER_FILE)
    cov = _covered_mask(d)
    assert cov.sum() == 3 * PER_FILE - (PER_FILE - 20_000)
    for k2 in (K2, 70):
        want = _oracle_sums(orc, stored, real, cov, k2=k2)
        assert want[0] is not None
        for plist in LISTS:
            proof, _, chk, rep = _sums(b2, pr, su, d, plist, k2=k2)
            assert _unpack(vf, proof, k2) == want, (k2, plist)
            assert {r[0] for r in rep.bad} <= {0, PER_FILE, 2 * PER_FILE} and rep.healed_blocks == rep.bad_blocks and chk.proof_verified


def test_no_sidecars_is_the_checked_call(mods, b2, orc, real, base, forged, tmp_path):
    su, pr, vf = mods
    d, stored = _damage(base, tmp_path / "p", real, {i: forged[5][i] for i in range(K2)})
    for p in Path(d).glob("*.sum"):
        p.unlink()
    for plist in ([0], [0, 0, 0]):
        proof, meta, chk, rep = _sums(b2, pr, su, d, plist)
        cproof, _, _, crep = _checked(pr, su, d, plist)
        assert proof == cproof and (chk.damaged, chk.damaged_index) == (crep.damaged, crep.damaged_index)
        assert rep.blocks_checked == 0 and rep.labels_verified == 0 and rep.labels_uncovered > 0
    # and the same status when no window has a proof
    with pytest.raises(b2.B200PostError) as e:
        _sums(b2, pr, su, d, k2=500)
    with pytest.raises(b2.B200PostError) as c:
        _checked(pr, su, d, k2=500)
    assert e.value.code == c.value.code == b2.ERR_INVALID_PROOF


def test_damage_around_shard_boundaries(mods, b2, orc, real, base, base_b, forged, tmp_path):
    """K2 = 70 puts the decision past the shard boundaries; forged hits of several nonces sit on both sides of every file
    start and every 2^16 boundary (where the plan cuts chunks and shards).  Every list and chunk size gives the pristine
    proof."""
    su, pr, vf = mods
    k2 = 70
    w, idx = _pristine(orc, real, k2)
    for d0, per_file in ((base, PER_FILE), (base_b, PER_FILE_B)):
        cuts = sorted({f * per_file for f in range(1, -(-NUM // per_file))} |
                      {f * per_file + k * B for f in range(-(-NUM // per_file)) for k in range(1, 3)} - {0})
        cuts = [c for c in cuts if c < NUM]
        rows, j = {}, 0
        for b in cuts:
            for off in (-3, -2, -1, 0, 1, 2):
                rows[b + off] = forged[(w, 1, 2, 3)[j % 4]][j]
                j += 1
        d, _ = _damage(d0, tmp_path / f"p{per_file}", real, rows, per_file)
        for chunk in (4099, B):
            for plist in LISTS:
                proof, _, _, rep = _sums(b2, pr, su, d, plist, chunk, k2=k2)
                assert _unpack(vf, proof, k2) == (w, idx), (per_file, plist, chunk)
                assert rep.healed_blocks == rep.bad_blocks > 0


@pytest.mark.parametrize("per_pass", [1, 2])
def test_windows_with_damage(mods, b2, orc, real, base, forged, tmp_path, per_pass):
    """K2 above every window-0 nonce's hit count, and forged hits that give nonce 3 of window 0 K2 of them: the unchecked
    windowed proof comes from window 0; the sums proof is the pristine windowed one."""
    su, pr, vf = mods
    hits0 = orc.np_prove_hits(real, CH, NONCES, POWS, K1, NUM, NUM)
    k2 = max(len(h) for h in hits0.values()) + 1
    assert k2 <= 200
    free = [i for i in range(0, NUM, 997) if i not in set(hits0[3])][:k2]
    d, _ = _damage(base, tmp_path / "p", real, {i: forged[3][j] for j, i in enumerate(free)})
    kw = dict(max_windows="all", windows_per_pass=per_pass)
    pristine = _multi(pr, su, base, k2=k2, **kw)
    assert pristine.nonce >= NONCES
    assert _multi(pr, su, d, k2=k2, **kw).nonce == 3
    for plist in ([0], [0, 0, 0]):
        proof, _, _, rep = _sums(b2, pr, su, d, plist, k2=k2, **kw)
        assert proof == pristine, plist
        assert rep.bad_blocks == rep.healed_blocks == len({i // PER_FILE for i in free})


# ------------------------------------------------------------------------------------------- cap, cancel, N = 8192
def test_heal_cap(mods, b2, base, real, forged, tmp_path):
    su, pr, _ = mods
    d, _ = _damage(base, tmp_path / "p", real, {5: forged["none"], PER_FILE + 5: forged["none"]})
    with pytest.raises(b2.B200PostError) as e:
        _sums(b2, pr, su, d, chunk=0, max_heal_blocks=1)
    assert e.value.code == su.ERR_LABEL_MISMATCH and "more than 1 damaged blocks" in str(e.value)
    assert e.value.sums.bad == [(0, PER_FILE), (PER_FILE, PER_FILE)] and e.value.sums.bad_blocks == 2
    proof, _, _, rep = _sums(b2, pr, su, d, chunk=0, max_heal_blocks=2)
    assert rep.healed_blocks == 2


def test_cancel(mods, b2, base):
    su, pr, _ = mods
    flag = ctypes.c_int(0)

    def hook(ctx, nonce_group, challenge8, difficulty, node_id, pow_out):
        pow_out[0] = 0
        if nonce_group == NONCES // 16 - 1:
            flag.value = 1
        return 0

    for plist in ([0], [0, 0]):
        flag.value = 0
        with pytest.raises(b2.B200PostError) as e:
            _sums(b2, pr, su, base, plist, pow=hook, cancel=flag)
        assert e.value.code == b2.ERR_CANCELLED


def test_n8192_damaged_winner_with_builtin_pow(mods, b2, orc, tmp_path):
    """N = 8192, 2^14 labels, 288 nonces, K1 = 26, K2 = 37, the k2pow searched on the device: the pristine winner's first
    hits rewritten with random bytes (in covered blocks) are healed on the low-latency ROMix path, the proof is the
    pristine one and passes the verifier's pow check."""
    su, pr, vf = mods
    lpu, units, per_file, k1, k2, nonces = 1 << 13, 2, 10_007, 26, 37, 288
    num = lpu * units
    pow_difficulty = bytes([0x30]) + bytes(range(101, 132))
    cfg = _cfg(su, k1, k2, lpu, pow_difficulty=pow_difficulty)
    d = tmp_path / "clean"
    real = _write_setup(su, d, units, lpu, per_file, 8192)
    before = b2.get_option("rx_vms_per_sm")
    b2.set_option("rx_vms_per_sm", 1)
    try:
        pristine = pr.generate_proof(str(d), CH, cfg, nonces=nonces)[0]
        _, idx = _unpack(vf, pristine, k2, num)
        blocks = np.random.default_rng(8).integers(0, 256, (5, 16), dtype=np.uint8)
        dd, _ = _damage(str(d), tmp_path / "p", real, {i: blocks[j] for j, i in enumerate(idx[:5])}, per_file)
        proof, meta, chk, rep = pr.generate_proof_sums(dd, CH, cfg, nonces=nonces)
    finally:
        b2.set_option("rx_vms_per_sm", before)
    assert proof == pristine and chk.proof_verified
    bad = sorted({i // per_file for i in idx[:5]})
    assert rep.bad == [(f * per_file, min(per_file, num - f * per_file)) for f in bad] and rep.healed_blocks == len(bad)
    v = vf.PostVerifier()
    try:
        v.verify(proof, meta, vf.VerifyParams(k1=k1, k2=k2, scrypt_n=8192, pow_difficulty=pow_difficulty))
    finally:
        v.close()


# ------------------------------------------------------------------------------------------------- two devices
def test_two_devices(mods, b2, orc, real, base, forged, tmp_path):
    su, pr, vf = mods
    if len(b2.providers()) < 2:
        pytest.skip("needs two GPUs")
    proof, _, chk, rep = _sums(b2, pr, su, base, [0, 1])
    assert proof == _multi(pr, su, base, [0, 1]) and rep.bad_blocks == 0 and chk.labels_rechecked == 0
    d, _ = _damage(base, tmp_path / "p", real, {i: forged[5][i] for i in range(K2)})
    proof, _, _, rep = _sums(b2, pr, su, d, [0, 1])
    assert _unpack(vf, proof, K2) == _pristine(orc, real) and rep.bad == [(0, PER_FILE)]
