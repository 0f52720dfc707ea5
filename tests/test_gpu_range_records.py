"""GPU tier: range records and their merge (request_range_record, merge_range_records).

One POST is initialised in file ranges on "several machines", each range keeping a record; the merge of the records
must write exactly the VRF nonce and initial_post.json that one uninterrupted full session with the initial proof
writes, and what search_vrf_nonce plus generate_proof find over the merged files, without reading a stored label.
Stopped range sessions resume to the same record whatever became of it."""
import ctypes
import importlib
import json
import os
import shutil
import struct
import subprocess
import threading
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ATX = bytes(range(3, 35))
ZERO = bytes(32)
FILES = 4
# scrypt-N -> (labels per file, compute batch): 4 files each, two units
SHAPES = {2: (256, 128), 8192: (64, 64)}
K1, K2, NONCES = 200, 10, 16
EASY = b"\x0f" + b"\xff" * 31
# a record's header with the proof part and no cache key: 140 bytes, then 88; then the pows, then upto
REC_HEADER = 228


@pytest.fixture(scope="module")
def mods(b2, gpu_ready):
    return (importlib.import_module("go-spacemesh_b200.setup"), importlib.import_module("go-spacemesh_b200.prove"),
            importlib.import_module("go-spacemesh_b200.verify"), importlib.import_module("go-spacemesh_b200.k2pow"))


def _num(n):
    return SHAPES[n][0] * FILES


def _cfg(su, n, k1=K1, k2=K2, pow_difficulty=None, lpu=None):
    return su.PostConfig(labels_per_unit=lpu or _num(n) // 2, k1=k1, k2=k2, k3=k2, pow_difficulty=pow_difficulty)


def _opts(su, d, n, provider=0, per_file=None, batch=None):
    pf, b = SHAPES.get(n, (None, None))
    return su.PostSetupOpts(data_dir=str(d), num_units=2, max_file_size=16 * (per_file or pf), provider_id=provider, scrypt_n=n,
                            compute_batch_size=batch or b)


def _callback(base, calls=None):
    def pow_(ctx, group, ch, diff, node, out):
        if calls is not None:
            calls.append(group)
        out[0] = base + group
        return 0
    return pow_


def _session(su, d, n, node, *, files=None, record=None, initial=None, provider=0, cfg=None, opts=None, cancel_at=None):
    """prepare (whole POST, or files) + record / initial-proof request + start.  record: None (no record) or the kwargs of
    request_range_record; cancel_at: stop once that many labels are written (the call must then be cancelled)."""
    mgr = su.PostSetupManager(cfg or _cfg(su, n))
    o = opts or _opts(su, d, n, provider)
    if files is None:
        mgr.prepare_initializer(o, node, ATX)
    else:
        mgr.prepare_files(o, node, ATX, *files)
    if record is not None:
        mgr.request_range_record(**record)
    if initial is not None:
        mgr.request_initial_proof(**initial)
    cancel = ctypes.c_int(0)
    if cancel_at is None:
        mgr.start_session()
        assert mgr.status().state == su.STATE_COMPLETE
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


def _nonce_fields(su, d):
    md = su.load_metadata(str(d))
    return md["nonce"], md["nonce_value"], md["last_position"]


def _data(d):
    return {p.name: p.read_bytes() for p in sorted(Path(d).glob("postdata_*.bin"))}


def _gather(dst, parts, meta_from, order=None):
    """A merge directory: every part's postdata files and records (in `order` of parts), one part's metadata."""
    dst.mkdir()
    for part in order or parts:
        for p in list(part.glob("postdata_*.bin")) + list(part.glob("range_*.rec")):
            shutil.copy2(p, dst / p.name)
    shutil.copy(meta_from / "postdata_metadata.json", dst / "postdata_metadata.json")
    return dst


def _triple(proof):
    return proof.nonce, proof.indices, proof.pow


@pytest.fixture(scope="module")
def identities(orc):
    """Per N, an identity whose arg-min lies inside the POST but not in the first range (files 0-1), and one whose nonce
    comes from the past-the-end search, picked by seed with the oracle: {(n, "in" | "past"): node_id}."""
    out = {}
    for n in SHAPES:
        total, split = _num(n), 2 * SHAPES[n][0]
        diff = orc.c_vrf_difficulty(total)
        for seed in range(400):
            node = bytes([seed, n & 0xff, n >> 8, 0x5a]) + bytes(28)
            _, found, idx, _ = orc.c_labels_range(orc.c_commitment(node, ATX), n, 0, total, diff)
            kind = "in" if found else "past"
            if kind == "in" and not split <= idx < total - 1:
                continue
            out.setdefault((n, kind), node)
            if (n, "in") in out and (n, "past") in out:
                break
    assert len(out) == 2 * len(SHAPES)
    return out


@pytest.fixture(scope="module")
def posts(mods, identities, tmp_path_factory):
    """Per (N, kind): A = the whole POST with the initial proof; B = files 0-1 and C = files 2-3 (on PROVIDER_ALL), both
    with records and the proof scan."""
    su = mods[0]
    root = tmp_path_factory.mktemp("ranges")
    req = dict(nonces=NONCES, pow="skip")
    out = {}
    for (n, kind), node in identities.items():
        base = root / f"{n}-{kind}"
        _session(su, base / "A", n, node, initial=req)
        _session(su, base / "B", n, node, files=(0, 1), record=dict(initial_proof=True, **req))
        _session(su, base / "C", n, node, files=(2, -1), record=dict(initial_proof=True, **req), provider=su.PROVIDER_ALL)
        out[(n, kind)] = base
    return out


CASES = [(2, "in"), (2, "past"), (8192, "in"), (8192, "past")]


@pytest.mark.parametrize("meta_from", ["B", "C"])
@pytest.mark.parametrize("n,kind", CASES)
def test_merge_equals_one_session(mods, identities, posts, tmp_path, n, kind, meta_from):
    su, pr, _, _ = mods
    base, batch = posts[(n, kind)], SHAPES[n][1]
    a = _nonce_fields(su, base / "A")
    assert (a[0] >= _num(n)) == (kind == "past")
    for part, names in (("B", ["postdata_0.bin", "postdata_1.bin", "postdata_metadata.json", "range_0_1.rec"]),
                        ("C", ["postdata_2.bin", "postdata_3.bin", "postdata_metadata.json", "range_2_3.rec"])):
        assert sorted(p.name for p in (base / part).iterdir()) == names        # the record, and no nonce in the metadata
        md = su.load_metadata(str(base / part))
        assert md["vrf_scan_pending"] == 1 and md["nonce"] is None
    d = _gather(tmp_path / "D", [base / "B", base / "C"], base / meta_from)
    zeros = _gather(tmp_path / "Z", [base / "B", base / "C"], base / meta_from)
    for p in zeros.glob("postdata_*.bin"):
        p.write_bytes(bytes(p.stat().st_size))
    (d / "initial_post.json").write_text("{}")                                   # a stale one is replaced
    assert _data(d) == _data(base / "A")
    mtimes = {p.name: p.stat().st_mtime_ns for p in d.glob("postdata_*.bin")}

    r = su.merge_range_records(str(d), _cfg(su, n), compute_batch_size=batch)
    assert (r.ranges, r.proof_rc, r.past_end) == (2, 0, kind == "past"), r.proof_reason
    assert (r.nonce, r.nonce_value) == a[:2]
    assert _nonce_fields(su, d) == a
    assert "VrfScanPending" not in json.loads((d / "postdata_metadata.json").read_text())
    assert (d / "initial_post.json").read_bytes() == (base / "A" / "initial_post.json").read_bytes()
    assert {p.name: p.stat().st_mtime_ns for p in d.glob("postdata_*.bin")} == mtimes
    loaded = su.load_initial_proof(str(d), _cfg(su, n), NONCES)[0]
    assert _triple(loaded) == _triple(r.proof)

    # the same as searching the stored labels and proving over them
    e = tmp_path / "E"
    shutil.copytree(d, e)
    shutil.copy(base / meta_from / "postdata_metadata.json", e / "postdata_metadata.json")
    su.search_vrf_nonce(str(e), compute_batch_size=batch)
    assert _nonce_fields(su, e) == a
    assert _triple(pr.generate_proof(str(e), ZERO, _cfg(su, n), nonces=NONCES, pow="skip")[0]) == _triple(loaded)

    # no stored label is read: zeros of the same size give the same result
    rz = su.merge_range_records(str(zeros), _cfg(su, n), compute_batch_size=batch)
    assert rz.proof_rc == 0 and (rz.nonce, rz.nonce_value) == a[:2]
    assert (zeros / "postdata_metadata.json").read_bytes() == (d / "postdata_metadata.json").read_bytes()
    assert (zeros / "initial_post.json").read_bytes() == (d / "initial_post.json").read_bytes()


def test_three_ranges_in_any_order(mods, identities, posts, tmp_path):
    su = mods[0]
    n = 2
    node, base = identities[(n, "in")], posts[(n, "in")]
    req = dict(initial_proof=True, nonces=NONCES, pow="skip")
    parts = []
    for name, files in (("r3", (3, 3)), ("r12", (1, 2)), ("r0", (0, 0))):
        _session(su, tmp_path / name, n, node, files=files, record=req)
        parts.append(tmp_path / name)
    d = _gather(tmp_path / "D", parts, tmp_path / "r3")
    r = su.merge_range_records(str(d), _cfg(su, n), compute_batch_size=SHAPES[n][1])
    assert r.ranges == 3 and r.proof_rc == 0, r.proof_reason
    assert _nonce_fields(su, d) == _nonce_fields(su, base / "A")
    assert (d / "initial_post.json").read_bytes() == (base / "A" / "initial_post.json").read_bytes()


def _pick(orc, want, n=2, per_file=256, seeds=300):
    """The first identity (by seed) whose oracle labels satisfy want(labels)."""
    total = per_file * FILES
    for seed in range(seeds):
        node = bytes([seed, 0xa7]) + bytes(30)
        labels = orc.c_labels_range(orc.c_commitment(node, ATX), n, 0, total)
        labels = labels[0] if isinstance(labels, tuple) else labels
        if want(np.asarray(labels, dtype=np.uint8).reshape(total, 16)):
            return node
    pytest.fail("no identity found")


def _full_and_merged(su, tmp_path, n, node, cfg, req, ranges=((0, 1), (2, 3))):
    a = tmp_path / "A"
    _session(su, a, n, node, cfg=cfg, initial=req)
    parts = []
    for lo, hi in ranges:
        p = tmp_path / f"r{lo}"
        _session(su, p, n, node, files=(lo, hi), cfg=cfg, record=dict(initial_proof=True, **req))
        parts.append(p)
    d = _gather(tmp_path / "D", parts, parts[0])
    return a, d, su.merge_range_records(str(d), cfg, compute_batch_size=SHAPES[n][1])


def test_k1_below_k2_winner_spans_the_ranges(mods, orc, tmp_path):
    """K1 < K2: the winner's first hits lie in the first range and its K2-th in the second."""
    su, _, vf, _ = mods
    n, k1, k2, nonces, total, split = 2, 10, 12, 64, _num(2), 2 * SHAPES[2][0]

    def spans(labels):
        nonce, idx = orc.np_prove_multi(labels, ZERO, nonces, [0] * (nonces // 16), k1, k2, total)
        return nonce is not None and idx[0] < split <= idx[-1]
    node = _pick(orc, spans)
    cfg = _cfg(su, n, k1=k1, k2=k2)
    a, d, r = _full_and_merged(su, tmp_path, n, node, cfg, dict(nonces=nonces, pow="skip"))
    assert r.proof_rc == 0, r.proof_reason
    idx = vf.unpack_indices(r.proof.indices, vf.bits_per_index(total), k2)
    assert idx[0] < split <= idx[-1]
    assert (d / "initial_post.json").read_bytes() == (a / "initial_post.json").read_bytes()
    assert _nonce_fields(su, d) == _nonce_fields(su, a)


def test_three_windows_first_without_a_proof(mods, orc, tmp_path):
    su = mods[0]
    n, k1, k2, nonces, w, total = 2, 10, 16, 16, 3, _num(2)

    def later_window(labels):
        hits = orc.np_prove_hits(labels, ZERO, nonces * w, [0] * (nonces * w // 16), k1, k2, total)
        full = [nn for nn, h in hits.items() if len(h) == k2]
        return full and min(full) >= nonces
    node = _pick(orc, later_window)
    cfg = _cfg(su, n, k1=k1, k2=k2)
    a, d, r = _full_and_merged(su, tmp_path, n, node, cfg, dict(nonces=nonces, pow="skip", windows_per_pass=w))
    assert r.proof_rc == 0 and r.proof.nonce >= nonces, r.proof_reason
    assert json.loads((d / "initial_post.json").read_text())["Windows"] == w
    assert (d / "initial_post.json").read_bytes() == (a / "initial_post.json").read_bytes()


# resume: N = 8192, 2 x 8192 labels in files of 4096, batches of 512; the range is files 0-1 (16 batches)
R_N, R_LPU, R_PER_FILE, R_BATCH, R_NONCES = 8192, 8192, 4096, 512, 32


def _upto(rec: bytes, groups: int) -> int:
    return struct.unpack_from("<Q", rec, REC_HEADER + 8 * groups)[0]


def test_resume_gives_the_same_record(mods, tmp_path):
    """(a) the record as left, (b) deleted, (c) one byte flipped, (d) an older record below the labels on disk: every
    resumed session ends with the record of an uninterrupted one."""
    su = mods[0]
    node = bytes(range(50, 82))
    cfg = _cfg(su, R_N, k1=10, k2=12, lpu=R_LPU)

    def run(d, calls=None, cancel_at=None):
        o = _opts(su, d, R_N, per_file=R_PER_FILE, batch=R_BATCH)
        return _session(su, d, R_N, node, files=(0, 1), cfg=cfg, opts=o, cancel_at=cancel_at,
                        record=dict(initial_proof=True, nonces=R_NONCES, pow=_callback(1000, calls)))
    run(tmp_path / "ref")
    ref = (tmp_path / "ref" / "range_0_1.rec").read_bytes()
    assert _upto(ref, R_NONCES // 16) == 2 * R_PER_FILE
    half = tmp_path / "half"
    calls = []
    run(half, calls, cancel_at=1024)
    older = (half / "range_0_1.rec").read_bytes()
    mgr = run(half, calls, cancel_at=R_PER_FILE + 1024)
    assert mgr.status().state == su.STATE_STOPPED
    assert calls == list(range(R_NONCES // 16))                  # the resumed session used the record's pows
    state = (half / "range_0_1.rec").read_bytes()
    on_disk = sum(p.stat().st_size for p in half.glob("postdata_*.bin")) // 16
    assert 1024 <= _upto(older, R_NONCES // 16) < _upto(state, R_NONCES // 16) <= on_disk < 2 * R_PER_FILE
    for variant in "abcd":
        d = tmp_path / variant
        shutil.copytree(half, d)
        rec = d / "range_0_1.rec"
        if variant == "b":
            rec.unlink()
        elif variant == "c":
            raw = bytearray(rec.read_bytes())
            raw[len(raw) // 2] ^= 0x10
            rec.write_bytes(bytes(raw))
        elif variant == "d":
            rec.write_bytes(older)
        vcalls = []
        run(d, vcalls)
        assert rec.read_bytes() == ref, variant
        assert vcalls == ([] if variant in "ad" else list(range(R_NONCES // 16))), variant
        assert _data(d) == _data(tmp_path / "ref"), variant


def test_partial_records(mods, identities, posts, tmp_path):
    su = mods[0]
    n, batch = 2, SHAPES[2][1]
    node, base = identities[(n, "in")], posts[(n, "in")]
    a = _nonce_fields(su, base / "A")
    # a range session without a request writes no record
    _session(su, tmp_path / "plain", n, node, files=(0, 1))
    assert not list((tmp_path / "plain").glob("range_*"))
    # VRF-only records: the nonce, no proof, and a stale proof file removed
    for part, files in (("vb", (0, 1)), ("vc", (2, 3))):
        _session(su, tmp_path / part, n, node, files=files, record=dict())
    d = _gather(tmp_path / "V", [tmp_path / "vb", tmp_path / "vc"], tmp_path / "vb")
    shutil.copy(base / "A" / "initial_post.json", d / "initial_post.json")
    r = su.merge_range_records(str(d), _cfg(su, n), compute_batch_size=batch)
    assert r.proof_rc == su.ERR_STATE and "VRF only" in r.proof_reason and r.proof is None
    assert _nonce_fields(su, d) == a and not (d / "initial_post.json").exists()
    # records made with other pows: the nonce, no proof
    for part, files, pow_base in (("pb", (0, 1), 1000), ("pc", (2, 3), 2000)):
        _session(su, tmp_path / part, n, node, files=files, record=dict(initial_proof=True, nonces=NONCES, pow=_callback(pow_base)))
    d = _gather(tmp_path / "P", [tmp_path / "pb", tmp_path / "pc"], tmp_path / "pc")
    r = su.merge_range_records(str(d), _cfg(su, n), compute_batch_size=batch)
    assert r.proof_rc == su.ERR_STATE and "pows" in r.proof_reason
    assert _nonce_fields(su, d) == a
    # a missing range: nothing changes
    d = _gather(tmp_path / "M", [base / "B", base / "C"], base / "B")
    (d / "range_2_3.rec").unlink()
    before = (d / "postdata_metadata.json").read_bytes()
    with pytest.raises(Exception) as e:
        su.merge_range_records(str(d), _cfg(su, n), compute_batch_size=batch)
    assert e.value.code == su.ERR_STATE and "[512, 1024)" in str(e.value)
    assert (d / "postdata_metadata.json").read_bytes() == before and not (d / "initial_post.json").exists()


def test_builtin_pows(mods, identities, tmp_path):
    """At an easy difficulty: both ranges find the same pows (those of k2pow's group search), and the merge's gate checks
    the pow of the proof it writes."""
    su, pr, _, k2 = mods
    n = 2
    node = identities[(n, "in")]
    cfg = _cfg(su, n, pow_difficulty=EASY)
    req = dict(initial_proof=True, nonces=NONCES, pow="builtin")
    for part, files in (("B", (0, 1)), ("C", (2, 3))):
        _session(su, tmp_path / part, n, node, files=files, cfg=cfg, record=req)
    pows, _ = k2.search_groups(ZERO[:8], node, k2.scale_difficulty(EASY, 2), NONCES // 16)
    for part, name in (("B", "range_0_1.rec"), ("C", "range_2_3.rec")):
        rec = (tmp_path / part / name).read_bytes()
        assert list(struct.unpack_from(f"<{NONCES // 16}Q", rec, REC_HEADER)) == list(pows), part
    d = _gather(tmp_path / "D", [tmp_path / "B", tmp_path / "C"], tmp_path / "B")
    r = su.merge_range_records(str(d), cfg, compute_batch_size=SHAPES[n][1])
    assert r.proof_rc == 0, r.proof_reason
    assert r.proof.pow == pows[r.proof.nonce // 16]
    assert _triple(r.proof) == _triple(pr.generate_proof(str(d), ZERO, cfg, nonces=NONCES, pow="builtin")[0])


def test_cli_round_trip(b2, mods, identities, tmp_path):
    su = mods[0]
    cli = Path(b2.LIB_PATH).parent / "b200postcli"
    if not cli.exists():
        pytest.skip("b200postcli not built")
    n = 8192
    per_file, batch = SHAPES[n]
    node = identities[(n, "in")]
    proof = ["-k1", str(K1), "-k2", str(K2), "-powDifficulty", EASY.hex()]
    common = ["-id", node.hex(), "-commitmentAtxId", ATX.hex(), "-numUnits", "2", "-labelsPerUnit", str(per_file * FILES // 2),
              "-maxFileSize", str(16 * per_file), "-scryptN", str(n), "-computeBatchSize", str(batch)]
    init = proof + ["-initialProof", "-nonces", str(NONCES)]
    r = subprocess.run([str(cli)] + common + init + ["-datadir", str(tmp_path / "A")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "initial proof: nonce" in r.stdout, r.stdout + r.stderr
    for part, lo, hi in (("B", "0", "1"), ("C", "2", "3")):
        r = subprocess.run([str(cli)] + common + init + ["-datadir", str(tmp_path / part), "-fromFile", lo, "-toFile", hi, "-rangeRecord"],
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0 and "-mergeRanges" in r.stdout, r.stdout + r.stderr
    d = _gather(tmp_path / "D", [tmp_path / "B", tmp_path / "C"], tmp_path / "C")
    r = subprocess.run([str(cli), "-mergeRanges", "-datadir", str(d), "-computeBatchSize", str(batch)] + proof,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "initial proof: nonce" in r.stdout, r.stdout + r.stderr
    assert (d / "initial_post.json").read_bytes() == (tmp_path / "A" / "initial_post.json").read_bytes()
    assert _nonce_fields(su, d) == _nonce_fields(su, tmp_path / "A")
    os.remove(d / "range_0_1.rec")
    r = subprocess.run([str(cli), "-mergeRanges", "-datadir", str(d)] + proof, capture_output=True, text=True, timeout=600)
    assert r.returncode == 1 and "[0, 128)" in r.stderr, r.stdout + r.stderr
