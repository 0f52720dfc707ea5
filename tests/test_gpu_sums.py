"""GPU tier: block checksums (postdata_<N>.sum).  The BLAKE3 kernel against the `blake3` package; the sidecars of setup
sessions (batch seams, short blocks and files, PROVIDER_ALL, initial proof, range records, resume, growth, damaged
sidecars) against blake3 of the files they describe; check_sums on planted damage; repair; write_sums."""
import ctypes
import importlib
import shutil
import struct
import subprocess
import threading
from pathlib import Path

import blake3
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
NODE, ATX = bytes(range(9, 41)), bytes(range(60, 92))
B = 1 << 16   # labels per block
HEADER = 112  # magic, version, block labels, NodeId, CommitmentAtxId, N, labels per file, file, covered


@pytest.fixture(scope="module")
def su(b2, gpu_ready):
    return importlib.import_module("go-spacemesh_b200.setup")


def _digests(data: bytes) -> list[bytes]:
    """blake3 of each 1 MiB block of one file's bytes, the last one short."""
    return [blake3.blake3(data[o:o + 16 * B]).digest() for o in range(0, len(data), 16 * B)]


def _read_sums(p: Path) -> tuple[int, list[bytes]]:
    raw = p.read_bytes()
    assert raw[:8] == b"B2PSUMS1" and struct.unpack_from("<II", raw, 8) == (1, B)
    covered = struct.unpack_from("<Q", raw, 104)[0]
    n = (covered + B - 1) // B
    assert len(raw) == HEADER + 32 * n + 8
    return covered, [raw[HEADER + 32 * i:HEADER + 32 * i + 32] for i in range(n)]


def _assert_sums_describe_files(d: Path, per_file: int, files=None):
    bins = sorted(d.glob("postdata_*.bin"), key=lambda p: int(p.stem.split("_")[1]))
    for p in bins:
        f = int(p.stem.split("_")[1])
        if files is not None and f not in files:
            continue
        data = p.read_bytes()
        covered, got = _read_sums(d / f"postdata_{f}.sum")
        assert covered == len(data) // 16, f
        assert got == _digests(data), f


def _others(d: Path) -> dict:
    return {p.name: p.read_bytes() for p in sorted(d.iterdir()) if not p.name.endswith(".sum")}


def _session(su, d, *, lpu, units, per_file, n=2, batch=1 << 12, provider_id=0, sums=True, proof=None, files=None,
             record=None, cancel_at=None):
    """prepare (+ requests) + start; cancel_at: stop once that many labels are written (the call must be cancelled)."""
    mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=lpu, max_num_units=16, k1=200, k2=10, k3=10))
    o = su.PostSetupOpts(data_dir=str(d), num_units=units, max_file_size=16 * per_file, provider_id=provider_id, scrypt_n=n,
                         compute_batch_size=batch)
    if files is None:
        mgr.prepare_initializer(o, NODE, ATX)
    else:
        mgr.prepare_files(o, NODE, ATX, *files)
    if record is not None:
        mgr.request_range_record(**record)
    if proof is not None:
        mgr.request_initial_proof(**proof)
    if sums:
        mgr.request_checksums()
    if cancel_at is None:
        mgr.start_session()
        assert mgr.status().state == su.STATE_COMPLETE
        return mgr
    cancel, done = ctypes.c_int(0), threading.Event()

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


# ---------------------------------------------------------------------------------------------------------- kernel
def test_kernel_matches_blake3(su):
    rng = np.random.default_rng(7)
    for count in (1, 63, 64, 65, 127, 1024, 4095, B - 1, B, B + 1, 5 * B + 17, 70 * B + 3):
        labels = rng.integers(0, 256, count * 16, dtype=np.uint8)
        got = su.label_block_digests(labels)
        want = _digests(labels.tobytes())
        assert [bytes(r) for r in got] == want, count


# ------------------------------------------------------------------------------------------------------------ init
# 3 x 50000 labels in files of 70000 (not a multiple of a block): files of 70000, 70000 and 10000 labels
LAYOUT = dict(lpu=50000, units=3, per_file=70000)


@pytest.mark.parametrize("batch", [8, 24, B + 8])
def test_init_sidecars_match_blake3_and_change_nothing_else(su, tmp_path, batch):
    plain, summed = tmp_path / "plain", tmp_path / "summed"
    _session(su, plain, batch=batch, sums=False, **LAYOUT)
    _session(su, summed, batch=batch, **LAYOUT)
    assert not list(plain.glob("*.sum"))
    assert sorted(p.name for p in summed.glob("*.sum")) == ["postdata_0.sum", "postdata_1.sum", "postdata_2.sum"]
    _assert_sums_describe_files(summed, LAYOUT["per_file"])
    assert _others(plain) == _others(summed)


def test_init_on_every_device(su, tmp_path):
    plain, summed = tmp_path / "plain", tmp_path / "summed"
    _session(su, plain, provider_id=su.PROVIDER_ALL, sums=False, batch=3000, **LAYOUT)
    _session(su, summed, provider_id=su.PROVIDER_ALL, batch=3000, **LAYOUT)
    _assert_sums_describe_files(summed, LAYOUT["per_file"])
    assert _others(plain) == _others(summed)


def test_init_with_initial_proof_and_range_records(su, tmp_path):
    proof = dict(nonces=16, pow="skip")
    plain, summed = tmp_path / "plain", tmp_path / "summed"
    _session(su, plain, sums=False, proof=proof, batch=5000, **LAYOUT)
    _session(su, summed, proof=proof, batch=5000, **LAYOUT)
    _assert_sums_describe_files(summed, LAYOUT["per_file"])
    assert _others(plain) == _others(summed)
    rec = dict(initial_proof=True, nonces=16, pow="skip")
    rplain, rsummed = tmp_path / "rplain", tmp_path / "rsummed"
    _session(su, rplain, sums=False, files=(1, 2), record=rec, batch=5000, **LAYOUT)
    _session(su, rsummed, files=(1, 2), record=rec, batch=5000, **LAYOUT)
    assert sorted(p.name for p in rsummed.glob("*.sum")) == ["postdata_1.sum", "postdata_2.sum"]
    assert list(rsummed.glob("range_*.rec"))
    _assert_sums_describe_files(rsummed, LAYOUT["per_file"])
    assert _others(rplain) == _others(rsummed)


def test_resume_recomputes_the_open_block_and_does_not_read_it_back(su, tmp_path):
    d = tmp_path / "r"
    lay = dict(lpu=100000, units=8, per_file=800000)
    _session(su, d, batch=1000, cancel_at=150000, **lay)
    written = (d / "postdata_0.bin").stat().st_size // 16
    assert 0 < written < 800000 and written % B
    start = written // B * B
    # damage a stored label of the block the resume recomputes: the sidecar must still describe the right label
    data = bytearray((d / "postdata_0.bin").read_bytes())
    data[(start + 3) * 16 + 5] ^= 0x10
    (d / "postdata_0.bin").write_bytes(bytes(data))
    _session(su, d, batch=1000, **lay)
    r = su.check_sums(str(d))
    assert r.code == su.ERR_LABEL_MISMATCH and r.bad_blocks == 1 and r.bad == [(start, B)]


def test_growth_extends_the_last_sidecar_and_a_damaged_sidecar_is_rebuilt(su, tmp_path):
    d = tmp_path / "g"
    lay = dict(lpu=50000, per_file=200000)
    _session(su, d, units=2, **lay)                     # one file of 100000 labels: a short last block
    assert _read_sums(d / "postdata_0.sum")[0] == 100000
    _session(su, d, units=3, **lay)                     # grown to 150000
    _assert_sums_describe_files(d, 200000)
    good = (d / "postdata_0.sum").read_bytes()
    bad = bytearray(good)
    bad[HEADER + 40] ^= 1
    (d / "postdata_0.sum").write_bytes(bytes(bad))
    with pytest.raises(Exception) as e:                 # a damaged sidecar is unusable: nothing is covered
        su.check_sums(str(d))
    assert e.value.code == su.ERR_STATE and "no checksums" in str(e.value)
    _session(su, d, units=3, **lay)                     # every label is on disk: the session only rebuilds the sidecar
    assert (d / "postdata_0.sum").read_bytes() == good
    # an intact sidecar made for another file is replaced too
    body = good[:96] + struct.pack("<Q", 7) + good[104:-8]
    (d / "postdata_0.sum").write_bytes(body + struct.pack("<Q", _fnv(body)))
    _session(su, d, units=3, **lay)
    assert (d / "postdata_0.sum").read_bytes() == good


# ------------------------------------------------------------------------------------------------------- check
@pytest.fixture(scope="module")
def clean(su, tmp_path_factory):
    """3 x 100000 labels in files of 140000: files of 140000, 140000 and 20000 labels, with sidecars."""
    d = tmp_path_factory.mktemp("clean") / "p"
    _session(su, d, lpu=100000, units=3, per_file=140000, batch=1 << 15)
    return d


def _copy(src: Path, dst: Path) -> Path:
    shutil.copytree(src, dst)
    return dst


def _flip(d: Path, label: int, per_file=140000, bit=0x01):
    p = d / f"postdata_{label // per_file}.bin"
    data = bytearray(p.read_bytes())
    data[(label % per_file) * 16 + 7] ^= bit
    p.write_bytes(bytes(data))


def test_check_clean(su, clean):
    r = su.check_sums(str(clean))
    assert r.code == su.OK and r.labels_checked == 300000 and r.labels_unchecked == 0 and r.bad == []
    assert r.files_checked == 3 and r.files_unchecked == 0 and r.bytes_read == 300000 * 16 and r.blocks_checked == 3 + 3 + 1


def test_check_reports_exactly_the_damaged_blocks(su, clean, tmp_path):
    d = _copy(clean, tmp_path / "p")
    planted = [B, 2 * B - 1, 140000 + 3, 299999]   # first and last label of block 1, file 1's first block, the POST's last label
    for i in planted:
        _flip(d, i)
    r = su.check_sums(str(d))
    assert r.code == su.ERR_LABEL_MISMATCH and r.bad_blocks == 3
    assert r.bad == [(B, B), (140000, B), (280000, 20000)]
    r = su.check_sums(str(d), from_file=1, to_file=1)
    assert r.code == su.ERR_LABEL_MISMATCH and r.bad == [(140000, B)] and r.labels_checked == 140000
    r = su.check_sums(str(d), from_file=2)
    assert r.bad == [(280000, 20000)] and r.files_checked == 1
    cli = subprocess.run([str(ROOT / "go-spacemesh_b200" / "b200postcli"), "-checkSums", "-datadir", str(d)], capture_output=True, text=True)
    assert cli.returncode == 1, cli.stderr
    assert "file 0 labels [65536, 131072)" in cli.stdout and "file 2 labels [280000, 300000)" in cli.stdout


def test_partly_covered_file_is_incomplete(su, clean, tmp_path):
    d = _copy(clean, tmp_path / "p")
    # rewrite file 0's sidecar to cover its first block only (format restated here)
    raw = (d / "postdata_0.sum").read_bytes()
    body = raw[:104] + struct.pack("<Q", B) + raw[HEADER:HEADER + 32]
    (d / "postdata_0.sum").write_bytes(body + struct.pack("<Q", _fnv(body)))
    r = su.check_sums(str(d))
    assert r.code == su.ERR_STATE and r.labels_unchecked == 140000 - B and r.labels_checked == 300000 - (140000 - B)


def _fnv(b: bytes) -> int:
    h = 0xcbf29ce484222325
    for c in b:
        h = ((h ^ c) * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
    return h


# ------------------------------------------------------------------------------------------------------ repair
def test_repair_restores_the_files(su, tmp_path):
    lay = dict(lpu=100000, units=3, per_file=140000)
    pristine = tmp_path / "pristine"
    _session(su, pristine, proof=dict(nonces=16, pow="skip"), batch=1 << 15, **lay)
    d = _copy(pristine, tmp_path / "p")
    for i in (5, B + 9, 140000 + B, 299999):
        _flip(d, i, bit=0x80)
    r = su.check_sums(str(d), repair=True)
    assert r.code == su.OK and r.bad_blocks == 4 and r.repaired_blocks == 4
    for p in pristine.iterdir():
        assert (d / p.name).read_bytes() == p.read_bytes(), p.name
    assert su.check_sums(str(d)).code == su.OK
    v = su.verify_pos(str(d), fraction=100)
    assert v.code == su.OK and v.mismatches == 0


def test_repair_at_n8192(su, tmp_path):
    lay = dict(lpu=40000, units=2, per_file=80000, n=8192)
    pristine = tmp_path / "pristine"
    _session(su, pristine, batch=1 << 14, **lay)
    d = _copy(pristine, tmp_path / "p")
    _flip(d, B + 100, per_file=80000, bit=0x04)
    r = su.check_sums(str(d), repair=True)
    assert r.code == su.OK and r.bad == [(B, 80000 - B)] and r.repaired_blocks == 1
    assert (d / "postdata_0.bin").read_bytes() == (pristine / "postdata_0.bin").read_bytes()
    assert (d / "postdata_metadata.json").read_bytes() == (pristine / "postdata_metadata.json").read_bytes()


# -------------------------------------------------------------------------------------------------- write_sums
def test_write_sums_matches_init(su, clean, tmp_path):
    d = _copy(clean, tmp_path / "p")
    for p in d.glob("*.sum"):
        p.unlink()
    r = su.write_sums(str(d))
    assert r.code == su.OK and r.files_checked == 3 and r.labels_checked == 300000
    for p in clean.glob("*.sum"):
        assert (d / p.name).read_bytes() == p.read_bytes(), p.name
    # one damaged file: no sidecar for it, the damage reported, the others written
    e = _copy(clean, tmp_path / "e")
    for p in e.glob("*.sum"):
        p.unlink()
    _flip(e, 140000 + B + 2)
    r = su.write_sums(str(e))
    assert r.code == su.ERR_LABEL_MISMATCH and r.files_unchecked == 1 and r.files_checked == 2
    assert r.bad == [(140000 + B, B)]
    assert sorted(p.name for p in e.glob("*.sum")) == ["postdata_0.sum", "postdata_2.sum"]
