"""CPU tier: range records (request_range_record) and their merge (merge_range_records) without a device: when a record
may be requested, the merge's host checks in order (each leaves the metadata as it was), NO_DEVICE once they pass,
reset, and the b200postcli usage errors.  Records are written here by restating their layout (DESIGN.md §3c)."""
import ctypes
import importlib
import struct
import subprocess
from pathlib import Path

import pytest

NODE, ATX = bytes(range(32)), bytes(range(32, 64))
# 2 x 512 labels in files of 256: four files, two ranges of two files each
LPU, UNITS, PER_FILE, N = 512, 2, 256, 2
NUM = LPU * UNITS


@pytest.fixture()
def su(b2):
    return importlib.import_module("go-spacemesh_b200.setup")


def _opts(su, d, **kw):
    o = dict(data_dir=str(d), num_units=UNITS, max_file_size=16 * PER_FILE, provider_id=0, scrypt_n=N, compute_batch_size=1 << 10)
    o.update(kw)
    return su.PostSetupOpts(**o)


def _cfg(su):
    return su.PostConfig(labels_per_unit=LPU)


def _raises(b2, fn, *a, **kw) -> int:
    with pytest.raises(b2.B200PostError) as e:
        fn(*a, **kw)
    return e.value.code


def _fnv(b: bytes) -> int:
    h = 0xcbf29ce484222325
    for c in b:
        h = ((h ^ c) * 0x100000001b3) & (2**64 - 1)
    return h


def record(from_file, to_file, upto=None, *, node=NODE, units=UNITS, vrf=None) -> bytes:
    """A VRF-only record of files [from_file, to_file]: header | upto | VRF best (found, index, label32) | FNV-1a 64."""
    lo, hi = from_file * PER_FILE, min((to_file + 1) * PER_FILE, LPU * units)
    h = b"B2RNGREC" + struct.pack("<I", 1) + node + ATX + struct.pack("<IQQ", units, LPU, N)
    h += struct.pack("<QQQQQI", 16 * PER_FILE, from_file, to_file, lo, hi, 0)
    found, index, label = vrf or (0, 0, bytes(32))
    body = h + struct.pack("<Q", hi if upto is None else upto) + struct.pack("<IQ", found, index) + label
    return body + struct.pack("<Q", _fnv(body))


def _merged_dir(su, d, records):
    """Metadata of range session 0-1, every postdata file, and the given {name: bytes} records."""
    su.PostSetupManager(_cfg(su)).prepare_files(_opts(su, d), NODE, ATX, 0, 1)
    for f in range(4):
        (d / f"postdata_{f}.bin").write_bytes(bytes(16 * PER_FILE))
    for name, raw in records.items():
        (d / name).write_bytes(raw)
    return d


def test_request_needs_a_prepared_range_without_a_nonce(b2, su, tmp_path):
    mgr = su.PostSetupManager(_cfg(su))
    assert _raises(b2, mgr.request_range_record) == su.ERR_STATE                        # never prepared
    full = su.PostSetupManager(_cfg(su))
    full.prepare_initializer(_opts(su, tmp_path / "w"), NODE, ATX)
    assert _raises(b2, full.request_range_record) == su.ERR_STATE                       # a whole-POST session
    whole = su.PostSetupManager(_cfg(su))
    whole.prepare_files(_opts(su, tmp_path / "w2"), NODE, ATX, 0, 3)                   # the whole POST named as a range
    assert _raises(b2, whole.request_range_record, initial_proof=True, pow="skip") == su.ERR_STATE
    # re-initialising a lost file of a finished POST needs no record
    d = tmp_path / "done"
    su.PostSetupManager(_cfg(su)).prepare_initializer(_opts(su, d), NODE, ATX)
    meta = d / "postdata_metadata.json"
    meta.write_text(meta.read_text().replace('"Nonce": null', '"Nonce": 5').replace('"NonceValue": null', '"NonceValue": "' + "00" * 32 + '"'))
    mgr = su.PostSetupManager(_cfg(su))
    mgr.prepare_files(_opts(su, d), NODE, ATX, 2, 2)
    assert _raises(b2, mgr.request_range_record) == su.ERR_STATE
    # a range without a nonce: both kinds, and a second call replaces the first
    mgr = su.PostSetupManager(_cfg(su))
    mgr.prepare_files(_opts(su, tmp_path / "r"), NODE, ATX, 0, 1)
    mgr.request_range_record()
    mgr.request_range_record(initial_proof=True, nonces=32, pow="skip", windows_per_pass=3)
    mgr.request_range_record(initial_proof=True, nonces=16, pow="builtin", pow_cache_key=b"key")
    assert mgr.status().state == su.STATE_PREPARED


def test_request_argument_errors(b2, su, tmp_path):
    pr = importlib.import_module("go-spacemesh_b200.prove")
    mgr = su.PostSetupManager(_cfg(su))
    mgr.prepare_files(_opts(su, tmp_path / "r"), NODE, ATX, 2, 3)
    for bad in (8, 17, 4112):
        assert _raises(b2, mgr.request_range_record, initial_proof=True, nonces=bad, pow="skip") == b2.ERR_INVALID_ARGUMENT, bad
    assert _raises(b2, mgr.request_range_record, initial_proof=True, pow="callback-missing") == b2.ERR_UNSUPPORTED
    opts, _ = pr._opts(None, None, 16, 0, "skip")
    opts.pow_mode = 7
    assert su._bind().b200post_setup_request_range_record(mgr._h, ctypes.byref(opts)) == b2.ERR_UNSUPPORTED
    assert su._bind().b200post_setup_request_range_record(None, None) == b2.ERR_INVALID_ARGUMENT


def test_start_with_a_record_and_no_device(b2, su, tmp_path):
    if b2.providers():
        pytest.skip("a CUDA device is present: the no-device contract is covered on CPU-only boxes")
    for proof in (False, True):
        d = tmp_path / f"p{proof}"
        mgr = su.PostSetupManager(_cfg(su))
        mgr.prepare_files(_opts(su, d), NODE, ATX, 0, 1)
        mgr.request_range_record(initial_proof=proof, pow="skip")
        assert _raises(b2, mgr.start_session) == b2.ERR_NO_DEVICE
        assert not list(d.glob("range_*")) and mgr.status().state == su.STATE_ERROR


def test_merge_host_checks_in_order(b2, su, tmp_path):
    """Each refusal names its cause and leaves the metadata byte-identical; the checks run in the documented order."""
    cfg = _cfg(su)
    e = pytest.raises(b2.B200PostError, su.merge_range_records, str(tmp_path / "nowhere"), cfg)
    assert e.value.code == su.ERR_IO and "metadata" in str(e.value)                     # no metadata

    good = {"range_0_1.rec": record(0, 1), "range_2_3.rec": record(2, 3)}
    steps = [
        ("damaged", {**good, "range_2_3.rec": good["range_2_3.rec"][:40] + b"\xff" + good["range_2_3.rec"][41:]}, su.ERR_IO, "range_2_3.rec"),
        ("truncated", {**good, "range_2_3.rec": good["range_2_3.rec"][:-3]}, su.ERR_IO, "damaged"),
        ("identity", {**good, "range_2_3.rec": record(2, 3, node=bytes(32))}, su.ERR_CONFIG_MISMATCH, "another POST"),
        ("units", {**good, "range_2_3.rec": record(2, 3, units=UNITS + 1)}, su.ERR_CONFIG_MISMATCH, "another POST"),
        ("gap", {"range_0_0.rec": record(0, 0), "range_2_3.rec": record(2, 3)}, su.ERR_STATE, "[256, 512)"),
        ("tail", {"range_0_1.rec": record(0, 1)}, su.ERR_STATE, "[512, 1024)"),
        ("none", {}, su.ERR_STATE, "[0, 1024)"),
        ("overlap", {**good, "range_1_2.rec": record(1, 2)}, su.ERR_STATE, "overlap"),
        ("incomplete", {**good, "range_2_3.rec": record(2, 3, upto=700)}, su.ERR_STATE, "incomplete"),
    ]
    for name, recs, code, text in steps:
        d = _merged_dir(su, tmp_path / name, recs)
        before = (d / "postdata_metadata.json").read_bytes()
        e = pytest.raises(b2.B200PostError, su.merge_range_records, str(d), cfg)
        assert e.value.code == code and text in str(e.value), (name, str(e.value))
        assert (d / "postdata_metadata.json").read_bytes() == before, name
    # the records pass; the data does not
    for name, fix in (("missing", lambda d: (d / "postdata_3.bin").unlink()),
                      ("short", lambda d: (d / "postdata_1.bin").write_bytes(bytes(16 * PER_FILE - 16)))):
        d = _merged_dir(su, tmp_path / name, good)
        fix(d)
        before = (d / "postdata_metadata.json").read_bytes()
        e = pytest.raises(b2.B200PostError, su.merge_range_records, str(d), cfg)
        assert e.value.code == su.ERR_IO and "incomplete" in str(e.value), name
        assert (d / "postdata_metadata.json").read_bytes() == before, name
    # another LabelsPerUnit asked for
    d = _merged_dir(su, tmp_path / "lpu", good)
    assert _raises(b2, su.merge_range_records, str(d), su.PostConfig(labels_per_unit=LPU * 2)) == su.ERR_CONFIG_MISMATCH


def test_merge_without_a_device(b2, su, tmp_path):
    d = _merged_dir(su, tmp_path / "m", {"range_0_1.rec": record(0, 1, vrf=(1, 3, bytes(32))), "range_2_3.rec": record(2, 3)})
    (d / "initial_post.json").write_text("{}")
    before = {p.name: p.read_bytes() for p in d.iterdir()}
    assert _raises(b2, su.merge_range_records, str(d), _cfg(su), provider_id=0xffffffff) == b2.ERR_UNSUPPORTED
    if b2.providers():
        pytest.skip("a CUDA device is present: NO_DEVICE cannot be observed")
    for prov in (0, su.PROVIDER_ALL):
        assert _raises(b2, su.merge_range_records, str(d), _cfg(su), provider_id=prov) == b2.ERR_NO_DEVICE
    assert {p.name: p.read_bytes() for p in d.iterdir()} == before                     # nothing written, nothing removed


def test_reset_removes_records(su, tmp_path):
    d = tmp_path / "r"
    mgr = su.PostSetupManager(_cfg(su))
    mgr.prepare_files(_opts(su, d), NODE, ATX, 0, 1)
    (d / "range_0_1.rec").write_bytes(record(0, 1))
    (d / "range_2_3.rec.tmp").write_bytes(b"x")
    (d / "range_notes.txt").write_text("not ours")
    mgr.reset()
    assert sorted(p.name for p in d.iterdir()) == ["range_notes.txt"]


def _cli(b2):
    cli = Path(b2.LIB_PATH).parent / "b200postcli"
    if not cli.exists():
        pytest.skip("b200postcli not built")
    return str(cli)


def test_cli_usage_errors(b2, tmp_path):
    init = [_cli(b2), "-id", NODE.hex(), "-commitmentAtxId", ATX.hex(), "-datadir", str(tmp_path / "c"), "-numUnits", str(UNITS),
            "-labelsPerUnit", str(LPU), "-maxFileSize", str(16 * PER_FILE), "-scryptN", str(N)]
    for extra in (["-fromFile", "0", "-toFile", "1", "-initialProof"],      # the initial proof of a range needs a record
                  ["-rangeRecord"],                                         # a record needs a range
                  ["-rangeRecord", "-initialProof"],
                  ["-fromFile", "0", "-toFile", "3", "-rangeRecord"],       # the whole POST named as a range
                  ["-fromFile", "0", "-toFile", "1", "-rangeRecord", "-initialProof", "-nonces", "17"]):
        r = subprocess.run(init + extra, capture_output=True, text=True, timeout=60)
        assert r.returncode == 2, (extra, r.stdout + r.stderr)
        assert not list((tmp_path / "c").glob("postdata_*.bin")) if (tmp_path / "c").exists() else True
    merge = [_cli(b2), "-mergeRanges", "-datadir", str(tmp_path / "nothing")]
    r = subprocess.run(merge + ["-provider", "4294967295"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 2, r.stdout + r.stderr
    r = subprocess.run(merge, capture_output=True, text=True, timeout=60)
    assert r.returncode == 1 and "metadata" in r.stderr, r.stdout + r.stderr
    r = subprocess.run(merge + ["-powDifficulty", "zz"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 2, r.stdout + r.stderr
