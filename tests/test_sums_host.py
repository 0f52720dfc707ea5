"""CPU tier: the host side of block checksums.  The order and codes of the host checks of check_sums, write_sums and
the init request, on sidecars written here by a restatement of the postdata_<N>.sum format; reset removing sidecars and
their leftovers; b200postcli's usage errors for the checksum flags."""
import importlib
import struct
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
CLI = ROOT / "go-spacemesh_b200" / "b200postcli"
NODE, ATX = bytes(range(32)), bytes(range(32, 64))
B = 1 << 16
PER_FILE, N = 1000, 2   # 2 x 1200 labels in files of 1000: files of 1000, 1000 and 400 labels


@pytest.fixture()
def su(b2):
    return importlib.import_module("go-spacemesh_b200.setup")


def _fnv(b: bytes) -> int:
    h = 0xcbf29ce484222325
    for c in b:
        h = ((h ^ c) * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
    return h


def sidecar(file: int, covered: int, *, node=NODE, atx=ATX, n=N, per_file=PER_FILE, version=1, digest=b"\x11" * 32) -> bytes:
    """postdata_<file>.sum: magic | version | block labels | NodeId | CommitmentAtxId | N | labels per file | file |
    covered | one digest per block | FNV-1a 64 of everything before it."""
    body = b"B2PSUMS1" + struct.pack("<II", version, B) + node + atx + struct.pack("<QQQQ", n, per_file, file, covered)
    body += digest * ((covered + B - 1) // B)
    return body + struct.pack("<Q", _fnv(body))


def _post(su, d: Path, *, files=(1000, 1000, 400)) -> Path:
    """metadata from a prepare, and zero-filled files of the given label counts"""
    mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=1200))
    mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=2, max_file_size=16 * PER_FILE, provider_id=0, scrypt_n=N,
                                             compute_batch_size=1 << 10), NODE, ATX)
    for i, n in enumerate(files):
        (d / f"postdata_{i}.bin").write_bytes(bytes(16 * n))
    return d


def _code(b2, fn, *a, **kw):
    with pytest.raises(b2.B200PostError) as e:
        fn(*a, **kw)
    return e.value.code, str(e.value)


def test_sidecar_format_constants():
    s = sidecar(0, 1000)
    assert len(s) == 112 + 32 + 8


@pytest.mark.parametrize("call", ["check_sums", "write_sums"])
def test_missing_metadata_and_incomplete_files(su, b2, tmp_path, call):
    fn = getattr(su, call)
    code, msg = _code(b2, fn, str(tmp_path / "none"))
    assert code == su.ERR_IO and "metadata file is missing" in msg
    d = _post(su, tmp_path / "short", files=(1000, 999, 400))
    (d / "postdata_0.sum").write_bytes(sidecar(0, 1000))
    code, msg = _code(b2, fn, str(d))
    assert code == su.ERR_IO and "incomplete" in msg
    # a file range that leaves the short file out passes the size check
    if not b2.providers():
        code, _ = _code(b2, fn, str(d), to_file=0)
        assert code == b2.ERR_NO_DEVICE
    code, _ = _code(b2, fn, str(d), from_file=2, to_file=1)
    assert code == b2.ERR_INVALID_ARGUMENT


def _unusable(su, b2, d: Path, name: str, data: bytes):
    for p in d.glob("*.sum"):
        p.unlink()
    (d / name).write_bytes(data)
    code, msg = _code(b2, su.check_sums, str(d))
    assert code == su.ERR_STATE and "no checksums" in msg, name


def test_unusable_sidecars_leave_nothing_to_check(su, b2, tmp_path):
    d = _post(su, tmp_path / "p")
    code, msg = _code(b2, su.check_sums, str(d))                       # none at all
    assert code == su.ERR_STATE and "no checksums" in msg
    good = sidecar(1, 1000)
    bad_sum = good[:-1] + bytes([good[-1] ^ 1])
    _unusable(su, b2, d, "postdata_1.sum", bad_sum)                    # damaged checksum
    _unusable(su, b2, d, "postdata_1.sum", good[:-9] + good[-8:])      # truncated
    _unusable(su, b2, d, "postdata_1.sum", sidecar(1, 1000, node=bytes(32)))
    _unusable(su, b2, d, "postdata_1.sum", sidecar(1, 1000, atx=bytes(32)))
    _unusable(su, b2, d, "postdata_1.sum", sidecar(1, 1000, n=4))
    _unusable(su, b2, d, "postdata_1.sum", sidecar(1, 1000, per_file=2000))
    _unusable(su, b2, d, "postdata_1.sum", sidecar(0, 1000))           # made for file 0
    _unusable(su, b2, d, "postdata_1.sum", sidecar(1, 1000, version=2))
    _unusable(su, b2, d, "postdata_2.sum", sidecar(2, 401))            # covers more than the file holds
    _unusable(su, b2, d, "postdata_1.sum", sidecar(1, 0))              # covers nothing


def test_valid_sidecars_reach_the_device(su, b2, tmp_path):
    d = _post(su, tmp_path / "p")
    (d / "postdata_2.sum").write_bytes(sidecar(2, 400))
    (d / "postdata_1.sum").write_bytes(sidecar(1, 500))                # partly covered is usable
    code, _ = _code(b2, su.check_sums, str(d), provider_id=b2.CPU_PROVIDER_ID)
    assert code == b2.ERR_UNSUPPORTED
    code, _ = _code(b2, su.write_sums, str(d), provider_id=b2.CPU_PROVIDER_ID)
    assert code == b2.ERR_UNSUPPORTED
    # the check runs on one device: PROVIDER_ALL is for write_sums only
    code, _ = _code(b2, su.check_sums, str(d), provider_id=su.PROVIDER_ALL)
    assert code == b2.ERR_INVALID_ARGUMENT
    if b2.providers():
        pytest.skip("a CUDA device is present: NO_DEVICE cannot be observed")
    code, _ = _code(b2, su.check_sums, str(d))
    assert code == b2.ERR_NO_DEVICE
    code, _ = _code(b2, su.check_sums, str(d), from_file=1, to_file=1, repair=True)
    assert code == b2.ERR_NO_DEVICE
    code, _ = _code(b2, su.write_sums, str(d))
    assert code == b2.ERR_NO_DEVICE
    code, _ = _code(b2, su.write_sums, str(d), provider_id=su.PROVIDER_ALL)
    assert code == b2.ERR_NO_DEVICE


def test_init_request(su, b2, tmp_path):
    mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=1200))
    code, msg = _code(b2, mgr.request_checksums)                       # before prepare
    assert code == su.ERR_STATE and "not prepared" in msg
    opts = su.PostSetupOpts(data_dir=str(tmp_path / "i"), num_units=2, max_file_size=16 * PER_FILE, provider_id=0, scrypt_n=N,
                            compute_batch_size=1 << 10)
    mgr.prepare_initializer(opts, NODE, ATX)
    mgr.request_checksums()
    mgr.request_checksums()                                            # asking twice is asking once
    # a file-range session takes the request too
    rng = su.PostSetupManager(su.PostConfig(labels_per_unit=1200))
    rng.prepare_files(su.PostSetupOpts(data_dir=str(tmp_path / "r"), num_units=2, max_file_size=16 * PER_FILE, provider_id=0,
                                       scrypt_n=N, compute_batch_size=1 << 10), NODE, ATX, 1, 2)
    rng.request_checksums()
    if b2.providers():
        pytest.skip("a CUDA device is present: NO_DEVICE cannot be observed")
    for m in (mgr, rng):
        code, _ = _code(b2, m.start_session)
        assert code == b2.ERR_NO_DEVICE and m.status().state == su.STATE_ERROR
    # complete data still has sidecars to make: the request needs a provider
    d = _post(su, tmp_path / "done")
    m = su.PostSetupManager(su.PostConfig(labels_per_unit=1200))
    m.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=2, max_file_size=16 * PER_FILE, scrypt_n=N,
                                           compute_batch_size=1 << 10), NODE, ATX)
    m.request_checksums()
    code, msg = _code(b2, m.start_session)
    assert code == su.ERR_NO_PROVIDER


def test_reset_deletes_sidecars_and_leftovers(su, tmp_path):
    d = _post(su, tmp_path / "p")
    mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=1200))
    mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=2, max_file_size=16 * PER_FILE, provider_id=0, scrypt_n=N,
                                             compute_batch_size=1 << 10), NODE, ATX)
    (d / "postdata_0.sum").write_bytes(sidecar(0, 1000))
    (d / "postdata_1.sum.tmp").write_bytes(b"partial")
    (d / "postdata_x.txt").write_bytes(b"not ours")
    (d / "notes.sum").write_bytes(b"not ours")
    mgr.reset()
    assert sorted(p.name for p in d.iterdir()) == ["notes.sum", "postdata_x.txt"]


def _cli(*args):
    return subprocess.run([str(CLI), *args], capture_output=True, text=True)


def test_cli_usage_errors(su, tmp_path):
    d = str(tmp_path)
    r = _cli("-verify", "-writeSums", "-datadir", d)                   # default fraction 0.2
    assert r.returncode == 2 and "-fraction 100" in r.stderr
    r = _cli("-verify", "-fraction", "50", "-writeSums", "-datadir", d)
    assert r.returncode == 2
    r = _cli("-writeSums", "-fraction", "100", "-datadir", d)          # without -verify
    assert r.returncode == 2
    r = _cli("-repair", "-datadir", d)
    assert r.returncode == 2 and "-checkSums" in r.stderr
    r = _cli("-verify", "-repair", "-datadir", d)
    assert r.returncode == 2
    r = _cli("-checkSums", "-datadir", d, "-provider", "4294967295")
    assert r.returncode == 2
    r = _cli("-checkSums", "-datadir", d)                              # no metadata: an error, not a usage error
    assert r.returncode == 1 and "metadata file is missing" in r.stderr
