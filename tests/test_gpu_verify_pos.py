"""GPU tier: b200post_verify_pos / b200postcli -verify on POST data written by setup sessions, clean and with labels
corrupted on disk.  Layer shapes are forced with max_scratch_mib so that the low-latency, single-layer and pipelined
(speculating) engine paths all compare labels."""
import ctypes
import importlib
import json
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NODE, ATX = bytes(range(40, 72)), bytes(range(3, 35))


@pytest.fixture(scope="module")
def su(b2, gpu_ready):
    return importlib.import_module("go-spacemesh_b200.setup")


class Opt:
    """Sets engine options for a block and restores them."""

    def __init__(self, b2, **kw):
        self.b2, self.kw = b2, kw

    def __enter__(self):
        self.old = {k: self.b2.get_option(k) for k in self.kw}
        for k, v in self.kw.items():
            self.b2.set_option(k, v)

    def __exit__(self, *a):
        for k, v in self.old.items():
            self.b2.set_option(k, v)


def _init(su, d: Path, *, labels_per_unit, num_units, labels_per_file, scrypt_n=2, batch=1 << 16):
    mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=labels_per_unit, max_num_units=max(10, num_units)))
    mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=num_units, max_file_size=16 * labels_per_file,
                                             provider_id=0, scrypt_n=scrypt_n, compute_batch_size=batch), NODE, ATX)
    mgr.start_session()
    assert mgr.status().state == su.STATE_COMPLETE
    return d


@pytest.fixture(scope="module")
def posts(su, b2, tmp_path_factory):
    """Clean POSTs, written once; tests work on copies.
    small: 2 x 512 labels in 4 files (BASELINE.json configs[0]); odd: 3000 labels in files of 700 (the last CTA of the
    check is partial); aligned: 4096 labels in files of 1024 (two whole 2048-slot layers under max_scratch_mib = 1)."""
    root = tmp_path_factory.mktemp("posts")
    return {
        "small": (_init(su, root / "small", labels_per_unit=512, num_units=2, labels_per_file=256), 256),
        "odd": (_init(su, root / "odd", labels_per_unit=1000, num_units=3, labels_per_file=700), 700),
        "aligned": (_init(su, root / "aligned", labels_per_unit=1024, num_units=4, labels_per_file=1024), 1024),
    }


def _copy(posts, name, tmp_path):
    src, per_file = posts[name]
    dst = tmp_path / name
    shutil.copytree(src, dst)
    return str(dst), per_file


def _flip(d, per_file, index, byte=5, bit=3):
    p = Path(d) / f"postdata_{index // per_file}.bin"
    with open(p, "r+b") as f:
        f.seek((index % per_file) * 16 + byte)
        v = f.read(1)[0]
        f.seek(-1, 1)
        f.write(bytes([v ^ (1 << bit)]))


def test_clean_small_post_full_check(su, b2, posts, tmp_path):
    d, _ = _copy(posts, "small", tmp_path)
    prog = ctypes.c_uint64(0)
    r = su.verify_pos(d, fraction=100.0, progress=prog)
    assert r.code == b2.OK and r.labels_checked == 1024 and r.files_checked == 4 and r.mismatches == 0
    assert r.nonce_ok and r.argmin_checked and r.argmin_ok and r.bad_index == []
    assert prog.value == 1024
    assert "b200post_post_data_labels_verified_total" in b2.metrics_text()


def test_clean_n8192_post_pipelined(su, b2, tmp_path):
    """N = 8192 with 256-slot layers: 4096 labels are 16 layers, checked in two calls of 8 (the second resumes the
    first's speculative fill)."""
    with Opt(b2, max_scratch_mib=512):
        assert b2.wave_slots(8192) == 256
        d = _init(su, tmp_path / "n8192", labels_per_unit=4096, num_units=1, labels_per_file=1024, scrypt_n=8192, batch=4096)
        r = su.verify_pos(str(d), fraction=100.0)
        assert r.code == b2.OK and r.labels_checked == 4096 and r.mismatches == 0 and r.nonce_ok and r.argmin_ok
        for i in (0, 1023, 2047, 2048, 4095):
            _flip(d, 1024, i)
        r = su.verify_pos(str(d), fraction=100.0)
        assert r.code == su.ERR_LABEL_MISMATCH and r.bad_index == [0, 1023, 2047, 2048, 4095] and r.mismatches == 5


@pytest.mark.parametrize("shape", ["lowlat", "single_layer", "two_layers"])
def test_single_bit_flips_are_reported_exactly(su, b2, posts, tmp_path, shape):
    """0, the last label of file 0, the first of file 1, one in the last (partial) CTA, and the last label."""
    d, per_file = _copy(posts, "odd", tmp_path)
    flips = [0, 699, 700, 2950, 2999]
    for i in flips:
        _flip(d, per_file, i)
    opts = {"lowlat": {}, "single_layer": dict(lowlat_max_labels=0), "two_layers": dict(max_scratch_mib=1, lowlat_max_labels=0)}[shape]
    with Opt(b2, **opts):
        r = su.verify_pos(d, fraction=100.0)
    assert r.code == su.ERR_LABEL_MISMATCH and r.mismatches == 5 and r.bad_index == flips and r.labels_checked == 3000
    assert r.nonce_ok


@pytest.mark.parametrize("name", ["aligned", "odd"])
def test_many_flips_report_the_lowest_64(su, b2, posts, tmp_path, name):
    d, per_file = _copy(posts, name, tmp_path)
    total = {"aligned": 4096, "odd": 3000}[name]
    flips = np.sort(np.random.default_rng(5).choice(total, 100, replace=False))
    for k, i in enumerate(flips):
        _flip(d, per_file, int(i), byte=k % 16, bit=k % 8)
    with Opt(b2, max_scratch_mib=1):
        r = su.verify_pos(d, fraction=100.0)
    assert r.code == su.ERR_LABEL_MISMATCH and r.mismatches == 100 and r.bad_index == [int(x) for x in flips[:64]]


def test_file_range(su, b2, posts, tmp_path):
    d, per_file = _copy(posts, "small", tmp_path)
    _flip(d, per_file, 3 * 256 + 17)
    r = su.verify_pos(d, fraction=100.0, from_file=0, to_file=2)
    assert r.code == b2.OK and r.labels_checked == 768 and r.files_checked == 3 and not r.argmin_checked
    r = su.verify_pos(d, fraction=100.0, from_file=3, to_file=3)
    assert r.code == su.ERR_LABEL_MISMATCH and r.labels_checked == 256 and r.bad_index == [3 * 256 + 17]


def _expected_sampled(su, seed, per_file, total, fraction, flips):
    chosen = set()
    n = 0
    for f in range((total + per_file - 1) // per_file):
        L = min(per_file, total - f * per_file)
        s = su.verify_pos_sample(seed, f, L, fraction)
        n += len(s)
        chosen |= {f * per_file + int(x) for x in s}
    return n, sorted(i for i in flips if i in chosen)


@pytest.mark.parametrize("fraction", [25.0, 50.0])
def test_sampled_check(su, b2, posts, tmp_path, fraction):
    d, per_file = _copy(posts, "odd", tmp_path)
    flips = sorted(int(x) for x in np.random.default_rng(8).choice(3000, 300, replace=False))
    for i in flips:
        _flip(d, per_file, i)
    r = su.verify_pos(d, fraction=fraction, seed=1234)
    n, bad = _expected_sampled(su, 1234, per_file, 3000, fraction, flips)
    assert r.seed == 1234 and r.labels_checked == n and r.files_checked == 5
    assert r.mismatches == len(bad) and r.bad_index == bad[:64] and r.code == su.ERR_LABEL_MISMATCH
    assert not r.argmin_checked and r.nonce_ok
    assert su.verify_pos(d, fraction=fraction, seed=1234) == r                       # same seed, same result
    r0 = su.verify_pos(d, fraction=fraction)                                          # seed 0: drawn, and returned
    assert r0.seed != 0 and su.verify_pos(d, fraction=fraction, seed=r0.seed) == r0


def test_sparse_sample_of_a_large_post_takes_positioned_reads_and_the_low_latency_kernel(su, b2, tmp_path):
    """0.1 % of a 2^20-label POST: 262 positions per 2^18-label file (far below 1 per 4 KiB page), 1048 items in one
    indexed job of <= 4096 items: K1 + K2 low-latency + K3c, three launches, plus the nonce label's four."""
    per_file = 1 << 18
    d = _init(su, tmp_path / "big", labels_per_unit=1 << 18, num_units=4, labels_per_file=per_file, batch=1 << 18)
    n, _ = _expected_sampled(su, 77, per_file, 1 << 20, 0.1, [])
    victims = [f * per_file + int(su.verify_pos_sample(77, f, per_file, 0.1)[k]) for f, k in ((0, 0), (1, 100), (3, 261))]
    for i in victims:
        _flip(str(d), per_file, i)
    before = b2.launch_count()
    r = su.verify_pos(str(d), fraction=0.1, seed=77)
    assert b2.launch_count() - before == 3 + 4
    assert r.code == su.ERR_LABEL_MISMATCH and r.labels_checked == n == 4 * 262 and r.bad_index == victims


def test_file_samples_spanning_two_compare_jobs(su, b2, tmp_path):
    """Two files of 2^23 labels at 30 %: 2 516 582 positions each, 5 033 164 in all, more than one indexed job holds
    (2^22), so the second file's streamed sample is split between the two jobs."""
    per_file = 1 << 23
    d = _init(su, tmp_path / "two", labels_per_unit=1 << 23, num_units=2, labels_per_file=per_file, batch=1 << 22)
    s = [f * per_file + su.verify_pos_sample(21, f, per_file, 30.0).astype(np.int64) for f in range(2)]
    chosen = np.concatenate(s)
    assert len(chosen) > 1 << 22
    rng = np.random.default_rng(4)
    flips = sorted(set(int(x) for x in rng.choice(chosen, 40, replace=False)) | {int(x) for x in rng.integers(0, 2 * per_file, 40)})
    for i in flips:
        _flip(str(d), per_file, i)
    r = su.verify_pos(str(d), fraction=30.0, seed=21)
    bad = [i for i in flips if np.isin(i, chosen)]
    assert r.code == su.ERR_LABEL_MISMATCH and r.labels_checked == len(chosen) and r.files_checked == 2
    assert r.mismatches == len(bad) and r.bad_index == bad[:64]


def test_post_without_nonce_is_unfinished_not_corrupt(su, b2, tmp_path):
    """Metadata from prepare_initializer only (no VRF nonce yet), complete label files: every label is checked, the call
    says initialisation has not finished (ERR_STATE) instead of reporting a mismatch; a bad label still wins."""
    d = tmp_path / "nononce"
    mgr = su.PostSetupManager()
    mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=2, max_file_size=4096, provider_id=0, scrypt_n=2),
                            NODE, ATX)
    labels, _ = b2.labels_range(b2.commitment(NODE, ATX), 2, 0, 1024)
    for f in range(4):
        (d / f"postdata_{f}.bin").write_bytes(labels[256 * f: 256 * (f + 1)].tobytes())
    assert su.load_metadata(str(d))["nonce"] is None
    for fraction in (100.0, 10.0):
        r = su.verify_pos(str(d), fraction=fraction, seed=3)
        assert r.code == su.ERR_STATE and r.mismatches == 0 and not r.nonce_ok and not r.argmin_checked
        assert r.labels_checked == (1024 if fraction == 100.0 else 4 * 25)
    _flip(str(d), 256, 600)
    r = su.verify_pos(str(d), fraction=100.0)
    assert r.code == su.ERR_LABEL_MISMATCH and r.bad_index == [600]


def test_corrupted_nonce_value(su, b2, posts, tmp_path):
    d, _ = _copy(posts, "small", tmp_path)
    meta = Path(d) / "postdata_metadata.json"
    doc = json.loads(meta.read_text())
    v = bytearray(bytes.fromhex(doc["NonceValue"]))
    v[31] ^= 1
    doc["NonceValue"] = v.hex()
    meta.write_text(json.dumps(doc))
    for fraction in (100.0, 1.0):
        r = su.verify_pos(d, fraction=fraction)
        assert r.code == su.ERR_LABEL_MISMATCH and not r.nonce_ok and r.mismatches == 0
    assert not su.verify_pos(d, fraction=100.0).argmin_ok


def test_preset_cancel(su, b2, posts, tmp_path):
    d, _ = _copy(posts, "small", tmp_path)
    for fraction in (100.0, 10.0):
        r = su.verify_pos(d, fraction=fraction, cancel=ctypes.c_int(1))
        assert r.code == b2.ERR_CANCELLED and r.labels_checked == 0


def test_all_providers_match_provider_0(su, b2, posts, tmp_path):
    if len(b2.providers()) < 2:
        pytest.skip("needs >= 2 GPUs")
    d, per_file = _copy(posts, "odd", tmp_path)
    for i in (3, 1500, 2999):
        _flip(d, per_file, i)
    for fraction in (100.0, 30.0):
        a = su.verify_pos(d, fraction=fraction, seed=5)
        b = su.verify_pos(d, fraction=fraction, seed=5, provider_id=su.PROVIDER_ALL)
        assert a == b


def test_cli_verify(b2, posts, tmp_path):
    cli = Path(b2.LIB_PATH).parent / "b200postcli"
    if not cli.exists():
        pytest.skip("b200postcli not built")
    d, per_file = _copy(posts, "small", tmp_path)
    args = [str(cli), "-verify", "-datadir", d, "-fraction", "100"]
    r = subprocess.run(args, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "valid" in r.stdout
    _flip(d, per_file, 300)
    r = subprocess.run(args, capture_output=True, text=True, timeout=120)
    assert r.returncode == 1 and "file 1 offset 704 (label 300)" in r.stdout, r.stdout + r.stderr
