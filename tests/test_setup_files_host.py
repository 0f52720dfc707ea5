"""CPU tier: file-range setup sessions (prepare_files), the VrfScanPending marker, b200postcli -printNumFiles, the host
checks of search_vrf_nonce, and the stored-arg-min rule it applies, restated here against the oracle's VRF scan."""
import importlib
import json
import subprocess
from pathlib import Path

import numpy as np
import pytest

NODE, ATX = bytes(range(32)), bytes(range(32, 64))


@pytest.fixture()
def su(b2):
    return importlib.import_module("go-spacemesh_b200.setup")


def _opts(su, d, **kw):
    # 2 x 512 labels in files of 256: four files
    o = dict(data_dir=str(d), num_units=2, max_file_size=4096, provider_id=0, scrypt_n=2, compute_batch_size=1 << 10)
    o.update(kw)
    return su.PostSetupOpts(**o)


def test_prepare_files_rejects_ranges_outside_the_post(su, b2, tmp_path):
    for lo, hi in ((2, 1), (0, 4), (3, 7), (4, -1), (0, -2), (1, -5)):
        mgr = su.PostSetupManager()
        with pytest.raises(b2.B200PostError) as e:
            mgr.prepare_files(_opts(su, tmp_path / "p"), NODE, ATX, lo, hi)
        assert e.value.code == b2.ERR_INVALID_ARGUMENT, (lo, hi)
        assert mgr.status().state == su.STATE_ERROR
    for lo, hi in ((0, 3), (3, 3), (3, -1), (1, 2)):
        mgr = su.PostSetupManager()
        mgr.prepare_files(_opts(su, tmp_path / f"ok{lo}{hi}"), NODE, ATX, lo, hi)
        assert mgr.status().state == su.STATE_PREPARED


def test_range_prepare_sets_the_marker_and_a_full_prepare_does_not(su, tmp_path):
    su.PostSetupManager().prepare_files(_opts(su, tmp_path / "r"), NODE, ATX, 1, 2)
    md = su.load_metadata(str(tmp_path / "r"))
    assert md["vrf_scan_pending"] == 1 and md["nonce"] is None
    assert json.loads((tmp_path / "r" / "postdata_metadata.json").read_text())["VrfScanPending"] is True
    su.PostSetupManager().prepare_initializer(_opts(su, tmp_path / "f"), NODE, ATX)
    assert su.load_metadata(str(tmp_path / "f"))["vrf_scan_pending"] == 0
    assert "VrfScanPending" not in json.loads((tmp_path / "f" / "postdata_metadata.json").read_text())
    # the whole POST named as a range is a full session
    su.PostSetupManager().prepare_files(_opts(su, tmp_path / "w"), NODE, ATX, 0, 3)
    assert su.load_metadata(str(tmp_path / "w"))["vrf_scan_pending"] == 0
    # a full prepare keeps the marker of merged data
    su.PostSetupManager().prepare_initializer(_opts(su, tmp_path / "r"), NODE, ATX)
    assert su.load_metadata(str(tmp_path / "r"))["vrf_scan_pending"] == 1


def test_metadata_without_the_key_and_with_a_nonce(su, tmp_path):
    d = tmp_path / "n"
    su.PostSetupManager().prepare_initializer(_opts(su, d), NODE, ATX)
    meta = d / "postdata_metadata.json"
    doc = json.loads(meta.read_text())
    assert "VrfScanPending" not in doc and su.load_metadata(str(d))["vrf_scan_pending"] == 0
    doc["Nonce"], doc["NonceValue"] = 77, "00" * 32
    meta.write_text(json.dumps(doc))
    mgr = su.PostSetupManager()
    mgr.prepare_files(_opts(su, d), NODE, ATX, 2, 2)                 # re-initialising one file of a finished POST
    md = su.load_metadata(str(d))
    assert md["vrf_scan_pending"] == 0 and md["nonce"] == 77 and md["nonce_value"] == bytes(32)


def test_range_resume_counts_the_range_only(su, b2, tmp_path):
    d = tmp_path / "res"
    d.mkdir()
    (d / "postdata_0.bin").write_bytes(bytes(4096))                    # outside the range: not counted, not touched
    (d / "postdata_2.bin").write_bytes(bytes(4096))
    (d / "postdata_3.bin").write_bytes(bytes(1600))
    mgr = su.PostSetupManager()
    mgr.prepare_files(_opts(su, d), NODE, ATX, 2, 3)
    st = mgr.status()
    assert st.state == su.STATE_PREPARED and st.num_labels_written == 256 + 100
    assert sorted(p.name for p in d.iterdir()) == ["postdata_0.bin", "postdata_2.bin", "postdata_3.bin", "postdata_metadata.json"]
    (d / "postdata_2.bin").write_bytes(bytes(4112))                    # one label too many for a file
    with pytest.raises(b2.B200PostError) as e:
        su.PostSetupManager().prepare_files(_opts(su, d), NODE, ATX, 2, 3)
    assert e.value.code == su.ERR_CONFIG_MISMATCH


def _cli(b2):
    cli = Path(b2.LIB_PATH).parent / "b200postcli"
    if not cli.exists():
        pytest.skip("b200postcli not built")
    return str(cli)


@pytest.mark.parametrize("units,lpu,size,want", [(2, 512, 4096, 4), (3, 1000, 700 * 16, 5), (1, 4096, 1 << 30, 1),
                                                 (4, 1 << 20, 1 << 24, 4), (32, 1 << 32, 1 << 32, 512)])
def test_cli_print_num_files(b2, units, lpu, size, want):
    r = subprocess.run([_cli(b2), "-printNumFiles", "-numUnits", str(units), "-labelsPerUnit", str(lpu), "-maxFileSize", str(size)],
                       capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.strip() == str(want), r.stdout + r.stderr


def test_cli_range_usage_errors(b2, tmp_path):
    args = [_cli(b2), "-id", NODE.hex(), "-commitmentAtxId", ATX.hex(), "-datadir", str(tmp_path / "c"), "-numUnits", "2",
            "-labelsPerUnit", "512", "-maxFileSize", "4096", "-scryptN", "2"]
    r = subprocess.run(args + ["-fromFile", "3", "-toFile", "4"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 2, r.stdout + r.stderr
    assert not (tmp_path / "c" / "postdata_3.bin").exists()


def _complete_files(su, d, labels=None):
    su.PostSetupManager().prepare_initializer(_opts(su, d), NODE, ATX)
    for f in range(4):
        (d / f"postdata_{f}.bin").write_bytes(bytes(4096) if labels is None else labels[256 * f: 256 * (f + 1)].tobytes())


def test_search_host_checks_come_before_the_device(su, b2, tmp_path):
    with pytest.raises(b2.B200PostError) as e:
        su.search_vrf_nonce(str(tmp_path / "nowhere"))
    assert e.value.code == su.ERR_IO and "metadata" in str(e.value)
    d = tmp_path / "s"
    _complete_files(su, d)
    (d / "postdata_2.bin").write_bytes(bytes(4080))                    # short
    with pytest.raises(b2.B200PostError) as e:
        su.search_vrf_nonce(str(d))
    assert e.value.code == su.ERR_IO and "incomplete" in str(e.value) and "postdata_2.bin" in str(e.value)
    (d / "postdata_2.bin").unlink()                                    # missing
    with pytest.raises(b2.B200PostError) as e:
        su.search_vrf_nonce(str(d))
    assert e.value.code == su.ERR_IO and "incomplete" in str(e.value)
    (d / "postdata_2.bin").write_bytes(bytes(4096))
    before = (d / "postdata_metadata.json").read_bytes()
    if b2.providers():
        pytest.skip("a CUDA device is present: NO_DEVICE cannot be observed")
    for prov in (0, su.PROVIDER_ALL):
        with pytest.raises(b2.B200PostError) as e:                   # complete data, no GPU: no CPU fallback
            su.search_vrf_nonce(str(d), provider_id=prov)
        assert e.value.code == b2.ERR_NO_DEVICE
    assert (d / "postdata_metadata.json").read_bytes() == before


def stored_argmin_rule(orc, stored: np.ndarray, commitment: bytes, n: int, num_labels: int):
    """The rule b200post_search_vrf_nonce applies, restated: the lowest stored 16-byte prefix decides the arg-min of
    label32 (lowest index on ties); each position at that prefix has its label32 recomputed; it is the nonce only if
    strictly below floor(2^256 / numLabels).  Returns (index, label32) or None (the past-the-end search decides)."""
    keys = [bytes(stored[i]) for i in range(len(stored))]
    low = min(keys)
    ties = [i for i, k in enumerate(keys) if k == low]
    full = [(orc.c_label32(commitment, i, n), i) for i in ties]
    for l32, i in full:
        assert l32[:16] == low, f"damaged at {i}"
    l32, i = min(full)
    return (i, l32) if l32 < orc.py_vrf_difficulty(num_labels) else None


def _py_stored_argmin(stored: np.ndarray):
    keys = [bytes(r) for r in stored]
    low = min(keys)
    ties = [i for i, k in enumerate(keys) if k == low]
    return ties[0], ties


def _planted(rng, n, rows):
    """n random rows whose first byte is at least 1, with `rows` (16-byte strings) planted at distinct random positions."""
    a = rng.integers(0, 256, (n, 16), dtype=np.uint8)
    a[:, 0] |= 1
    for p, r in zip(rng.choice(n, len(rows), replace=False), rows):
        a[p] = np.frombuffer(r, dtype=np.uint8)
    return a


def test_np_stored_argmin_matches_a_bytes_min(orc):
    """np_stored_argmin (the GPU stored-scan tests' reference) against Python's min over bytes, with the orderings a
    word-wise compare gets wrong planted among random rows."""
    rng = np.random.default_rng(7)
    z = bytes(16)

    def b(**at):   # zero row with byte i set to at[f"b{i}"]
        r = bytearray(16)
        for k, v in at.items():
            r[int(k[1:])] = v
        return bytes(r)
    cases = {
        "same first 8 bytes": [b(b3=1, b9=5), b(b3=1, b9=4), b(b3=1, b15=9)],
        "same first 15 bytes": [b(b2=7, b15=3), b(b2=7, b15=2), b(b2=7, b15=4)],
        "byte order in the high word": [b(b2=1), b(b3=1), b(b7=1)],
        "byte order in the low word": [b(b1=1, b10=1), b(b1=1, b11=1), b(b1=1, b15=0x80)],
        "smaller low half, larger high half": [b(b7=2), b(b7=1, b8=0xff, b15=0xff), b(b7=2, b8=1)],
        "exact ties": [b(b5=3)] * 5 + [b(b5=4)],
        "all-ones minimum": [],
        "zero rows": [z] * 3 + [b(b15=1)],
    }
    for name, rows in cases.items():
        for trial in range(4):
            a = _planted(rng, 3000 + trial, rows)
            if name == "all-ones minimum":
                a[:] = 0xff
            got_first, got_ties = orc.np_stored_argmin(a)
            want_first, want_ties = _py_stored_argmin(a)
            assert got_first == want_first and got_ties.tolist() == want_ties, name
    for trial in range(20):                                              # random 0/1 bytes: long shared prefixes and ties
        a = rng.integers(0, 2, (1 + 97 * trial, 16), dtype=np.uint8)
        got_first, got_ties = orc.np_stored_argmin(a)
        assert (got_first, got_ties.tolist()) == _py_stored_argmin(a)


def test_stored_argmin_rule_matches_the_oracle_scan(orc):
    """Small N = 2 POSTs; seeds chosen so that both outcomes occur (P(min >= threshold) is about 1/e)."""
    seen = set()
    for seed in range(12):
        node = bytes([seed]) * 32
        c = orc.c_commitment(node, ATX)
        count = 600 + 37 * seed
        labels, found, idx, l32 = orc.c_labels_range(c, 2, 0, count, orc.c_vrf_difficulty(count))
        got = stored_argmin_rule(orc, labels, c, 2, count)
        assert got == ((idx, l32) if found else None), seed
        seen.add(found)
    assert seen == {True, False}
