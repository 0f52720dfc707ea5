"""GPU tier: one POST initialised in file ranges (prepare_files) on "several machines", merged, and its VRF nonce found
from the stored labels (search_vrf_nonce, K8) or by a full session on the merged directory; chunk seams of the stored
scan; damaged stored labels; cancel/resume and repair of range sessions; the b200postcli round trip."""
import ctypes
import importlib
import os
import shutil
import subprocess
import threading
import time
from pathlib import Path

import pytest

pytestmark = pytest.mark.gpu

ATX = bytes(range(3, 35))
FILES = 4
# scrypt-N -> (labels per file, compute batch): 4 files each
SHAPES = {2: (256, 128), 8192: (64, 64)}


@pytest.fixture(scope="module")
def su(b2, gpu_ready):
    return importlib.import_module("go-spacemesh_b200.setup")


def _num_labels(n):
    return SHAPES[n][0] * FILES


@pytest.fixture(scope="module")
def identities(orc):
    """Per N, an identity whose arg-min lies inside the POST (not at its ends) and one whose nonce comes from the
    past-the-end search, picked by seed with the oracle: {(n, "in" | "past"): (node_id, oracle index, oracle label32)}."""
    out = {}
    for n in SHAPES:
        total = _num_labels(n)
        diff = orc.c_vrf_difficulty(total)
        for seed in range(200):
            node = bytes([seed, n & 0xff, n >> 8]) + bytes(29)
            _, found, idx, l32 = orc.c_labels_range(orc.c_commitment(node, ATX), n, 0, total, diff)
            kind = "in" if found else "past"
            if kind == "in" and not 0 < idx < total - 1:
                continue
            out.setdefault((n, kind), (node, idx, l32))
            if (n, "in") in out and (n, "past") in out:
                break
    assert len(out) == 2 * len(SHAPES)
    return out


def _mgr(su, n):
    per_file, _ = SHAPES[n]
    return su.PostSetupManager(su.PostConfig(labels_per_unit=per_file * FILES // 2))


def _opts(su, d, n, provider=0):
    per_file, batch = SHAPES[n]
    return su.PostSetupOpts(data_dir=str(d), num_units=2, max_file_size=16 * per_file, provider_id=provider, scrypt_n=n,
                            compute_batch_size=batch)


def _run(su, n, d, node, files=None, provider=0):
    mgr = _mgr(su, n)
    if files is None:
        mgr.prepare_initializer(_opts(su, d, n, provider), node, ATX)
    else:
        mgr.prepare_files(_opts(su, d, n, provider), node, ATX, *files)
    mgr.start_session()
    assert mgr.status().state == su.STATE_COMPLETE
    return mgr


def _nonce_fields(su, d):
    md = su.load_metadata(str(d))
    return md["nonce"], md["nonce_value"], md["last_position"]


def _data(d):
    return {p.name: p.read_bytes() for p in sorted(Path(d).glob("postdata_*.bin"))}


@pytest.fixture(scope="module")
def posts(su, identities, tmp_path_factory):
    """Per (N, kind): A = the whole POST in one session; B = files 0-1; C = files 2-3 on PROVIDER_ALL."""
    root = tmp_path_factory.mktemp("vrf")
    out = {}
    for (n, kind), (node, _, _) in identities.items():
        base = root / f"{n}-{kind}"
        _run(su, n, base / "A", node)
        _run(su, n, base / "B", node, (0, 1))
        _run(su, n, base / "C", node, (2, -1), provider=su.PROVIDER_ALL)
        out[(n, kind)] = base
    return out


def _merge(base, dst, meta_from):
    dst.mkdir()
    for part in ("B", "C"):
        for p in (base / part).glob("postdata_*.bin"):
            shutil.copy(p, dst / p.name)
    shutil.copy(base / meta_from / "postdata_metadata.json", dst / "postdata_metadata.json")
    return dst


CASES = [(2, "in"), (2, "past"), (8192, "in"), (8192, "past")]


@pytest.mark.parametrize("n,kind", CASES)
def test_distributed_equals_single(su, b2, identities, posts, tmp_path, n, kind):
    node, o_idx, o_l32 = identities[(n, kind)]
    base, total = posts[(n, kind)], _num_labels(n)
    a = _nonce_fields(su, base / "A")
    if kind == "in":
        assert a[:2] == (o_idx, o_l32) and a[2] == 0
    else:
        assert a[0] >= total and a[2] > a[0]
    for part, names in (("B", ["postdata_0.bin", "postdata_1.bin"]), ("C", ["postdata_2.bin", "postdata_3.bin"])):
        assert sorted(_data(base / part)) == names                     # nothing outside the range
        md = su.load_metadata(str(base / part))
        assert md["vrf_scan_pending"] == 1 and md["nonce"] is None and md["last_position"] == 0
    for meta_from in ("B", "C"):
        d = _merge(base, tmp_path / f"D{meta_from}", meta_from)
        assert _data(d) == _data(base / "A")
        mtimes = {p.name: p.stat().st_mtime_ns for p in d.glob("postdata_*.bin")}
        mgr = _mgr(su, n)
        mgr.prepare_initializer(_opts(su, d, n), node, ATX)
        assert mgr.status().num_labels_written == total
        mgr.start_session()
        assert mgr.status().state == su.STATE_COMPLETE
        assert {p.name: p.stat().st_mtime_ns for p in d.glob("postdata_*.bin")} == mtimes   # no label bytes written
        assert _data(d) == _data(base / "A")
        assert _nonce_fields(su, d) == a and su.load_metadata(str(d))["vrf_scan_pending"] == 0
        r = su.verify_pos(str(d), fraction=100.0)
        assert r.code == b2.OK and r.argmin_checked and r.argmin_ok
    # the same through search_vrf_nonce, with the batch of the init
    d = _merge(base, tmp_path / "S", "C")
    prog = ctypes.c_uint64(0)
    got = su.search_vrf_nonce(str(d), compute_batch_size=SHAPES[n][1], progress=prog)
    assert got == a[:2] and _nonce_fields(su, d) == a and prog.value == total
    assert su.load_metadata(str(d))["vrf_scan_pending"] == 0
    # a full session continuing B's partial data: the marker makes it search the stored labels at the end
    e = tmp_path / "E"
    shutil.copytree(base / "B", e)
    _run(su, n, e, node)
    assert _data(e) == _data(base / "A") and _nonce_fields(su, e) == a
    # repair: one lost file of a finished POST, re-initialised by a range session
    r2 = tmp_path / "R"
    shutil.copytree(base / "A", r2)
    (r2 / "postdata_2.bin").unlink()
    _run(su, n, r2, node, (2, 2))
    assert _data(r2) == _data(base / "A") and _nonce_fields(su, r2) == a
    assert su.load_metadata(str(r2))["vrf_scan_pending"] == 0


def test_chunk_seams(su, identities, posts, tmp_path):
    """m first or last in a chunk, chunks across file boundaries, a prime chunk size, one label per chunk."""
    n = 2
    _, m, l32 = identities[(n, "in")]
    per_file = SHAPES[n][0]
    d = tmp_path / "seams"
    shutil.copytree(posts[(n, "in")] / "A", d)
    meta = (d / "postdata_metadata.json").read_bytes()
    for chunk in sorted({1, m, m + 1, per_file - 1, per_file + 1, 97, 3 * per_file + 5}):
        assert su.search_vrf_nonce(str(d), chunk_labels=chunk) == (m, l32), chunk
        assert (d / "postdata_metadata.json").read_bytes() == meta


def _label(d, per_file, i):
    with open(Path(d) / f"postdata_{i // per_file}.bin", "rb") as f:
        f.seek(i % per_file * 16)
        return f.read(16)


def _put(d, per_file, i, b):
    with open(Path(d) / f"postdata_{i // per_file}.bin", "r+b") as f:
        f.seek(i % per_file * 16)
        f.write(b)


def test_damage_is_reported_and_the_metadata_kept(su, b2, identities, posts, tmp_path):
    n = 2
    _, m, _ = identities[(n, "in")]
    per_file, total = SHAPES[n][0], _num_labels(n)
    cases = [("zero", 700 if m != 700 else 701), ("copy-earlier", m // 2), ("copy-later", (m + total) // 2)]
    for name, j in cases:
        d = tmp_path / name
        shutil.copytree(posts[(n, "in")] / "A", d)
        meta = (d / "postdata_metadata.json").read_bytes()
        _put(d, per_file, j, bytes(16) if name == "zero" else _label(d, per_file, m))
        for chunk in (0, 300):
            with pytest.raises(b2.B200PostError) as e:
                su.search_vrf_nonce(str(d), chunk_labels=chunk)
            assert e.value.code == su.ERR_LABEL_MISMATCH and f"index {j} " in str(e.value), (name, str(e.value))
            assert (d / "postdata_metadata.json").read_bytes() == meta


def test_range_cancel_then_resume(su, b2, tmp_path):
    """Files 5..20 of a 40-file POST: stopped mid-range, resumed to the same bytes; no file outside the range appears."""
    node = bytes(range(100, 132))
    cfg = su.PostConfig(labels_per_unit=1 << 14)
    per_file = 4096
    o = su.PostSetupOpts(data_dir=str(tmp_path / "r"), num_units=10, max_file_size=16 * per_file, provider_id=0, scrypt_n=256,
                         compute_batch_size=1024)
    mgr = su.PostSetupManager(cfg)
    mgr.prepare_files(o, node, ATX, 5, 20)
    cancel, result = ctypes.c_int(0), {}

    def run():
        try:
            mgr.start_session(cancel)
            result["rc"] = 0
        except b2.B200PostError as e:
            result["rc"] = e.code

    t = threading.Thread(target=run)
    t.start()
    deadline = time.time() + 20
    while time.time() < deadline:
        st = mgr.status()
        if st.state == su.STATE_IN_PROGRESS and st.num_labels_written > 0:
            break
        time.sleep(0.001)
    cancel.value = 1
    t.join()
    expect = [f"postdata_{f}.bin" for f in range(5, 21)]
    st = mgr.status()
    if result["rc"] == 0:
        pytest.skip("session finished before the cancel landed")
    assert result["rc"] == b2.ERR_CANCELLED and st.state == su.STATE_STOPPED and 0 < st.num_labels_written < 16 * per_file
    assert set(_data(o.data_dir)) <= set(expect)
    mgr2 = su.PostSetupManager(cfg)
    mgr2.prepare_files(o, node, ATX, 5, 20)
    assert mgr2.status().num_labels_written == st.num_labels_written
    mgr2.start_session()
    assert mgr2.status().state == su.STATE_COMPLETE and mgr2.status().num_labels_written == 16 * per_file
    got = _data(o.data_dir)
    assert sorted(got) == sorted(expect)
    labels, _ = b2.labels_range(b2.commitment(node, ATX), 256, 5 * per_file, 16 * per_file)
    assert b"".join(got[f"postdata_{f}.bin"] for f in range(5, 21)) == labels.tobytes()
    assert su.load_metadata(o.data_dir)["vrf_scan_pending"] == 1


def test_cli_round_trip(b2, su, identities, posts, tmp_path):
    cli = Path(b2.LIB_PATH).parent / "b200postcli"
    if not cli.exists():
        pytest.skip("b200postcli not built")
    n = 8192
    per_file, batch = SHAPES[n]
    node = identities[(n, "past")][0]
    a = _nonce_fields(su, posts[(n, "past")] / "A")
    common = ["-id", node.hex(), "-commitmentAtxId", ATX.hex(), "-numUnits", "2", "-labelsPerUnit", str(per_file * FILES // 2),
              "-maxFileSize", str(16 * per_file), "-scryptN", str(n), "-computeBatchSize", str(batch)]
    r = subprocess.run([str(cli), "-printNumFiles"] + common, capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.strip() == "4"
    for part, lo, hi in (("B", "0", "1"), ("C", "2", "3")):
        r = subprocess.run([str(cli)] + common + ["-datadir", str(tmp_path / part), "-fromFile", lo, "-toFile", hi],
                           capture_output=True, text=True, timeout=300)
        assert r.returncode == 0 and "-searchForNonce" in r.stdout, r.stdout + r.stderr
    d = _merge(tmp_path, tmp_path / "D", "B")
    r = subprocess.run([str(cli), "-searchForNonce", "-datadir", str(d), "-computeBatchSize", str(batch)],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and f"VRF nonce {a[0]}" in r.stdout, r.stdout + r.stderr
    assert _nonce_fields(su, d) == a and _data(d) == _data(posts[(n, "past")] / "A")
    _put(d, per_file, 77, bytes(16))
    r = subprocess.run([str(cli), "-searchForNonce", "-datadir", str(d)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 1 and "index 77 " in r.stderr, r.stdout + r.stderr
    os.remove(d / "postdata_3.bin")
    r = subprocess.run([str(cli), "-searchForNonce", "-datadir", str(d)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 1 and "incomplete" in r.stderr
