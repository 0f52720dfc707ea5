"""GPU tier: full POST setup sessions through the C ABI, mirroring activation/post_test.go
(TestPostSetupManager :24-73, _InitialStatus :180-205, _Stop :207-235, _Stop_WhileInProgress :237-281,
_StartSession_WithoutProviderAfterInit_OK :118-139) with byte-level checks against the oracle added."""
import ctypes
import importlib
import threading
import time
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NODE, ATX = bytes(range(100, 132)), bytes(range(7, 39))


@pytest.fixture()
def su(b2, gpu_ready):
    return importlib.import_module("go-spacemesh_b200.setup")


def _opts(su, tmp_path, **kw):
    # newTestPostManager (post_test.go:351-381): DefaultPostConfig (2 x 512 labels), Scrypt.N = 2
    d = dict(data_dir=str(tmp_path / "post"), num_units=2, max_file_size=4096, provider_id=0, scrypt_n=2,
             compute_batch_size=128, self_check_every=4)
    d.update(kw)
    return su.PostSetupOpts(**d)


def _read_all(data_dir: str) -> bytes:
    files = sorted(Path(data_dir).glob("postdata_*.bin"), key=lambda p: int(p.stem.split("_")[1]))
    return b"".join(p.read_bytes() for p in files)


def test_full_session_matches_oracle(su, orc, tmp_path):
    """BASELINE.json configs[0] through the setup manager: 1024 labels, N = 2, files of 256 labels."""
    mgr = su.PostSetupManager()
    o = _opts(su, tmp_path)
    mgr.prepare_initializer(o, NODE, ATX)
    mgr.start_session()
    st = mgr.status()
    assert st.state == su.STATE_COMPLETE and st.num_labels_written == 1024
    c = orc.py_commitment(NODE, ATX)
    exp, found, idx, l32 = orc.c_labels_range(c, 2, 0, 1024, orc.py_vrf_difficulty(1024))
    assert _read_all(o.data_dir) == exp.tobytes()
    assert len(list(Path(o.data_dir).glob("postdata_*.bin"))) == 4            # 1024 labels / (4096 B / 16 B)
    md = su.load_metadata(o.data_dir)
    assert md["nonce"] is not None
    if found:
        assert (md["nonce"], md["nonce_value"]) == (idx, l32)
    else:                                                                    # searched past the last label
        assert md["nonce"] >= 1024 and md["nonce_value"] < orc.py_vrf_difficulty(1024)
        assert orc.c_label32(c, md["nonce"], 2) == md["nonce_value"]

    # "Create data (same opts)" / Reset / again (post_test.go:60-72)
    mgr.prepare_initializer(o, NODE, ATX)
    mgr.start_session()
    assert mgr.status().state == su.STATE_COMPLETE
    mgr.reset()
    assert mgr.status().state == su.STATE_NOT_STARTED and not list(Path(o.data_dir).glob("postdata_*"))
    mgr.prepare_initializer(o, NODE, ATX)
    mgr.start_session()
    assert mgr.status().state == su.STATE_COMPLETE and _read_all(o.data_dir) == exp.tobytes()


def test_complete_data_needs_no_provider(su, tmp_path):
    """post_test.go:118-139."""
    mgr = su.PostSetupManager()
    o = _opts(su, tmp_path)
    mgr.prepare_initializer(o, NODE, ATX)
    mgr.start_session()
    o2 = _opts(su, tmp_path, provider_id=None)
    mgr.prepare_initializer(o2, NODE, ATX)
    mgr.start_session()
    assert mgr.status().state == su.STATE_COMPLETE


def test_status_is_monotone_while_in_progress(su, b2, tmp_path):
    """post_test.go:24-58: a watcher sees NumLabelsWritten grow and only Prepared / InProgress states."""
    mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=1 << 15))
    o = _opts(su, tmp_path, num_units=4, scrypt_n=64, compute_batch_size=2048, max_file_size=1 << 19)
    seen, bad = [], []
    stop = threading.Event()

    def watch():
        last = 0
        while not stop.is_set():
            st = mgr.status()
            if st.num_labels_written < last:
                bad.append((last, st.num_labels_written))
            last = st.num_labels_written
            seen.append((st.state, st.num_labels_written))
            time.sleep(0.002)

    t = threading.Thread(target=watch)
    mgr.prepare_initializer(o, NODE, ATX)
    t.start()
    mgr.start_session()
    stop.set(); t.join()
    assert not bad
    assert mgr.status() == su.PostSetupStatus(su.STATE_COMPLETE, 4 << 15)
    assert {s for s, _ in seen} <= {su.STATE_PREPARED, su.STATE_IN_PROGRESS, su.STATE_COMPLETE}
    assert len({n for _, n in seen}) > 3, "the watcher never saw intermediate progress"


def test_stop_while_in_progress_then_resume(su, b2, orc, tmp_path):
    """post_test.go:237-281: cancel -> Stopped, Prepare+Start continues, final data identical to one run."""
    cfg = su.PostConfig(labels_per_unit=1 << 14)
    mgr = su.PostSetupManager(cfg)
    o = _opts(su, tmp_path, num_units=cfg.max_num_units, scrypt_n=256, compute_batch_size=1024, max_file_size=4096 * 16)
    mgr.prepare_initializer(o, NODE, ATX)
    cancel = ctypes.c_int(0)
    result = {}

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
    total = cfg.max_num_units * cfg.labels_per_unit
    st = mgr.status()
    if result["rc"] == 0:
        pytest.skip("session finished before the cancel landed")
    assert result["rc"] == b2.ERR_CANCELLED and st.state == su.STATE_STOPPED and 0 < st.num_labels_written < total
    partial = _read_all(o.data_dir)
    assert len(partial) == 16 * st.num_labels_written

    mgr.prepare_initializer(o, NODE, ATX)                                   # continue to create data
    assert mgr.status().num_labels_written == st.num_labels_written          # resume point = NumLabelsWritten
    mgr.start_session()
    st = mgr.status()
    assert st.state == su.STATE_COMPLETE and st.num_labels_written == total
    data = _read_all(o.data_dir)
    assert data[: len(partial)] == partial
    c = orc.py_commitment(NODE, ATX)
    sample = np.unique(np.random.default_rng(9).integers(0, total, 400))
    comms = np.tile(np.frombuffer(c, dtype=np.uint8), (len(sample), 1))
    exp = orc.c_labels_gather(comms, sample.astype(np.uint64), 256)
    got = np.frombuffer(data, dtype=np.uint8).reshape(-1, 16)[sample]
    assert (got == exp).all()


def test_nonce_search_continues_past_the_last_label(su, orc, tmp_path):
    """A space so small that usually no label is below 2^256/numLabels: the session still ends with a nonce."""
    mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=8, max_num_units=4))
    for k, node in enumerate((b"\x01" * 32, b"\x02" * 32, b"\x03" * 32)):
        o = _opts(su, tmp_path / str(k), num_units=1, compute_batch_size=8, max_file_size=64)
        mgr.prepare_initializer(o, node, ATX)
        mgr.start_session()
        md = su.load_metadata(o.data_dir)
        c = orc.py_commitment(node, ATX)
        assert md["nonce"] is not None and md["nonce_value"] < orc.py_vrf_difficulty(8)
        assert orc.c_label32(c, md["nonce"], 2) == md["nonce_value"]
        # it is the first qualifying label in scan order, as the oracle sees it
        _, found, idx, _ = orc.c_labels_range(c, 2, 0, max(md["nonce"] + 1, 8), orc.py_vrf_difficulty(8), threads=1)
        assert found and (idx == md["nonce"] or md["nonce"] < 8)
        assert len(_read_all(o.data_dir)) == 8 * 16


def test_all_providers_extension(su, orc, tmp_path):
    mgr = su.PostSetupManager()
    o = _opts(su, tmp_path, provider_id=su.PROVIDER_ALL)
    mgr.prepare_initializer(o, NODE, ATX)
    mgr.start_session()
    c = orc.py_commitment(NODE, ATX)
    assert _read_all(o.data_dir) == orc.c_labels_range(c, 2, 0, 1024)[0].tobytes()


def test_postcli_compatible_cli(b2, orc, tmp_path):
    """systest/cluster/nodes.go:990-999 flag set, with a GPU provider instead of the CPU one."""
    import subprocess
    cli = Path(b2.LIB_PATH).parent / "b200postcli"
    if not cli.exists():
        pytest.skip("b200postcli not built")
    d = tmp_path / "data"
    args = [str(cli), "-id", NODE.hex(), "-commitmentAtxId", ATX.hex(), "-datadir", str(d), "-numUnits", "3",
            "-labelsPerUnit", "256", "-scryptN", "2", "-provider", "0", "-yes", "-maxFileSize", "8192"]
    r = subprocess.run(args, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    c = orc.py_commitment(NODE, ATX)
    assert _read_all(str(d)) == orc.c_labels_range(c, 2, 0, 768)[0].tobytes()
    assert "VRF nonce" in r.stdout
    r = subprocess.run(args[:-5] + ["-provider", "4294967295", "-yes"], capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and "CPU" in r.stderr


def test_fault_injection_trips_the_cpu_reference_check(su, b2, tmp_path):
    """ErrReferenceLabelMismatch contract (activation/post.go:299-312): a batch whose bytes differ from the label the HOST
    computes ends the session in state Error with B200POST_ERR_LABEL_MISMATCH, the call returns (no crash, no hang), and
    nothing of the bad batch is on disk.  The checker is independent of the device (b200post_reference_label)."""
    mgr = su.PostSetupManager()
    o = _opts(su, tmp_path, self_check_every=1)
    mgr.prepare_initializer(o, NODE, ATX)
    try:
        b2.set_option("debug_corrupt_check_all", 1)
        b2.set_option("debug_corrupt_next_batch", 1)
        with pytest.raises(b2.B200PostError) as e:
            mgr.start_session()
        assert e.value.code == su.ERR_LABEL_MISMATCH and "reference label mismatch" in str(e.value)
        st = mgr.status()
        assert st.state == su.STATE_ERROR and st.num_labels_written == 0
        assert "b200post_setup_label_mismatch_total 1" in b2.metrics_text() or "label_mismatch" in b2.metrics_text()
        # the one-shot fault is gone: the session can be resumed and completes with correct data
        mgr.prepare_initializer(o, NODE, ATX)
        mgr.start_session()
        assert mgr.status().state == su.STATE_COMPLETE
    finally:
        b2.set_option("debug_corrupt_check_all", 0)
        b2.set_option("debug_corrupt_next_batch", 0)
