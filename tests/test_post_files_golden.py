"""The bytes of every file a POST data directory holds besides the labels, pinned by committed fixtures.

postdata_metadata.json, initial_post.json, initial_post.scan and range_<from>_<to>.rec are read by other programs and
by later versions of this library, so their bytes are an interface.  The fixtures under tests/golden/post_files/ were
written by this test's writer mode:

    python tests/test_post_files_golden.py --write DIR     (on an H100: the session cases need a device)

CPU tier: the metadata of a prepared session is written again and compared byte for byte; every fixture loads through
the public API (load_metadata, load_initial_proof, and a load + save of the metadata by prepare_initializer gives the
same bytes); the golden records, with their metadata and zero-filled postdata files, pass every host check of
merge_range_records.  GPU tier: the sessions and merges are run again and every file is compared byte for byte."""
import ctypes
import importlib
import shutil
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
FIXTURES = ROOT / "tests" / "golden" / "post_files"
NODE, ATX = bytes(range(7, 39)), bytes(range(100, 132))
# the "N2" case of test_gpu_initial_proof: (N, LabelsPerUnit, units, K1, K2, nonces, batch, labels per file); four files
N, LPU, UNITS, K1, K2, NONCES, BATCH, PER_FILE = 2, 2048, 2, 300, 12, 64, 1 << 10, 1024
FILES = LPU * UNITS // PER_FILE
KEY = b"golden-cache-key"
META = "postdata_metadata.json"

# case -> the files it pins.  CPU cases need no device; the others are sessions and merges.
CPU_CASES = {"prepared": [META], "range_prepared": [META]}
GPU_CASES = {
    "full_w1": [META, "initial_post.json", "initial_post.scan"],
    "full_w3": [META, "initial_post.json", "initial_post.scan"],
    "rec_proof_0_1": [META, "range_0_1.rec"],
    "rec_proof_2_3": [META, "range_2_3.rec"],
    "rec_vrf_0_1": [META, "range_0_1.rec"],
    "rec_vrf_2_3": [META, "range_2_3.rec"],
    "merged_proof": [META, "initial_post.json"],
    "merged_vrf": [META],
}
MERGES = {"merged_proof": ("rec_proof_0_1", "rec_proof_2_3"), "merged_vrf": ("rec_vrf_0_1", "rec_vrf_2_3")}


def _su():
    if str(ROOT) not in sys.path:
        sys.path.insert(0, str(ROOT))
    return importlib.import_module("go-spacemesh_b200.setup")


def _cfg(su):
    return su.PostConfig(labels_per_unit=LPU, k1=K1, k2=K2, k3=K2, max_num_units=8)


def _opts(su, d):
    return su.PostSetupOpts(data_dir=str(d), num_units=UNITS, max_file_size=16 * PER_FILE, provider_id=0, scrypt_n=N,
                            compute_batch_size=BATCH)


def _proof_request(windows):
    return dict(nonces=NONCES, pow="skip", pow_cache_key=KEY, windows_per_pass=windows)


def _run(su, case, d):
    """Writes `case` into the empty directory d."""
    mgr = su.PostSetupManager(_cfg(su))
    if case == "prepared":
        mgr.prepare_initializer(_opts(su, d), NODE, ATX)
    elif case == "range_prepared":
        mgr.prepare_files(_opts(su, d), NODE, ATX, 0, 1)
    elif case.startswith("full_w"):
        mgr.prepare_initializer(_opts(su, d), NODE, ATX)
        mgr.request_initial_proof(**_proof_request(int(case[-1])))
        mgr.start_session()
        assert mgr.status().state == su.STATE_COMPLETE
    elif case.startswith("rec_"):
        kind, a, b = case.split("_")[1:]
        mgr.prepare_files(_opts(su, d), NODE, ATX, int(a), int(b))
        if kind == "proof":
            mgr.request_range_record(initial_proof=True, **_proof_request(1))
        else:
            mgr.request_range_record()
        mgr.start_session()
        assert mgr.status().state == su.STATE_COMPLETE
    else:
        parts = MERGES[case]
        d.mkdir(parents=True, exist_ok=True)
        for part in parts:
            src = d.parent / (case + "-" + part)
            _run(su, part, src)
            for p in list(src.glob("postdata_*.bin")) + list(src.glob("range_*.rec")):
                shutil.copy2(p, d / p.name)
        shutil.copy(d.parent / (case + "-" + parts[0]) / META, d / META)
        r = su.merge_range_records(str(d), _cfg(su))
        assert r.ranges == 2 and (r.proof is not None) == (case == "merged_proof"), r


def _check_case(su, case, d):
    for name in (CPU_CASES | GPU_CASES)[case]:
        assert (d / name).read_bytes() == (FIXTURES / case / name).read_bytes(), (case, name)


# ---------------------------------------------------------------- CPU tier

@pytest.mark.parametrize("case", sorted(CPU_CASES))
def test_prepared_metadata_bytes(b2, tmp_path, case):
    su = _su()
    _run(su, case, tmp_path / case)
    _check_case(su, case, tmp_path / case)


@pytest.mark.parametrize("case", sorted(CPU_CASES | GPU_CASES))
def test_metadata_loads_and_saves_unchanged(b2, tmp_path, case):
    """load_metadata reads every fixture, and prepare_initializer's load + save of it writes the same bytes."""
    su = _su()
    d = tmp_path / case
    d.mkdir()
    shutil.copy(FIXTURES / case / META, d / META)
    md = su.load_metadata(str(d))
    assert (md["node_id"], md["commitment_atx_id"], md["labels_per_unit"], md["num_units"]) == (NODE, ATX, LPU, UNITS)
    assert (md["max_file_size"], md["scrypt_n"]) == (16 * PER_FILE, N)
    has_nonce = case.startswith(("full_", "merged_"))
    assert (md["nonce"] is not None) == has_nonce, md
    assert md["vrf_scan_pending"] == (not has_nonce and case != "prepared"), md
    su.PostSetupManager(_cfg(su)).prepare_initializer(_opts(su, d), NODE, ATX)
    assert (d / META).read_bytes() == (FIXTURES / case / META).read_bytes()


@pytest.mark.parametrize("case", ["full_w1", "full_w3", "merged_proof"])
def test_initial_proof_loads(b2, tmp_path, case):
    su = _su()
    d = tmp_path / case
    shutil.copytree(FIXTURES / case, d)
    proof, meta, scanned = su.load_initial_proof(str(d), _cfg(su), NONCES)
    assert (meta.node_id, meta.commitment_atx_id, meta.challenge) == (NODE, ATX, bytes(32)) and scanned == LPU * UNITS
    windows = 3 if case == "full_w3" else 1
    assert proof.nonce < NONCES * windows and proof.pow == 0
    # another nonce count is another proof request
    e = pytest.raises(b2.B200PostError, su.load_initial_proof, str(d), _cfg(su), NONCES * 2)
    assert e.value.code == su.ERR_IO and "no initial proof" in str(e.value)


@pytest.mark.parametrize("case", sorted(MERGES))
def test_golden_records_pass_the_merge_host_checks(b2, tmp_path, case):
    """The records and metadata of two range sessions, over zero-filled postdata files: every host check passes, so the
    merge stops at the device (and writes nothing)."""
    if b2.providers():
        pytest.skip("a CUDA device is present: NO_DEVICE cannot be observed")
    su = _su()
    d = tmp_path / case
    d.mkdir()
    parts = MERGES[case]
    for part in parts:
        for name in GPU_CASES[part][1:]:
            shutil.copy(FIXTURES / part / name, d / name)
    shutil.copy(FIXTURES / parts[0] / META, d / META)
    for f in range(FILES):
        (d / f"postdata_{f}.bin").write_bytes(bytes(16 * PER_FILE))
    before = {p.name: p.read_bytes() for p in d.iterdir()}
    e = pytest.raises(b2.B200PostError, su.merge_range_records, str(d), _cfg(su))
    assert e.value.code == b2.ERR_NO_DEVICE, str(e.value)
    assert {p.name: p.read_bytes() for p in d.iterdir()} == before


# ---------------------------------------------------------------- GPU tier

@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(GPU_CASES))
def test_session_files_bytes(b2, gpu_ready, tmp_path, case):
    su = _su()
    _run(su, case, tmp_path / case)
    _check_case(su, case, tmp_path / case)


def _write(out: Path):
    su = _su()
    work = out / "_work"
    for case, names in (CPU_CASES | GPU_CASES).items():
        _run(su, case, work / case)
        (out / case).mkdir(parents=True, exist_ok=True)
        for name in names:
            shutil.copy(work / case / name, out / case / name)
    shutil.rmtree(work)


if __name__ == "__main__":
    if len(sys.argv) != 3 or sys.argv[1] != "--write":
        sys.exit("usage: python tests/test_post_files_golden.py --write DIR")
    _write(Path(sys.argv[2]))
