"""The return code and b200post_last_error() text of every C entry point that takes a provider id or a provider list,
when the provider is what answers: the CPU id (no CPU path: UNSUPPORTED), an id that names no device, and provider
lists with a failing entry in either position.  Every other argument is valid, so these cases pin each entry point's
order of checks and which list entry's text comes back.

The fixture tests/golden/device_entry.json was written by this test's writer mode, in two sections:

    python tests/test_device_entry_host.py --write DIR no_device      (on a machine without a CUDA device)
    python tests/test_device_entry_host.py --write DIR with_device    (on an H100)

CPU tier: `no_device` is compared on a machine without a device.  GPU tier: `with_device` is compared on the H100.
The only device work a case does is a four-label labels_range on device 0 (labels_range_multi with [0, CPU])."""
import ctypes
import importlib
import json
import shutil
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
FIXTURE = ROOT / "tests" / "golden" / "device_entry.json"
POST_FILES = ROOT / "tests" / "golden" / "post_files"
CPU, NONE = 0xFFFFFFFF, 0xFFFFFFFE   # NONE: past the last ordinal on any machine
NODE, ATX = bytes(range(7, 39)), bytes(range(100, 132))
# the POST of tests/golden/post_files (N, LabelsPerUnit, units, K1, K2, labels per file; four files)
N, LPU, UNITS, K1, K2, PER_FILE = 2, 2048, 2, 300, 12, 1024

u32, u64, sz, dbl = ctypes.c_uint32, ctypes.c_uint64, ctypes.c_size_t, ctypes.c_double


def _mod(name):
    if str(ROOT) not in sys.path:
        sys.path.insert(0, str(ROOT))
    return importlib.import_module("go-spacemesh_b200" + name)


def _ids(providers):
    return None if providers is None else (u32 * max(len(providers), 1))(*providers)


def _n(providers):
    return 2 if providers is None else len(providers)   # a NULL list is given with n = 2


def _post_dir(d: Path, case: str, metas_from: str | None = None) -> str:
    """A POST directory: the metadata (and range records) of a golden case over zero-filled postdata files."""
    d.mkdir(parents=True)
    for p in (POST_FILES / case).iterdir():
        shutil.copy(p, d / p.name)
    if metas_from:
        for p in (POST_FILES / metas_from).glob("range_*.rec"):
            shutil.copy(p, d / p.name)
    for f in range(LPU * UNITS // PER_FILE):
        (d / f"postdata_{f}.bin").write_bytes(bytes(16 * PER_FILE))
    return str(d)


def _cases(tmp: Path) -> dict:
    """name -> (return value, last error text), in a fixed order."""
    b2 = _mod("")
    su, pv, vf, k2 = _mod(".setup"), _mod(".prove"), _mod(".verify"), _mod(".k2pow")
    C = ctypes.CDLL(str(b2.LIB_PATH))   # a handle of its own: no argtypes, every argument typed here
    C.b200post_last_error.restype = ctypes.c_char_p
    C.b200post_timer_elapsed_ms.restype = dbl
    C.b200post_last_call_ms.restype = dbl
    C.new_initializer.restype = ctypes.c_void_p

    comm = b2.commitment(NODE, ATX)
    cfg = su.PostConfig(labels_per_unit=LPU, k1=K1, k2=K2, k3=K2, max_num_units=8)
    ccfg = pv._c_cfg(cfg)
    kp = k2._params(1, bytes(8), NODE, b"\x00" * 31 + b"\x01", None)
    skip, _ = vf._verifier_opts("skip")
    no_pow_fn = vf._VerifierOpts()
    no_pow_fn.pow_mode = 1   # CALLBACK without a function: refused, but after the provider
    proofs, metas, vparams = (vf._Proof * 2)(), (vf._Meta * 2)(), vf._Params()
    vchecks = (b2.VrfCheck * 2)(*[b2.vrf_check(NODE, ATX, i, 4, 1024, N) for i in range(2)])
    prove_dir = _post_dir(tmp / "prove", "full_w1")
    search_dir = _post_dir(tmp / "search", "full_w1")
    verify_dir = _post_dir(tmp / "verify", "full_w1")

    def out(n):
        return ctypes.create_string_buffer(max(n, 1))

    def labels_range_multi(ps, count=4):
        return C.b200post_labels_range_multi(_ids(ps), _n(ps), comm, u64(N), u64(0), u64(count), out(16 * count),
                                             None, None, None)

    def k2pow_search_multi(ps):
        return C.b200post_k2pow_search_multi(_ids(ps), _n(ps), ctypes.byref(kp), u64(0), u64(1),
                                             ctypes.byref(u64()), ctypes.byref(u64()), None)

    def k2pow_groups_multi(ps):
        return C.b200post_k2pow_search_groups_multi(_ids(ps), _n(ps), ctypes.byref(kp), u32(1), u64(1), (u64 * 1)(),
                                                    ctypes.byref(u64()), None)

    def k2pow_group_range_multi(ps):
        return C.b200post_k2pow_search_group_range_multi(_ids(ps), _n(ps), ctypes.byref(kp), u32(3), u32(1), u64(1),
                                                         (u64 * 1)(), ctypes.byref(u64()), None)

    def verifier_new_multi(ps, opts=skip):
        h = ctypes.c_void_p()
        rc = C.b200post_verifier_new_multi(_ids(ps), _n(ps), ctypes.byref(opts), ctypes.byref(h))
        assert not h.value, "a verifier was created"
        return rc

    def verify_batch_multi(ps, n=2):
        return C.b200post_verify_batch_multi(_ids(ps), _n(ps), sz(n), proofs, metas, ctypes.byref(vparams), None,
                                             ctypes.byref(skip), (ctypes.c_int * 2)(), (u64 * 2)())

    def vrf_nonces_multi(ps, n=2):
        return C.b200post_verify_vrf_nonces_multi(_ids(ps), _n(ps), sz(n), vchecks, (ctypes.c_int * 2)(),
                                                  (ctypes.c_int * 2)(), out(64))

    def generate_multi(ps):
        opts, _ = pv._opts(None, None, 16, 0, "skip")
        return C.b200post_generate_proof_multi(prove_dir.encode(), bytes(32), ctypes.byref(ccfg), ctypes.byref(opts), _ids(ps),
                                               _n(ps), ctypes.byref(pv._ProofOut()), ctypes.byref(vf._Meta()), None)

    def generate_checked(ps):
        opts, _ = pv._opts(None, None, 16, 0, "skip")
        return C.b200post_generate_proof_checked(prove_dir.encode(), bytes(32), ctypes.byref(ccfg), ctypes.byref(opts), _ids(ps),
                                                 _n(ps), ctypes.byref(pv._ProofOut()), ctypes.byref(vf._Meta()),
                                                 ctypes.byref(pv._ProveCheck()), None)

    def single(p):
        """Every entry point that takes one provider id."""
        def generate():
            opts, _ = pv._opts(p, None, 16, 0, "skip")
            return C.b200post_generate_proof(prove_dir.encode(), bytes(32), ctypes.byref(ccfg), ctypes.byref(opts),
                                             ctypes.byref(pv._ProofOut()), ctypes.byref(vf._Meta()), None)

        def verifier_new(opts=skip):
            h = ctypes.c_void_p()
            rc = C.b200post_verifier_new(u32(p), ctypes.byref(opts), ctypes.byref(h))
            assert not h.value, "a verifier was created"
            return rc

        return {
            "labels_range": lambda: C.b200post_labels_range(u32(p), comm, u64(N), u64(0), u64(4), out(64), None, None, None),
            "labels_range_dev": lambda: C.b200post_labels_range_dev(u32(p), comm, u64(N), u64(0), u64(4), None, None, None, None),
            "labels_gather": lambda: C.b200post_labels_gather(u32(p), sz(2), comm * 2, (u64 * 2)(1, 2), u64(N), out(32)),
            "labels_gather_indexed": lambda: C.b200post_labels_gather_indexed(u32(p), sz(2), sz(1), comm, (u32 * 2)(), (u64 * 2)(1, 2),
                                                                              u64(N), out(32)),
            "verify_vrf_nonce": lambda: C.b200post_verify_vrf_nonce(u32(p), u64(5), NODE, ATX, u32(4), u64(1024), u64(N),
                                                                    ctypes.byref(ctypes.c_int())),
            "vrf_nonce_label": lambda: C.b200post_vrf_nonce_label(u32(p), u64(5), NODE, ATX, u64(N), out(32)),
            "benchmark": lambda: C.b200post_benchmark(u32(p), u64(N), dbl(0.0), ctypes.byref(dbl())),
            "wave_slots": lambda: C.b200post_wave_slots(u32(p), u64(N), ctypes.byref(u64())),
            "romix_time": lambda: C.b200post_romix_time(u32(p), None, None, None, 0),
            "timer_mark": lambda: C.b200post_timer_mark(u32(p), 0),
            "timer_elapsed_ms": lambda: C.b200post_timer_elapsed_ms(u32(p)),
            "last_call_ms": lambda: C.b200post_last_call_ms(u32(p)),
            "vrf_comm_init": lambda: C.b200post_vrf_comm_init(u32(p), 0, 1, bytes(128), ctypes.byref(ctypes.c_void_p())),
            "new_initializer": lambda: C.new_initializer(u32(p), sz(N), comm, None) is not None,
            "poet_pow_find": lambda: C.b200post_poet_pow_find(u32(p), b"pc", sz(2), b"ch", sz(2), NODE, u32(8), u64(0), u64(16),
                                                              ctypes.byref(u64()), ctypes.byref(u64()), None),
            "randomx_prepare": lambda: C.b200post_randomx_prepare(u32(p), None, sz(0)),
            "randomx_hash": lambda: C.b200post_randomx_hash(u32(p), None, sz(0), b"12345678", sz(8), sz(1), out(32)),
            "randomx_dataset_read": lambda: C.b200post_randomx_dataset_read(u32(p), None, sz(0), u64(0), u64(1), out(64)),
            "randomx_last_timing": lambda: C.b200post_randomx_last_timing(u32(p), None, None, None, None),
            "randomx_batch_size": lambda: C.b200post_randomx_batch_size(u32(p), ctypes.byref(u64())),
            "k2pow_hashes": lambda: C.b200post_k2pow_hashes(u32(p), ctypes.byref(kp), u64(0), u64(1), out(32)),
            "k2pow_search": lambda: C.b200post_k2pow_search(u32(p), ctypes.byref(kp), u64(0), u64(1), ctypes.byref(u64()),
                                                            ctypes.byref(u64()), None),
            "k2pow_search_groups": lambda: C.b200post_k2pow_search_groups(u32(p), ctypes.byref(kp), u32(1), u64(1), (u64 * 1)(),
                                                                          ctypes.byref(u64()), None),
            "k2pow_search_group_range": lambda: C.b200post_k2pow_search_group_range(u32(p), ctypes.byref(kp), u32(3), u32(1), u64(1),
                                                                                    (u64 * 1)(), ctypes.byref(u64()), None),
            "k2pow_verify": lambda: C.b200post_k2pow_verify(u32(p), ctypes.byref(kp), u64(0), ctypes.byref(ctypes.c_int())),
            "verifier_new": verifier_new,
            "verifier_new/pow_fn_missing": lambda: verifier_new(no_pow_fn),
            "verify_batch": lambda: C.b200post_verify_batch(u32(p), sz(2), proofs, metas, ctypes.byref(vparams), None,
                                                            ctypes.byref(skip), (ctypes.c_int * 2)(), (u64 * 2)()),
            "verify_batch/pow_fn_missing": lambda: C.b200post_verify_batch(u32(p), sz(2), proofs, metas, ctypes.byref(vparams), None,
                                                                           ctypes.byref(no_pow_fn), (ctypes.c_int * 2)(), (u64 * 2)()),
            "verify_vrf_nonces": lambda: C.b200post_verify_vrf_nonces(u32(p), sz(2), vchecks, (ctypes.c_int * 2)(),
                                                                      (ctypes.c_int * 2)(), out(64)),
            "verify_vrf_nonces/n0": lambda: C.b200post_verify_vrf_nonces(u32(p), sz(0), vchecks, (ctypes.c_int * 2)(),
                                                                         (ctypes.c_int * 2)(), out(64)),
            "prove_scan": lambda: C.b200post_prove_scan(u32(p), out(16 * 64), u64(0), u64(64), bytes(32), u32(16), (u64 * 1)(),
                                                        u32(K1), u32(K2), u64(4096), ctypes.byref(pv._ProofOut())),
            "generate_proof": generate,
        }

    def lists(ps):
        """Every entry point that takes a provider list."""
        return {
            "labels_range_multi": lambda: labels_range_multi(ps),
            "k2pow_search_multi": lambda: k2pow_search_multi(ps),
            "k2pow_search_groups_multi": lambda: k2pow_groups_multi(ps),
            "k2pow_search_group_range_multi": lambda: k2pow_group_range_multi(ps),
            "verifier_new_multi": lambda: verifier_new_multi(ps),
            "verifier_new_multi/pow_fn_missing": lambda: verifier_new_multi(ps, no_pow_fn),
            "verify_batch_multi": lambda: verify_batch_multi(ps),
            "verify_batch_multi/n0": lambda: verify_batch_multi(ps, 0),
            "verify_batch_multi/n1": lambda: verify_batch_multi(ps, 1),
            "verify_vrf_nonces_multi": lambda: vrf_nonces_multi(ps),
            "verify_vrf_nonces_multi/n0": lambda: vrf_nonces_multi(ps, 0),
            "verify_vrf_nonces_multi/n1": lambda: vrf_nonces_multi(ps, 1),
            "generate_proof_multi": lambda: generate_multi(ps),
            "generate_proof_checked": lambda: generate_checked(ps),
        }

    def session(p, kind):
        d = tmp / f"session-{kind}-{p:x}"
        mgr = su.PostSetupManager(cfg)
        opts = su.PostSetupOpts(data_dir=str(d), num_units=UNITS, max_file_size=16 * PER_FILE, provider_id=p, scrypt_n=N,
                                compute_batch_size=1 << 10)
        if kind == "range_record":
            mgr.prepare_files(opts, NODE, ATX, 0, 1)
            mgr.request_range_record()
        else:
            mgr.prepare_initializer(opts, NODE, ATX)
            if kind == "initial_proof":
                mgr.request_initial_proof(nonces=64, pow="skip")
        mgr.start_session()

    def by_id(p):
        """The entry points that take an int64 provider id (in an options struct)."""
        return {
            "verify_pos": lambda: su.verify_pos(verify_dir, fraction=100.0, provider_id=p),
            "search_vrf_nonce": lambda: su.search_vrf_nonce(search_dir, provider_id=p),
            "merge_range_records": lambda: su.merge_range_records(
                _post_dir(tmp / f"merge-{p:x}", "rec_vrf_0_1", metas_from="rec_vrf_2_3"), cfg, provider_id=p),
            "setup_session": lambda: session(p, "plain"),
            "setup_session/initial_proof": lambda: session(p, "initial_proof"),
            "setup_session/range_record": lambda: session(p, "range_record"),
        }

    calls = {}
    for p, tag in ((CPU, "cpu"), (NONE, "none")):
        calls.update({f"{name}[{tag}]": f for name, f in single(p).items()})
        calls.update({f"{name}[{tag}]": f for name, f in by_id(p).items()})
    for ps, tag in ((None, "null"), ([], "n0"), ([NONE], "none"), ([CPU], "cpu"), ([NONE, CPU], "none,cpu"),
                    ([CPU, NONE], "cpu,none")):
        calls.update({f"{name}[{tag}]": f for name, f in lists(ps).items()})
    for ps, tag in (([0, CPU], "0,cpu"), ([CPU, 0], "cpu,0")):
        calls[f"labels_range_multi[{tag}]"] = lambda ps=ps: labels_range_multi(ps)
        calls[f"verify_vrf_nonces_multi/n0[{tag}]"] = lambda ps=ps: vrf_nonces_multi(ps, 0)

    got = {}
    for name, f in calls.items():
        C.b200post_set_option(b"-", u64(0))   # a known text, so a call that sets none shows it
        try:
            r = f()
        except b2.B200PostError as e:
            r = e.code
        got[name] = [r, C.b200post_last_error().decode(errors="replace")]
    return got


def _section():
    return "with_device" if _mod("").providers() else "no_device"


def _compare(b2, tmp_path, section):
    want = json.loads(FIXTURE.read_text())[section]
    got = _cases(tmp_path)
    assert sorted(got) == sorted(want)
    bad = {k: (got[k], want[k]) for k in want if got[k] != want[k]}
    assert not bad, bad


def test_provider_codes_and_texts_without_a_device(b2, tmp_path):
    if b2.providers():
        pytest.skip("a CUDA device is present: the no-device section is compared on machines without one")
    _compare(b2, tmp_path, "no_device")


@pytest.mark.gpu
def test_provider_codes_and_texts_with_a_device(b2, gpu_ready, tmp_path):
    _compare(b2, tmp_path, "with_device")


if __name__ == "__main__":
    if len(sys.argv) != 4 or sys.argv[1] != "--write" or sys.argv[3] not in ("no_device", "with_device"):
        sys.exit("usage: python tests/test_device_entry_host.py --write DIR no_device|with_device")
    if sys.argv[3] != _section():
        sys.exit(f"this machine writes the {_section()} section")
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        cases = _cases(Path(tmp))
    out = Path(sys.argv[2]) / FIXTURE.name   # one section replaced, the other kept
    doc = json.loads(out.read_text()) if out.exists() else {}
    doc[sys.argv[3]] = cases
    out.parent.mkdir(parents=True, exist_ok=True)
    out.write_text(json.dumps(doc, indent=1, sort_keys=True) + "\n")
