"""GPU tier: gathers that ride a running range job's ROMix layers (DeviceEngine riders).

While a labels_range call runs, gathers from several threads (labels_gather, labels_gather_indexed, the verifier's wide
gathers of VRF-nonce checks, verify_pos's compare gathers) at the same N join its layers instead of waiting for it:

* the range labels and its VRF candidate are byte-identical to a solo call;
* every gather equals a solo gather and the oracle;
* b200post_engine_rider_calls_total grows; a gather at another N does not ride and is still right;
* cancelling the range job with riders in flight leaves every rider right;
* a setup session with a concurrent verifier gives the same files, metadata and verdicts as the two run apart.

Small N with a capped scratch gives range calls of hundreds of layers; one case runs at N = 8192 with the full layer."""
import ctypes
import importlib
import re
import threading
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

COMMIT = bytes(range(40, 72))


def _counter(b2, name):
    m = re.search(rf"^{name} (\d+)$", b2.metrics_text(), re.M)
    assert m, name
    return int(m.group(1))


@pytest.fixture()
def small_layers(b2, gpu_ready):
    """Scratch for 2048 two-pad slots at N: a phased layer of 4096 labels, a pipelined one of 2048."""
    keep = {k: b2.get_option(k) for k in ("max_scratch_mib", "romix_variant")}

    def cap(n):
        b2.set_option("max_scratch_mib", 2048 * 2 * 128 * n >> 20)
    yield cap
    for k, v in keep.items():
        b2.set_option(k, v)


def _gather_inputs(rng, count, n_commit=3):
    comms = rng.integers(0, 256, (n_commit, 32), dtype=np.uint8)
    row = rng.integers(0, n_commit, count).astype(np.uint32)
    idx = rng.integers(0, 2**40, count, dtype=np.uint64)
    return comms, row, idx


class Gathers:
    """Threads that submit gathers (plain and indexed, several sizes) at scrypt-N `n` until stopped."""

    def __init__(self, b2, n, threads=3, sizes=(1, 37, 700, 5000), seed=0, pause=0.002):
        self.b2, self.n, self.pause, self.results, self.errors = b2, n, pause, [], []
        self.stop = threading.Event()
        self.th = [threading.Thread(target=self._run, args=(seed + t, sizes)) for t in range(threads)]

    def _run(self, seed, sizes):
        rng = np.random.default_rng(seed)
        k = 0
        try:
            while not self.stop.is_set():
                size = sizes[k % len(sizes)]
                comms, row, idx = _gather_inputs(rng, size)
                if k % 2:
                    got = self.b2.labels_gather_indexed(comms, row, idx, self.n)
                else:
                    got = self.b2.labels_gather(comms[row], idx, self.n)
                self.results.append((comms[row], idx, got))
                k += 1
                self.stop.wait(self.pause)
        except Exception as e:  # noqa: BLE001
            self.errors.append(e)

    def __enter__(self):
        for t in self.th:
            t.start()
        return self

    def __exit__(self, *exc):
        self.stop.set()
        for t in self.th:
            t.join()

    def check(self, orc, oracle_items=64):
        assert not self.errors, self.errors
        assert self.results
        for comms, idx, got in self.results:
            assert (got == self.b2.labels_gather(comms, idx, self.n)).all()
        # the oracle on a sample of each call's items
        for comms, idx, got in self.results[:: max(1, len(self.results) // 8)]:
            pick = np.arange(min(len(idx), oracle_items))
            assert (got[pick] == orc.c_labels_gather(comms[pick], idx[pick], self.n)).all()


@pytest.mark.parametrize("variant", [5, 4], ids=["phased", "pipelined"])
@pytest.mark.parametrize("n", [64, 1024])
def test_gathers_ride_a_range_call(b2, orc, small_layers, variant, n):
    b2.set_option("romix_variant", variant)
    small_layers(n)
    count = (1 << 20) if n == 64 else (1 << 18) + 1234
    start = 2**33 - 77
    diff = b2.vrf_difficulty(count)
    solo, solo_vrf = b2.labels_range(COMMIT, n, start, count, vrf_difficulty_=diff)
    r0 = _counter(b2, "b200post_engine_rider_calls_total")
    l0 = _counter(b2, "b200post_engine_rider_labels_total")
    runs = []
    with Gathers(b2, n) as g:
        for _ in range(3):
            runs.append(b2.labels_range(COMMIT, n, start, count, vrf_difficulty_=diff))
    for got, vrf in runs:
        assert (got == solo).all() and vrf == solo_vrf
    g.check(orc)
    assert _counter(b2, "b200post_engine_rider_calls_total") > r0
    assert _counter(b2, "b200post_engine_rider_labels_total") > l0
    # and the range itself against the oracle on its first and last labels
    exp, *_ = orc.c_labels_range(COMMIT, n, start, 64)
    assert (solo[:64] == exp).all()
    exp, *_ = orc.c_labels_range(COMMIT, n, start + count - 64, 64)
    assert (solo[-64:] == exp).all()


def test_vrf_checks_ride_through_the_verifier(b2, orc, small_layers):
    """Wide gathers (K3w): VRF-nonce checks, batched and through a verifier handle, while a range call runs."""
    vf = importlib.import_module("go-spacemesh_b200.verify")
    n = 1024
    small_layers(n)
    rng = np.random.default_rng(5)
    checks = []
    for i in range(40):
        node, atx = bytes(rng.integers(0, 256, 32, dtype=np.uint8)), bytes(rng.integers(0, 256, 32, dtype=np.uint8))
        checks.append((node, atx, int(rng.integers(0, 2**34)), 4, 2**30, n))
    solo = b2.verify_vrf_nonces(checks)
    v = vf.PostVerifier(pow="skip")
    got, errors = [], []
    stop = threading.Event()

    def submit():
        try:
            while not stop.is_set():
                got.append(("batch", b2.verify_vrf_nonces(checks)))
                got.append(("handle", [v.verify_vrf_nonce(*c[:5], n) for c in checks[:3]]))
        except Exception as e:  # noqa: BLE001
            errors.append(e)
    r0 = _counter(b2, "b200post_engine_rider_calls_total")
    th = [threading.Thread(target=submit) for _ in range(2)]
    try:
        for t in th:
            t.start()
        for _ in range(2):
            b2.labels_range(COMMIT, n, 0, 1 << 19, discard=True)
    finally:
        stop.set()
        for t in th:
            t.join()
        v.close()
    assert not errors, errors
    assert _counter(b2, "b200post_engine_rider_calls_total") > r0
    for kind, res in got:
        if kind == "batch":
            assert res == solo
        else:
            assert res == [(ok, label) for _, ok, label in solo[:3]]
    for (node, atx, nonce, *_), (_, _, label) in zip(checks[:8], solo):
        assert orc.c_label32(b2.commitment(node, atx), nonce, n) == label


def test_gather_at_another_n_does_not_ride(b2, orc, small_layers):
    small_layers(1024)
    r0 = _counter(b2, "b200post_engine_rider_calls_total")
    with Gathers(b2, 64, threads=2, sizes=(37, 300)) as g:
        for _ in range(2):
            b2.labels_range(COMMIT, 1024, 0, 1 << 18, discard=True)
    g.check(orc)
    assert _counter(b2, "b200post_engine_rider_calls_total") == r0


@pytest.mark.parametrize("variant", [5, 4], ids=["phased", "pipelined"])
def test_cancel_with_riders_in_flight(b2, orc, small_layers, variant):
    b2.set_option("romix_variant", variant)
    n = 1024
    small_layers(n)
    cancel = ctypes.c_int(0)
    outcome = []
    r0 = _counter(b2, "b200post_engine_rider_calls_total")

    def host():
        try:
            b2.labels_range(COMMIT, n, 0, 1 << 22, discard=True, cancel=cancel)
            outcome.append(b2.OK)
        except b2.B200PostError as e:
            outcome.append(e.code)
    # the range job starts first; paced gathers leave it the engine between their own calls
    t = threading.Thread(target=host)
    t.start()
    with Gathers(b2, n, threads=3, sizes=(3000, 37, 9000), pause=0.005) as g:
        # cancel once some call has ridden, so that riders are queued and in layers when the job stops
        for _ in range(3000):
            if _counter(b2, "b200post_engine_rider_calls_total") > r0:
                break
            threading.Event().wait(0.002)
        cancel.value = 1
        t.join()
    assert outcome == [b2.ERR_CANCELLED]
    assert _counter(b2, "b200post_engine_rider_calls_total") > r0
    g.check(orc)


def test_rider_at_full_layer_n8192(b2, orc, gpu_ready):
    """N = 8192 with the default layer: a 2^20-label range call and 37-label gathers from two threads."""
    n, count = 8192, 1 << 20
    solo, solo_vrf = b2.labels_range(COMMIT, n, 12345, count, vrf_difficulty_=b2.vrf_difficulty(count))
    r0 = _counter(b2, "b200post_engine_rider_calls_total")
    with Gathers(b2, n, threads=2, sizes=(37, 1)) as g:
        got, vrf = b2.labels_range(COMMIT, n, 12345, count, vrf_difficulty_=b2.vrf_difficulty(count))
    assert (got == solo).all() and vrf == solo_vrf
    assert _counter(b2, "b200post_engine_rider_calls_total") > r0
    g.check(orc, oracle_items=4)


def test_compare_gathers_ride(b2, small_layers, tmp_path):
    """verify_pos's compare gathers (K3c) over stored data with one damaged label, while a range call runs."""
    su = importlib.import_module("go-spacemesh_b200.setup")
    n = 1024
    small_layers(n)
    opts = su.PostSetupOpts(data_dir=str(tmp_path / "post"), num_units=2, max_file_size=1 << 18, provider_id=0, scrypt_n=n,
                            compute_batch_size=1 << 14)
    mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=1 << 15))
    mgr.prepare_initializer(opts, bytes(range(32)), bytes(range(1, 33)))
    mgr.start_session()
    f = Path(opts.data_dir) / "postdata_1.bin"
    raw = bytearray(f.read_bytes())
    for k in range(64):
        raw[16 * (77 + 97 * k) + 3] ^= 0x40
    f.write_bytes(bytes(raw))
    solo = su.verify_pos(opts.data_dir, fraction=50, seed=7)
    assert solo.mismatches > 0
    results, errors = [], []
    stop = threading.Event()

    def check():
        try:
            while not stop.is_set():
                results.append(su.verify_pos(opts.data_dir, fraction=50, seed=7))
        except Exception as e:  # noqa: BLE001
            errors.append(e)
    r0 = _counter(b2, "b200post_engine_rider_calls_total")
    th = [threading.Thread(target=check) for _ in range(2)]
    for t in th:
        t.start()
    try:
        for _ in range(3):
            b2.labels_range(COMMIT, n, 0, 1 << 19, discard=True)
    finally:
        stop.set()
        for t in th:
            t.join()
    assert not errors, errors
    assert results and all(vars(r) == vars(solo) for r in results)
    assert _counter(b2, "b200post_engine_rider_calls_total") > r0


def test_setup_session_with_concurrent_verifier(b2, small_layers, tmp_path):
    su = importlib.import_module("go-spacemesh_b200.setup")
    vf = importlib.import_module("go-spacemesh_b200.verify")
    n = 1024
    small_layers(n)
    cfg = su.PostConfig(labels_per_unit=1 << 17)
    node, atx = bytes(range(9, 41)), bytes(range(3, 35))

    def session(d):
        o = su.PostSetupOpts(data_dir=str(d), num_units=2, max_file_size=1 << 21, provider_id=0, scrypt_n=n,
                             compute_batch_size=1 << 16)
        mgr = su.PostSetupManager(cfg)
        mgr.prepare_initializer(o, node, atx)
        mgr.start_session()
        files = {p.name: p.read_bytes() for p in sorted(Path(d).glob("postdata_*.bin"))}
        return files, su.load_metadata(str(d))

    rng = np.random.default_rng(11)
    bits = vf.bits_per_index(2**32)
    params = vf.VerifyParams(k1=2**31, k2=37, scrypt_n=n)
    proofs, metas = [], []
    for _ in range(64):
        a, b, ch = (bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(3))
        proofs.append(vf.Proof(int(rng.integers(0, 64)), vf.pack_indices([int(x) for x in rng.integers(0, 2**32, 37)], bits), 0))
        metas.append(vf.ProofMetadata(a, b, ch, 1, 2**32))
    v = vf.PostVerifier(pow="skip")

    def verdicts():
        out = []
        for p, m in zip(proofs, metas):
            try:
                v.verify(p, m, params)
                out.append(None)
            except vf.ErrInvalidIndex as e:
                out.append(e.index)
        return out
    try:
        apart_files, apart_md = session(tmp_path / "apart")
        apart_verdicts = verdicts()
        r0 = _counter(b2, "b200post_engine_rider_calls_total")
        together = []
        stop = threading.Event()

        def verify_loop():
            while not stop.is_set():
                together.append(verdicts())
        t = threading.Thread(target=verify_loop)
        t.start()
        try:
            files, md = session(tmp_path / "together")
        finally:
            stop.set()
            t.join()
    finally:
        v.close()
    assert files == apart_files and md == apart_md
    assert together and all(x == apart_verdicts for x in together)
    assert _counter(b2, "b200post_engine_rider_calls_total") > r0
