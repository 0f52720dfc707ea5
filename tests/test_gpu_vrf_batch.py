"""GPU tier: VRF-nonce checks in batches (b200post_verify_vrf_nonces[_multi]) and through the verifier handle
(b200post_verifier_verify_vrf_nonce), against the reference's real checkpoint data, the CPU oracle and the single call.

Every check returns (status, valid, label32).  valid is label32 < floor(2^256 / numLabels), strict: the UNPINNED rule of
b200post_verify_vrf_nonce, restated here in Python; label32 is what a caller applies the network's own rule to."""
import importlib
import threading
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# tests/golden/checkpoint_vrf.json positions whose real, network-accepted nonce lies above the unpinned threshold (the
# same list as tests/test_gpu_labels.py, restated so that this file stands on its own)
VRF_THRESHOLD_REJECTS_THESE_REAL_NONCES = [0, 5, 7, 11, 13, 15, 20, 23, 26, 28, 29, 30, 31, 33, 36, 41]


@pytest.fixture(scope="module")
def vf(b2, gpu_ready):
    return importlib.import_module("go-spacemesh_b200.verify")


@pytest.fixture(scope="module")
def devs(b2, gpu_ready):
    """Provider lists for the split and the verifier's workers: a one-GPU box lists its device twice."""
    gpus = [p["id"] for p in gpu_ready]
    return [[gpus[0]], [gpus[0], gpus[0]]] + ([gpus] if len(gpus) > 1 else [])


def _rule(label32: bytes, num_labels: int) -> bool:
    return int.from_bytes(label32, "big") < (1 << 256) // num_labels


def _random_checks(rng, count, n, idents=None):
    """(node, atx, nonce, units, lpu, n) tuples: nonces inside and past the end of the POST and above 2^32."""
    out = []
    for i in range(count):
        node, atx = idents[i % len(idents)] if idents else (bytes(rng.integers(0, 256, 32, dtype=np.uint8)),
                                                            bytes(rng.integers(0, 256, 32, dtype=np.uint8)))
        units, lpu = int(rng.integers(1, 200)), int(rng.choice([2, 1024, 2**20, 2**32, 2**40]))
        nl = units * lpu
        nonce = [int(rng.integers(0, nl)), nl + int(rng.integers(0, 1000)), 2**32 + int(rng.integers(0, 2**20)),
                 int(rng.integers(0, 2**63)) * 2 + 1, nl - 1][i % 5]
        out.append((node, atx, nonce, units, lpu, n))
    return out


def _oracle(orc, checks):
    return [orc.c_label32(orc.c_commitment(c[0], c[1]), c[2], c[5]) for c in checks]


def _expect_ok(b2, got, checks, labels):
    for k, ((st, ok, l32), c, exp) in enumerate(zip(got, checks, labels)):
        assert st == b2.OK and l32 == exp, (k, c[2], c[5])
        assert ok == _rule(exp, c[3] * c[4]), k


def test_real_checkpoint_identities_in_one_batch(b2, golden):
    """The 42 identities of the reference's checkpoint fixture: the golden label32 at every nonce, the documented rejects
    of the unpinned rule, and the same answer as the single calls."""
    items = golden["checkpoint_vrf"]["items"]
    checks = [(bytes.fromhex(it["node_id"]), bytes.fromhex(it["commitment_atx"]), it["vrf_nonce"], it["num_units"],
               it["labels_per_unit"], 8192) for it in items]
    got = b2.verify_vrf_nonces(checks)
    assert [g[0] for g in got] == [b2.OK] * len(items)
    assert [g[2].hex() for g in got] == [it["label32"] for it in items]
    assert [i for i, g in enumerate(got) if not g[1]] == VRF_THRESHOLD_REJECTS_THESE_REAL_NONCES
    for (st, ok, l32), c in zip(got, checks):
        assert b2.verify_vrf_nonce(c[2], c[0], c[1], c[3], c[4], 8192) == ok
        assert b2.vrf_nonce_label(c[2], c[0], c[1], 8192) == l32


@pytest.mark.parametrize("n,count", [(2, 400), (8192, 40)])
def test_random_identities_match_the_oracle(b2, orc, n, count):
    rng = np.random.default_rng(n + count)
    checks = _random_checks(rng, count, n)
    got = b2.verify_vrf_nonces(checks)
    _expect_ok(b2, got, checks, _oracle(orc, checks))
    assert 0 < sum(g[1] for g in got) < count or n == 8192   # N = 2 with lpu = 2: both verdicts occur


def test_per_item_thresholds_at_the_boundary(b2, orc, golden):
    """For items with known label L, numLabels nl with floor(2^256/nl) > L >= floor(2^256/(nl+1)): (nl, num_units 1)
    is valid and (nl + 1) is not.  All pairs go into ONE batch, shuffled, with N = 2 and N = 8192 items mixed, so a
    kernel that reads another item's threshold (or position) fails."""
    rng = np.random.default_rng(9)
    base = [(bytes.fromhex(it["node_id"]), bytes.fromhex(it["commitment_atx"]), it["vrf_nonce"], 8192,
             bytes.fromhex(it["label32"])) for it in golden["checkpoint_vrf"]["items"][:20]]
    for c in _random_checks(rng, 20, 2):
        base.append((c[0], c[1], c[2], 2, orc.c_label32(orc.c_commitment(c[0], c[1]), c[2], 2)))
    checks, expect = [], []
    for node, atx, nonce, n, l32 in base:
        L = int.from_bytes(l32, "big")
        nl = (1 << 256) // (L + 1)
        assert 1 <= nl < 2**64 - 1 and (1 << 256) // nl > L >= (1 << 256) // (nl + 1)
        for lpu, ok in ((nl, True), (nl + 1, False)):
            checks.append((node, atx, nonce, 1, lpu, n))
            expect.append((ok, l32))
    order = rng.permutation(len(checks))
    got = b2.verify_vrf_nonces([checks[i] for i in order])
    for k, i in enumerate(order):
        assert got[k] == (b2.OK, *expect[i]), (k, i)
    assert len({c[4] for c in checks}) > 30          # the thresholds really differ from item to item


def _seam_case(b2, orc, rng, count, n):
    idents = [(bytes(rng.integers(0, 256, 32, dtype=np.uint8)), bytes(rng.integers(0, 256, 32, dtype=np.uint8))) for _ in range(7)]
    checks = _random_checks(rng, count, n, idents)
    got = b2.verify_vrf_nonces(checks)
    assert len(got) == count and all(g[0] == b2.OK for g in got)
    comms = np.stack([np.frombuffer(orc.c_commitment(c[0], c[1]), dtype=np.uint8) for c in checks])
    lo = orc.c_labels_gather(comms, np.array([c[2] for c in checks], dtype=np.uint64), n)
    assert b"".join(g[2][:16] for g in got) == lo.tobytes()
    # the whole label32 and the verdict: around every 128-item CTA edge near the ends, at layer seams, and a sample
    pick = sorted({*range(min(count, 260)), *range(max(0, count - 260), count), *range(0, count, max(1, count // 300))})
    sub = [checks[i] for i in pick]
    _expect_ok(b2, [got[i] for i in pick], sub, _oracle(orc, sub))


@pytest.mark.parametrize("count", [1, 4096, 4097, "wave+1"])
def test_batch_seams(b2, orc, count):
    """1 and 4096 checks take the low-latency ROMix kernel, 4097 the pipelined one, wave_slots + 1 two layers."""
    n = 2
    count = b2.wave_slots(n) + 1 if count == "wave+1" else count
    _seam_case(b2, orc, np.random.default_rng(count), count, n)
    if count == 1:
        _seam_case(b2, orc, np.random.default_rng(0), 1, 8192)


def test_malformed_items_fail_alone(b2, orc):
    rng = np.random.default_rng(4)
    good = _random_checks(rng, 6, 2)
    node, atx = good[0][0], good[0][1]
    bad = [(node, atx, 5, 0, 1024, 2), (node, atx, 5, 4, 0, 2), (node, atx, 5, 2**32 - 1, 2**40, 2),
           (node, atx, 5, 4, 1024, 3), (node, atx, 5, 4, 1024, 2**21), (node, atx, 5, 4, 1024, 0)]
    checks = [x for pair in zip(good, bad) for x in pair]
    got = b2.verify_vrf_nonces(checks)
    assert [g for g in got[1::2]] == [(b2.ERR_INVALID_ARGUMENT, False, bytes(32))] * len(bad)
    _expect_ok(b2, got[0::2], good, _oracle(orc, good))
    # a batch of malformed items only, and one where a whole N group is invalid
    assert [g[0] for g in b2.verify_vrf_nonces(bad)] == [b2.ERR_INVALID_ARGUMENT] * len(bad)


def test_empty_batch(b2, devs):
    assert b2.verify_vrf_nonces([]) == []
    for d in devs:
        assert b2.verify_vrf_nonces([], providers=d) == []


def test_mixed_n_in_one_batch(b2, orc):
    rng = np.random.default_rng(8)
    a, b = _random_checks(rng, 30, 2), _random_checks(rng, 12, 8192)
    checks = [x for pair in zip(a[:12], b) for x in pair] + a[12:]
    _expect_ok(b2, b2.verify_vrf_nonces(checks), checks, _oracle(orc, checks))


def test_multi_equals_one_device(b2, devs):
    rng = np.random.default_rng(12)
    checks = _random_checks(rng, 777, 2) + _random_checks(rng, 9, 8192)
    one = b2.verify_vrf_nonces(checks)
    for d in devs:
        assert b2.verify_vrf_nonces(checks, providers=d) == one, d
        assert b2.verify_vrf_nonces(checks[:1], providers=d) == one[:1], d


# ------------------------------------------------------------------------------------------------ the verifier handle
@pytest.fixture(scope="module")
def space(orc, vf):
    """A 4 x 256-label POST at N = 2 with a brute-forced valid proof per nonce."""
    rng = np.random.default_rng(42)
    node_id, atx, challenge = (bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(3))
    meta = vf.ProofMetadata(node_id, atx, challenge, num_units=4, labels_per_unit=256)
    params = vf.VerifyParams(k1=200, k2=8, scrypt_n=2)
    proofs = []
    for nonce, pow_ in ((0, 0), (5, 77), (17, 2**40 + 3)):
        packed, hits = orc.py_prove(node_id, atx, challenge, 4, 256, params.k1, params.k2, 2, nonce=nonce, pow_=pow_)
        assert packed is not None
        proofs.append(vf.Proof(nonce, packed, pow_))
        bad = list(hits); bad[2] = (bad[2] + 1) % 1024
        proofs.append(vf.Proof(nonce, vf.pack_indices(bad, vf.bits_per_index(1024)), pow_))
    return meta, params, proofs


def _proof_verdict(vf, v, proof, meta, params):
    try:
        v.verify(proof, meta, params)
        return None
    except vf.ErrInvalidIndex as e:
        return e.index


@pytest.mark.parametrize("which", [0, 1, 2])
def test_verifier_mixes_proofs_and_vrf_checks(vf, b2, devs, space, which):
    """Concurrent proof and VRF callers on one handle: proofs as a proofs-only run says, checks as the batch call says,
    fewer batches than calls, and only the proofs counted as proofs."""
    if which >= len(devs):
        pytest.skip("one GPU: the real device list is [0]")
    meta, params, proofs = space
    st, bad = vf.verify_batch(proofs, [meta] * len(proofs), params, pow="skip")
    expect_proof = [None if s == b2.OK else i for s, i in zip(st, bad)]
    assert None in expect_proof and any(e is not None for e in expect_proof)
    checks = _random_checks(np.random.default_rng(1), 24, 2) + _random_checks(np.random.default_rng(2), 3, 8192)
    expect_vrf = [(g[1], g[2]) for g in b2.verify_vrf_nonces(checks)]
    v = vf.PostVerifier(pow="skip", providers=devs[which])
    errors, calls = [], 32 * 4

    def caller(k):
        try:
            for rep in range(4):
                j = k * 4 + rep
                if j % 2:
                    c = checks[j % len(checks)]
                    got = v.verify_vrf_nonce(c[0], c[1], c[2], c[3], c[4], c[5], prioritized=(k % 7 == 0))
                    if got != expect_vrf[j % len(checks)]:
                        errors.append(("vrf", j, got))
                else:
                    p = j % len(proofs)
                    got = _proof_verdict(vf, v, proofs[p], meta, params)
                    if got != expect_proof[p]:
                        errors.append(("proof", j, got, expect_proof[p]))
        except Exception as e:  # noqa: BLE001
            errors.append((k, repr(e)))

    threads = [threading.Thread(target=caller, args=(k,)) for k in range(32)]
    for t in threads: t.start()
    for t in threads: t.join()
    batches, n_proofs = v.stats()
    v.close()
    assert not errors, errors[:3]
    assert n_proofs == calls // 2 and batches < calls, (batches, n_proofs)


class _Gate:
    """pow CALLBACK that counts its calls and holds the FIRST one until released: the batch it belongs to stays on the
    device while the test queues what must go into the next batch."""

    def __init__(self):
        self.calls, self.started, self.release = 0, threading.Event(), threading.Event()

    def __call__(self, ctx, pow_, nonce_group, challenge8, difficulty, node_id):
        self.calls += 1
        if self.calls == 1:
            self.started.set()
            self.release.wait(30)
        return 0


def _settle():
    time.sleep(0.2)   # the callers just started block inside the library: give every one of them time to enqueue


def test_initial_atx_proof_and_vrf_check_share_a_batch(vf, b2, space):
    """The checks of an initial ATX, for one identity: its proof and its VRF nonce, queued behind a long batch, go out
    together in the next batch and both come back right.  The pow callback runs once per proof, never for a VRF check."""
    meta, params, proofs = space
    gate = _Gate()
    v = vf.PostVerifier(pow=gate)
    nl = meta.num_units * meta.labels_per_unit
    long_meta = vf.ProofMetadata(meta.node_id, meta.commitment_atx_id, meta.challenge, 1, 2**20)
    long_params = vf.VerifyParams(k1=2**19, k2=10000, scrypt_n=2)
    long_proof = vf.Proof(0, vf.pack_indices(list(range(0, 10000 * 97, 97)), vf.bits_per_index(2**20)), 0)
    nonce = 2 * nl + 3                                  # past the end: what the past-the-end search produces
    exp_vrf = b2.verify_vrf_nonces([(meta.node_id, meta.commitment_atx_id, nonce, meta.num_units, meta.labels_per_unit, 2)])[0]
    res = {}

    def run(tag, fn):
        try:
            res[tag] = fn()
        except Exception as e:  # noqa: BLE001
            res[tag] = e

    t_long = threading.Thread(target=run, args=("long", lambda: _proof_verdict(vf, v, long_proof, long_meta, long_params)))
    t_long.start()
    assert gate.started.wait(30)
    t_p = threading.Thread(target=run, args=("proof", lambda: _proof_verdict(vf, v, proofs[0], meta, params)))
    t_v = threading.Thread(target=run, args=("vrf", lambda: v.verify_vrf_nonce(meta.node_id, meta.commitment_atx_id, nonce,
                                                                               meta.num_units, meta.labels_per_unit, 2)))
    t_p.start(); t_v.start()
    _settle()
    gate.release.set()
    for t in (t_long, t_p, t_v): t.join()
    batches, n_proofs = v.stats()
    v.close()
    assert res["proof"] is None and res["vrf"] == (exp_vrf[1], exp_vrf[2]), res
    assert (batches, n_proofs) == (2, 2)               # {long} then {proof, VRF check}
    assert gate.calls == 2                             # one per proof, none for the VRF check


def test_prioritized_vrf_check_jumps_the_queue(vf, b2, space):
    meta, params, proofs = space
    gate = _Gate()
    v = vf.PostVerifier(pow=gate, max_batch_proofs=1)
    order, lock = [], threading.Lock()

    def call(tag, fn):
        fn()
        with lock:
            order.append(tag)

    first = threading.Thread(target=call, args=("n0", lambda: _proof_verdict(vf, v, proofs[0], meta, params)))
    first.start()
    assert gate.started.wait(30)
    normal = [threading.Thread(target=call, args=(f"n{i}", lambda: _proof_verdict(vf, v, proofs[1], meta, params)))
              for i in range(1, 9)]
    for t in normal: t.start()
    _settle()
    pr = threading.Thread(target=call, args=("PRIO", lambda: v.verify_vrf_nonce(meta.node_id, meta.commitment_atx_id, 7, 4, 256, 2,
                                                                                prioritized=True)))
    pr.start()
    _settle()
    gate.release.set()
    for t in [first, pr] + normal: t.join()
    batches, n_proofs = v.stats()
    v.close()
    assert (batches, n_proofs) == (10, 9)
    assert order.index("PRIO") <= 2, order             # the held batch, then the prioritised check
    assert gate.calls == 9


def test_close_wakes_vrf_waiters(vf, b2, space):
    meta, params, proofs = space
    gate = _Gate()
    v = vf.PostVerifier(pow=gate)
    res, lock = [], threading.Lock()

    def vrf_call(k):
        try:
            v.verify_vrf_nonce(meta.node_id, meta.commitment_atx_id, k, 4, 256, 2)
            r = "ok"
        except vf.ErrVerifierClosed:
            r = "closed"
        with lock:
            res.append(r)

    held = threading.Thread(target=lambda: _proof_verdict(vf, v, proofs[0], meta, params))
    held.start()
    assert gate.started.wait(30)
    waiters = [threading.Thread(target=vrf_call, args=(k,)) for k in range(6)]
    for t in waiters: t.start()
    _settle()
    closer = threading.Thread(target=v.close)
    closer.start()
    time.sleep(0.1)
    gate.release.set()
    for t in [held, closer] + waiters: t.join()
    assert res == ["closed"] * 6
    t0 = time.monotonic()
    with pytest.raises(vf.ErrVerifierClosed):
        v.verify_vrf_nonce(meta.node_id, meta.commitment_atx_id, 1, 4, 256, 2)
    assert time.monotonic() - t0 < 1.0
    assert gate.calls == 1


def test_verifier_vrf_argument_errors(vf, b2, space):
    meta, _, _ = space
    v = vf.PostVerifier(pow="skip")
    try:
        for units, lpu, n in ((0, 256, 2), (4, 0, 2), (2**32 - 1, 2**40, 2), (4, 256, 3), (4, 256, 2**21)):
            with pytest.raises(b2.B200PostError) as e:
                v.verify_vrf_nonce(meta.node_id, meta.commitment_atx_id, 1, units, lpu, n)
            assert e.value.code == b2.ERR_INVALID_ARGUMENT, (units, lpu, n)
        assert v.stats()[1] == 0
    finally:
        v.close()
