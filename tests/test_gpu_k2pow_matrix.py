"""GPU tier: k2pow (RandomX) against the CPU oracle (oracle/randomx_oracle.c) on the paths where the easy shapes of
test_gpu_k2pow.py do not go.

* The whole 2080 MiB dataset that `dataset_kernel` builds, byte for byte, including the final partial block of 255
  items that a hash reads with a probability of about 2e-9 per dataset access; a second key; the rebuild into the
  reused buffer.
* Batch seams: calls split over several device batches, for every VM kernel variant, across the 2^32 carry of the
  pow, and with batch buffers left over from a larger batch size (stride > batch).
* The top of the 56-bit nonce space.
* `b200post_k2pow_search_groups`, the prover's search: one pow per group of 16 nonces, groups sharing device batches
  in rounds while the list of groups still searching shrinks.
* `b200post_generate_proof` with the builtin pow, end to end, and the verifier's builtin pow verdict at its boundary
  (hash < floor(pow_difficulty / num_units), strict) over batches of proofs larger than one device batch.

Batch sizes come from the library under the options each case sets, never from constants; every option is restored.
About 3 800 oracle hashes in all, served by one fast-mode oracle for the default key."""
import contextlib
import importlib
import time
from pathlib import Path

import numpy as np
import pytest

from oracle import pyrandomx as orx

pytestmark = pytest.mark.gpu

ITEMS = orx.DATASET_ITEMS
READ_ITEMS = (64 << 20) // 64                  # dataset items per read-back: 64 MiB of host memory at a time
OTHER_KEY = b"test key 000"
NONCE_SPACE = 2**56                            # the k2pow input carries 7 bytes of pow


@pytest.fixture(scope="module")
def k2(b2, gpu_ready):
    return importlib.import_module("go-spacemesh_b200.k2pow")


@pytest.fixture(scope="module")
def mods(b2, gpu_ready):
    return (importlib.import_module("go-spacemesh_b200.setup"), importlib.import_module("go-spacemesh_b200.prove"),
            importlib.import_module("go-spacemesh_b200.verify"))


@pytest.fixture(scope="module")
def oracle():
    """Fast-mode oracle for the default key: its dataset is the whole-dataset reference and makes hashes cheap."""
    t0 = time.perf_counter()
    c = orx.Cache(orx.K2POW_CACHE_KEY)
    t1 = time.perf_counter()
    c.init_dataset()
    print(f"\noracle fixture: cache {t1 - t0:.1f} s, dataset {time.perf_counter() - t1:.1f} s")
    yield c
    c.close()


@contextlib.contextmanager
def options(b2, **values):
    before = {k: b2.get_option(k) for k in values}
    try:
        for k, v in values.items():
            b2.set_option(k, v)
        yield
    finally:
        for k, v in before.items():
            b2.set_option(k, v)


def _ids(seed: int):
    r = np.random.default_rng(seed)
    return bytes(r.integers(0, 256, 8, dtype=np.uint8)), bytes(r.integers(0, 256, 32, dtype=np.uint8))


def _rate(r: int) -> bytes:
    """A difficulty that a uniform hash passes with probability 1/r."""
    return (2**256 // r).to_bytes(32, "big")


def _rows_differ(got: np.ndarray, exp: np.ndarray) -> np.ndarray:
    return np.nonzero((got != exp).any(axis=1))[0]


# ------------------------------------------------------------------------------------------------------ a. dataset
def _dataset_mismatches(k2, ref: np.ndarray, provider: int, key=None):
    """(items that differ, first differing item) over the whole dataset, read back 64 MiB at a time."""
    bad, first_bad = 0, None
    for first in range(0, ITEMS, READ_ITEMS):
        n = min(READ_ITEMS, ITEMS - first)
        d = _rows_differ(k2.dataset(first, n, key, provider=provider), ref[first:first + n])
        if d.size:
            bad += d.size
            first_bad = first + int(d[0]) if first_bad is None else first_bad
    return bad, first_bad


def test_whole_dataset_equals_oracle_on_every_device(k2, b2, oracle):
    ref = oracle.dataset()
    for p in b2.providers():
        bad, first = _dataset_mismatches(k2, ref, p["id"])
        assert bad == 0, f"device {p['id']}: {bad} of {ITEMS} dataset items differ, first at item {first}"


def test_dataset_of_another_key_then_rebuild_of_the_default(k2, oracle):
    """Another key rebuilds the dataset into the same buffer; its head, tail, final partial block, the items at 2^31
    bytes and 65 536 random items must equal the oracle's light-mode items.  Switching back must rebuild the default
    key's dataset exactly."""
    assert ITEMS % 256 == 255                       # the last 256-thread block of dataset_kernel holds 255 items
    rng = np.random.default_rng(12)
    want = np.unique(np.concatenate([np.arange(4096), np.arange(ITEMS - 4096, ITEMS), np.arange(2**25 - 2, 2**25 + 3),
                                     rng.integers(0, ITEMS, 65536)]))
    light = orx.Cache(OTHER_KEY)
    try:
        exp = np.stack([light.dataset_item(int(i)) for i in want])
    finally:
        light.close()
    got = np.empty_like(exp)
    for first in range(0, ITEMS, READ_ITEMS):
        n = min(READ_ITEMS, ITEMS - first)
        sel = (want >= first) & (want < first + n)
        if sel.any():
            got[sel] = k2.dataset(first, n, OTHER_KEY)[want[sel] - first]
    d = _rows_differ(got, exp)
    assert d.size == 0, f"key {OTHER_KEY!r}: {d.size} of {want.size} items differ, first at item {int(want[d[0]])}"
    bad, first = _dataset_mismatches(k2, oracle.dataset(), 0)
    assert bad == 0, f"default key rebuilt: {bad} of {ITEMS} dataset items differ, first at item {first}"


# ------------------------------------------------------------------------------------------------- b. batch seams
def test_multi_batch_calls_equal_oracle_for_every_vm_variant(k2, b2, oracle):
    """2 * batch + 33 nonces from 2^32 - batch - 5: three device batches, the second of which crosses the 2^32 carry of
    the pow, for rx_vm_mode 0..3 at 1 and 3 VMs per SM.  One oracle range covers every configuration."""
    ch, node = _ids(21)
    ng = 0x5c
    batches = {}
    for per_sm in (1, 3):
        with options(b2, rx_vms_per_sm=per_sm):
            batches[per_sm] = k2.batch_size()
    top = max(batches.values())
    lo, hi = 2**32 - top - 5, 2**32 + top + 28
    exp, _, _ = oracle.k2pow_scan(ng, ch, node, lo, hi - lo)
    for mode in (0, 1, 2, 3):
        for per_sm, batch in batches.items():
            with options(b2, rx_vm_mode=mode, rx_vms_per_sm=per_sm):
                assert k2.batch_size() == batch
                start, count = 2**32 - batch - 5, 2 * batch + 33
                got = k2.hashes(ng, ch, node, start, count)
                t = k2.last_timing()
                d = _rows_differ(got, exp[start - lo:start - lo + count])
                assert d.size == 0, f"rx_vm_mode {mode}, batch {batch}: {d.size} of {count} hashes differ, first at pow {start + int(d[0])}"
                assert t["vm_launches"] == 8 * -(-count // batch) and t["hashes"] == count
                print(f"rx_vm_mode {mode}, {per_sm} VM/SM: {count} hashes in {t['total_ms']:.1f} ms = "
                      f"{count / t['total_ms'] * 1e3:.0f} H/s (VM kernel {t['vm_kernel_ms']:.1f} ms)")


def test_batch_buffers_left_from_a_larger_batch(k2, b2, oracle):
    """After a call at the default batch size the buffers hold more VMs than a later, smaller batch uses (stride > batch):
    hashes and randomx_hash must not change.  randomx_hash over batch + 1 inputs at lengths around Blake2b's 128-byte
    block splits into two launches."""
    ch, node = _ids(22)
    ng = 201
    big = k2.batch_size()
    with options(b2, rx_vms_per_sm=1):
        small = k2.batch_size()
    assert small < big
    start, count = 2**40 - small - 3, 2 * small + 9
    exp, _, _ = oracle.k2pow_scan(ng, ch, node, start, count)
    large = k2.hashes(ng, ch, node, start, big + 1)
    assert k2.last_timing()["vm_launches"] == 16
    d = _rows_differ(large[:count], exp)
    assert d.size == 0, f"default batch {big}: {d.size} of {count} hashes differ, first at pow {start + int(d[0])}"
    with options(b2, rx_vms_per_sm=1):
        got = k2.hashes(ng, ch, node, start, count)
        assert k2.last_timing()["vm_launches"] == 8 * -(-count // small)
        d = _rows_differ(got, exp)
        assert d.size == 0, f"batch {small} in buffers of {big}: {d.size} of {count} hashes differ, first at pow {start + int(d[0])}"
        rng = np.random.default_rng(23)
        for ln in (0, 48, 128, 256, 300):
            msgs = [bytes(rng.integers(0, 256, ln, dtype=np.uint8)) for _ in range(small + 1)]
            got = k2.randomx_hash(None, msgs)
            assert k2.last_timing()["vm_launches"] == 16
            bad = [i for i, (m, g) in enumerate(zip(msgs, got)) if g != oracle.hash(m)]
            assert not bad, f"input length {ln}: {len(bad)} of {small + 1} hashes differ, first at input {bad[0]}"


# ------------------------------------------------------------------------------------------ c. top of the nonce space
def test_top_of_the_nonce_space(k2, oracle):
    ch, node = _ids(24)
    ng = 3
    got = k2.hashes(ng, ch, node, NONCE_SPACE - 3, 3)
    exp, _, _ = oracle.k2pow_scan(ng, ch, node, NONCE_SPACE - 3, 3)
    assert (got == exp).all()
    top = bytes(exp[2])                                          # the hash of pow 2^56 - 1
    above = (int.from_bytes(top, "big") + 1).to_bytes(32, "big")
    assert not k2.verify(NONCE_SPACE - 1, ng, ch, node, top)    # strict: a hash equal to the difficulty fails
    assert k2.verify(NONCE_SPACE - 1, ng, ch, node, above)
    assert not k2.verify(NONCE_SPACE, ng, ch, node, b"\xff" * 32)
    assert k2.search(ng, ch, node, b"\x00" * 32, NONCE_SPACE - 40, 1000) == (None, 40)
    assert k2.search(ng, ch, node, b"\xff" * 32, NONCE_SPACE - 40, 1000) == (NONCE_SPACE - 40, 40)


# -------------------------------------------------------------------------------------------- d. search_groups
def _hashes_done(batch: int, n_groups: int, cap: int, pows) -> int:
    """The round schedule of b200post_k2pow_search_groups: every pending group tries `per` more nonces per round."""
    pending, nxt, total = list(range(n_groups)), 0, 0
    cap = cap or NONCE_SPACE
    while pending and nxt < cap:
        per = min(max(1, batch // len(pending)), cap - nxt)
        total += len(pending) * per
        pending = [g for g in pending if pows[g] is None or pows[g] >= nxt + per]
        nxt += per
    return total


GROUP_CASES = [   # (groups, rx_vms_per_sm or None = default, 1 / pass rate, max_nonces_per_group)
    (1, None, 16, 0),       # one group
    (18, 1, 16, 0),         # mainnet: 288 nonces, several rounds while the pending list shrinks
    (256, 1, 4, 0),         # more groups than a batch holds: one nonce each, group byte 255, two launches per round
    (5, 1, 64, 40),         # the cap ends the search with groups still pending
]


@pytest.mark.parametrize("case", GROUP_CASES, ids=[f"{c[0]}groups-1in{c[2]}-cap{c[3]}" for c in GROUP_CASES])
def test_search_groups_finds_the_smallest_pow_of_every_group(k2, b2, oracle, case):
    n_groups, per_sm, rate, cap = case
    ch, node = _ids(30 + GROUP_CASES.index(case))
    diff = _rate(rate)
    with options(b2, **({} if per_sm is None else {"rx_vms_per_sm": per_sm})):
        batch = k2.batch_size()
        pows, done = k2.search_groups(ch, node, diff, n_groups, cap)
    assert len(pows) == n_groups
    for g, pw in enumerate(pows):
        if pw is None:
            assert cap, f"group {g}: not found in the whole nonce space"
            _, found, _ = oracle.k2pow_scan(g, ch, node, 0, cap, diff, want_hashes=False)
            assert found is None, f"group {g}: the oracle finds pow {found} below the cap {cap}"
        else:
            assert pw < (cap or NONCE_SPACE)
            _, found, _ = oracle.k2pow_scan(g, ch, node, 0, pw + 1, diff, want_hashes=False)
            assert found == pw, f"group {g}: GPU pow {pw}, smallest valid pow {found}"
    if cap:
        assert None in pows and any(p is not None for p in pows)
    assert done == _hashes_done(batch, n_groups, cap, pows)


# --------------------------------------------------------------------------- e. generate_proof with the builtin pow
NODE, ATX = bytes(range(60, 92)), bytes(range(160, 192))


def _oracle_first_pow(oracle, group: int, ch8: bytes, node: bytes, diff: bytes, window: int = 16) -> int:
    start = 0
    while True:
        _, found, _ = oracle.k2pow_scan(group, ch8, node, start, window, diff, want_hashes=False)
        if found is not None:
            return found
        start += window


def test_generate_proof_with_the_builtin_pow_equals_oracle(mods, b2, orc, oracle, tmp_path):
    """3 units, so pow_difficulty / num_units truncates; 288 nonces (18 groups) at one VM per SM, so the search takes
    several rounds.  The proof must be the oracle's, with the oracle's smallest pow of the winning group, and the
    verifier's builtin pow check must accept it."""
    su, pr, vf = mods
    units, lpu, k1, kk2, nonces = 3, 4096, 300, 12, 288
    num_labels = units * lpu
    pow_difficulty = bytes([0x30]) + bytes(range(101, 132))
    d = int.from_bytes(pow_difficulty, "big")
    assert d % units                                             # the division truncates
    scaled = (d // units).to_bytes(32, "big")
    cfg = su.PostConfig(labels_per_unit=lpu, k1=k1, k2=kk2, k3=kk2, max_num_units=8, pow_difficulty=pow_difficulty)
    o = su.PostSetupOpts(data_dir=str(tmp_path), num_units=units, max_file_size=16 * 5000, provider_id=0, scrypt_n=2)
    mgr = su.PostSetupManager(cfg)
    mgr.prepare_initializer(o, NODE, ATX)
    mgr.start_session()
    assert mgr.status().state == su.STATE_COMPLETE
    files = sorted(Path(o.data_dir).glob("postdata_*.bin"), key=lambda f: int(f.stem.split("_")[1]))
    labels = np.concatenate([np.fromfile(f, dtype=np.uint8) for f in files]).reshape(-1, 16)
    assert labels.shape[0] == num_labels

    challenge = bytes(range(7, 39))
    pows = [_oracle_first_pow(oracle, g, challenge[:8], NODE, scaled) for g in range(nonces // 16)]
    nonce, idx = orc.np_prove_multi(labels, challenge, nonces, pows, k1, kk2, num_labels)
    assert nonce is not None
    with options(b2, rx_vms_per_sm=1):
        proof, meta, _ = pr.generate_proof(o.data_dir, challenge, cfg, nonces=nonces)
    assert (proof.nonce, vf.unpack_indices(proof.indices, vf.bits_per_index(num_labels), kk2), proof.pow) == \
        (nonce, idx, pows[nonce // 16])
    v = vf.PostVerifier()
    try:
        v.verify(proof, meta, vf.VerifyParams(k1=k1, k2=kk2, scrypt_n=2, pow_difficulty=pow_difficulty))
    finally:
        v.close()


# -------------------------------------------------------------------------------- f. the verifier's pow verdict
def _proofs(vf, rng, pows, num_labels: int, k2: int):
    bits = vf.bits_per_index(num_labels)
    return [vf.Proof(int(rng.integers(0, 4096)), vf.pack_indices(rng.integers(0, num_labels, k2), bits), int(p)) for p in pows]


def test_verifier_pow_verdict_over_several_launches_and_at_the_boundary(k2, mods, b2, oracle):
    """verify_batch with the builtin check over 2 * batch + 7 proofs at one VM per SM: POW_INVALID exactly where the
    oracle hash is >= floor(pow_difficulty / num_units).  A proof whose pow passes goes on to the label check (its
    labels are judged under the new key), so it may fail there, but never as POW_INVALID."""
    _, _, vf = mods
    ch32, node = bytes(range(200, 232)), bytes(range(40, 72))
    k1, kk2, num_labels = 100, 4, 1024
    rng = np.random.default_rng(40)
    with options(b2, rx_vms_per_sm=1):
        batch = k2.batch_size()
        n = 2 * batch + 7
        pow_list = [int(p) for p in rng.integers(0, NONCE_SPACE, n - 1, dtype=np.uint64)] + [NONCE_SPACE - 1]
        proofs = _proofs(vf, rng, pow_list, num_labels, kk2)
        hashes = [int.from_bytes(oracle.hash(orx.k2pow_input(p.pow, p.nonce // 16, ch32[:8], node)), "big") for p in proofs]

        meta2 = vf.ProofMetadata(node, ATX, ch32, 2, num_labels // 2)
        q = vf.VerifyParams(k1=k1, k2=kk2, scrypt_n=2, pow_difficulty=b"\xff" * 32)
        target = (2**256 - 1) // 2
        expect_bad = [h >= target for h in hashes]
        assert 0.3 * n < sum(expect_bad) < 0.7 * n
        st, bad = vf.verify_batch(proofs, [meta2] * n, q, pow="builtin")
        got_bad = [s == b2.ERR_INVALID_PROOF and b == vf.POW_INVALID for s, b in zip(st, bad)]
        assert got_bad == expect_bad, f"pow verdicts differ at proofs {[i for i in range(n) if got_bad[i] != expect_bad[i]][:10]}"
        assert all(s in (b2.OK, b2.ERR_INVALID_PROOF) for s in st)

        # the boundary, with num_units = 4: target = floor((4h + 3) / 4) = h fails, floor((4h + 4) / 4) = h + 1 passes
        meta4 = vf.ProofMetadata(node, ATX, ch32, 4, num_labels // 4)
        i = next(i for i, h in enumerate(hashes) if h < 2**254 - 1)
        p, h = proofs[i], hashes[i]
        for pd, pow_bad in ((4 * h + 3, True), (4 * h + 4, False)):
            q = vf.VerifyParams(k1=k1, k2=kk2, scrypt_n=2, pow_difficulty=pd.to_bytes(32, "big"))
            st, bad = vf.verify_batch([p], [meta4], q, pow="builtin")
            assert (st[0] == b2.ERR_INVALID_PROOF and bad[0] == vf.POW_INVALID) == pow_bad, (pd - 4 * h, st, bad)

        # pow 2^56 - 1 is judged by its hash; 2^56 does not fit the 7 hashed bytes and is refused whatever the difficulty
        meta1 = vf.ProofMetadata(node, ATX, ch32, 1, num_labels)
        q = vf.VerifyParams(k1=k1, k2=kk2, scrypt_n=2, pow_difficulty=b"\xff" * 32)
        last = proofs[-1]
        assert last.pow == NONCE_SPACE - 1 and hashes[-1] < 2**256 - 1
        refused = vf.Proof(last.nonce, last.indices, NONCE_SPACE)
        st, bad = vf.verify_batch([last, refused], [meta1] * 2, q, pow="builtin")
        assert bad[0] != vf.POW_INVALID
        assert st[1] == b2.ERR_INVALID_PROOF and bad[1] == vf.POW_INVALID
