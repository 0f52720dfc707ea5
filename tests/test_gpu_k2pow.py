"""k2pow (RandomX) on the GPU, through the C ABI (include/b200post_k2pow.h), against RandomX's own known-answer
vectors and against the CPU oracle (oracle/randomx_oracle.c) on >= 1000 nonces.
Reference seam: activation/nipost.go:171 (search), activation/post_verifier.go:150-160 (check)."""
import numpy as np
import pytest

from oracle import pyrandomx as orx

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def k2(b2, gpu_ready):
    import importlib
    return importlib.import_module("go-spacemesh_b200.k2pow")


def test_randomx_known_answers_on_gpu(k2):
    """RandomX src/tests/tests.cpp vectors, computed by the sm_90a kernels (dataset, AES generators, VM, Blake2b)."""
    assert k2.randomx_hash(b"test key 000", [b"This is a test"])[0].hex() == \
        "639183aae1bf4c9a35884cb46b09cad9175f04efd7684e7262a0ac1c2f0b4e3f"
    assert k2.randomx_hash(b"test key 000", [b"Lorem ipsum dolor sit amet"])[0].hex() == \
        "300a0adb47603dedb42228ccb2b211104f4da45af709cd7547cd049e9489c969"
    long_in = b"sed do eiusmod tempor incididunt ut labore et dolore magna aliqua"
    assert k2.randomx_hash(b"test key 000", [long_in])[0].hex() == "c36d4ed4191e617309867ed66a443be4075014e2b061bcdaf9ce7b721d2b77a8"
    assert k2.randomx_hash(b"test key 001", [long_in])[0].hex() == "e9ff4503201c0c2cca26d285c93ae883f9b1d30c9eb240b820756f2d5a7905fc"
    blob = bytes.fromhex("0b0b98bea7e805e0010a2126d287a2a0cc833d312cb786385a7c2f9de69d25537f584a9bc9977b00000000666fd8753bf61a"
                         "8631f12984e3fd44f4014eca629276817b56f32e9b68bd82f416")
    assert k2.randomx_hash(b"test key 001", [blob])[0].hex() == "c56414121acda1713c2f2a819d8ae38aed7c80c35c2a769298d34f03833cd5f1"


def test_inputs_of_awkward_lengths(k2):
    cache = orx.Cache(b"test key 000")
    try:
        for ln in (0, 1, 127, 128, 129, 300):
            msgs = [bytes((i * 7 + j) & 255 for j in range(ln)) for i in range(3)]
            got = k2.randomx_hash(b"test key 000", msgs)
            for m, g in zip(msgs, got):
                assert g == cache.hash(m), ln
    finally:
        cache.close()


@pytest.fixture(scope="module")
def oracle_default():
    c = orx.Cache(orx.K2POW_CACHE_KEY)
    c.init_dataset()          # fast mode for the checker too: 1000+ hashes in seconds
    yield c
    c.close()


def test_k2pow_hashes_equal_oracle_on_1200_nonces(k2, oracle_default):
    rng = np.random.default_rng(5)
    ch, node = bytes(rng.integers(0, 256, 8, dtype=np.uint8)), bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    for start, count, ng in ((0, 1000, 0), (2**56 - 100, 100, 17), (2**32 - 50, 100, 255)):
        got = k2.hashes(ng, ch, node, start, count)
        exp, _, _ = oracle_default.k2pow_scan(ng, ch, node, start, count)
        bad = np.nonzero((got != exp).any(axis=1))[0]
        assert bad.size == 0, f"{bad.size} of {count} hashes differ, first at pow {start + int(bad[0])}"


def test_every_vm_kernel_variant_equals_the_oracle(k2, b2, oracle_default):
    """rx_vm_mode 0..3 are four builds of the same interpreter (1- and 2-warp CTAs, 32 / 40 / 48 / 64-register budgets):
    each must give the oracle's hashes, including an odd count that leaves a 2-warp CTA half empty."""
    rng = np.random.default_rng(11)
    ch, node = bytes(rng.integers(0, 256, 8, dtype=np.uint8)), bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    exp, _, _ = oracle_default.k2pow_scan(3, ch, node, 12345, 71)
    before = b2.get_option("rx_vm_mode")
    try:
        for mode in (0, 1, 2, 3):
            b2.set_option("rx_vm_mode", mode)
            got = k2.hashes(3, ch, node, 12345, 71)
            assert (got == exp).all(), f"rx_vm_mode {mode}: {(got != exp).any(axis=1).sum()} of 71 hashes differ"
    finally:
        b2.set_option("rx_vm_mode", before)


def test_search_finds_the_first_valid_nonce_and_verify_agrees(k2, oracle_default):
    rng = np.random.default_rng(6)
    ch, node = bytes(rng.integers(0, 256, 8, dtype=np.uint8)), bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    hs = k2.hashes(3, ch, node, 1000, 512)
    order = sorted(range(512), key=lambda i: bytes(hs[i]))
    thr = bytes(hs[order[2]])                      # exactly two nonces of the range are strictly below it
    want = 1000 + min(order[0], order[1])
    found, done = k2.search(3, ch, node, thr, 1000, 512)
    assert found == want and done == 512
    _, ofound, _ = oracle_default.k2pow_scan(3, ch, node, 1000, 512, difficulty=thr, want_hashes=False)
    assert ofound == want
    assert k2.verify(want, 3, ch, node, thr)
    assert not k2.verify(1000 + order[2], 3, ch, node, thr)          # equal to the threshold: strict compare
    assert not k2.verify(want, 4, ch, node, thr) or bytes(k2.hashes(4, ch, node, want, 1)[0]) < thr
    found, done = k2.search(3, ch, node, b"\x00" * 32, 1000, 64)
    assert found is None and done == 64
    assert not k2.verify(2**56, 3, ch, node, b"\xff" * 32)             # does not fit the 7 input bytes


def test_search_walks_batches_and_stops_after_a_hit(k2, b2):
    rng = np.random.default_rng(7)
    ch, node = bytes(rng.integers(0, 256, 8, dtype=np.uint8)), bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    old = b2.get_option("rx_vms_per_sm")
    try:
        b2.set_option("rx_vms_per_sm", 1)
        batch = k2.batch_size()
        hs = k2.hashes(0, ch, node, 0, 3 * batch)
        # threshold = the smallest hash of the second batch, bumped by one: first hit lies in batch 2
        second = sorted(bytes(h) for h in hs[batch:2 * batch])[0]
        thr = (int.from_bytes(second, "big") + 1).to_bytes(32, "big")
        first_batch_min = min(bytes(h) for h in hs[:batch])
        found, done = k2.search(0, ch, node, thr, 0, 3 * batch)
        if first_batch_min < thr:
            assert done == batch
        else:
            assert done == 2 * batch and bytes(hs[found]) == second
        assert bytes(hs[found]) < thr
    finally:
        b2.set_option("rx_vms_per_sm", old)


def test_scale_difficulty(k2):
    d = bytes.fromhex("000dfb23b0979b4b" + "00" * 24)
    for units in (1, 4, 7, 1000):
        assert k2.scale_difficulty(d, units) == orx.scale_pow_difficulty(d, units)


def test_search_over_several_devices(k2, b2):
    """b200post_k2pow_search_multi: batch-interleaved nonce ranges, one host thread per device, same answer as one device
    (BASELINE.json configs[4] shards the nonce range over the box's GPUs; no data-path collective — SURVEY.md §8e)."""
    gpus = [p["id"] for p in b2.providers()]
    if len(gpus) < 2:
        pytest.skip("needs two GPUs")
    rng = np.random.default_rng(8)
    ch, node = bytes(rng.integers(0, 256, 8, dtype=np.uint8)), bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    old = b2.get_option("rx_vms_per_sm")
    try:
        b2.set_option("rx_vms_per_sm", 2)
        batch = k2.batch_size()
        n = 5 * batch + 17
        hs = k2.hashes(0, ch, node, 0, n)
        order = sorted(range(n), key=lambda i: bytes(hs[i]))
        thr = bytes(hs[order[1]])                                   # exactly one nonce of the range is below it
        found, done = k2.search(0, ch, node, thr, 0, n, providers=gpus[:2])
        assert found == order[0] and done <= n
        found1, _ = k2.search(0, ch, node, thr, 0, n, provider=gpus[0])
        assert found1 == found
        none, done = k2.search(0, ch, node, b"\x00" * 32, 0, n, providers=gpus[:2])
        assert none is None and done == n
    finally:
        b2.set_option("rx_vms_per_sm", old)


def test_committed_golden_fixture(k2, golden):
    """tests/golden/k2pow.json (oracle/gen_golden_k2pow.py): RandomX's own vectors and oracle-computed k2pow hashes."""
    g = golden["k2pow"]
    for it in g["randomx_kat"]:
        assert k2.randomx_hash(it["key"].encode(), [bytes.fromhex(it["input_hex"])])[0].hex() == it["hash"]
    for it in g["k2pow"]:
        got = k2.hashes(it["nonce_group"], bytes.fromhex(it["challenge8"]), bytes.fromhex(it["node_id"]), it["pow"], 1)
        assert bytes(got[0]).hex() == it["hash"]
