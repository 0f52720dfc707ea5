"""CPU tier: the oracle against public KATs, the real VRF nonces of the reference's checkpoint fixture, the
committed golden vectors and the independent numpy restatement."""
import hashlib
import os

import numpy as np
import pytest


def test_rfc7914_scrypt_vectors(orc, golden):
    for v in golden["kat_primitives"]["scrypt"]:
        got = orc.c_scrypt(v["P"].encode(), v["S"].encode(), v["N"], v["r"], v["p"], v["dkLen"])
        assert got.hex() == v["out"]


def test_pbkdf2_vectors(orc, golden):
    for v in golden["kat_primitives"]["pbkdf2_sha256"]:
        assert orc.c_pbkdf2(v["P"].encode(), v["S"].encode(), v["c"], v["dkLen"]).hex() == v["out"]


def test_sha256_and_hmac_against_hashlib(orc):
    import hmac
    rng = np.random.default_rng(11)
    for n in [0, 1, 55, 56, 63, 64, 65, 119, 120, 127, 128, 1000]:
        m = bytes(rng.integers(0, 256, n, dtype=np.uint8))
        assert orc.c_sha256(m) == hashlib.sha256(m).digest()
        for klen in (0, 32, 64, 65, 200):
            k = bytes(rng.integers(0, 256, klen, dtype=np.uint8))
            assert orc.c_hmac_sha256(k, m) == hmac.new(k, m, "sha256").digest()


def test_blake3_against_wheel(orc):
    blake3 = pytest.importorskip("blake3")
    rng = np.random.default_rng(12)
    for n in [0, 1, 63, 64, 65, 1023, 1024, 1025, 2048, 2049, 3072, 3073, 4096, 5000, 8192, 8193, 31744, 100000]:
        m = bytes(rng.integers(0, 256, n, dtype=np.uint8))
        assert orc.c_blake3(m) == blake3.blake3(m).digest()
        assert orc.c_blake3(m, 131) == blake3.blake3(m).digest(131)


def test_aes128_fips197(orc, golden):
    for v in golden["kat_primitives"]["aes128"]:
        assert orc.c_aes128(bytes.fromhex(v["key"]), bytes.fromhex(v["pt"])).hex() == v["ct"]


def test_aes128_against_cryptography(orc):
    ciphers = pytest.importorskip("cryptography.hazmat.primitives.ciphers")
    rng = np.random.default_rng(13)
    for _ in range(32):
        k = bytes(rng.integers(0, 256, 16, dtype=np.uint8)); b = bytes(rng.integers(0, 256, 16, dtype=np.uint8))
        enc = ciphers.Cipher(ciphers.algorithms.AES(k), ciphers.modes.ECB()).encryptor()
        assert enc.update(b) == orc.c_aes128(k, b)


def test_vrf_difficulty_table(orc, golden):
    for n, hx in golden["vrf_difficulty"].items():
        assert orc.c_vrf_difficulty(int(n)).hex() == hx
        assert orc.py_vrf_difficulty(int(n)).hex() == hx
    assert orc.c_vrf_difficulty(1) == b"\xff" * 32 and orc.c_vrf_difficulty(0) == b"\xff" * 32


def test_real_vrf_nonces_of_the_reference_checkpoint_fixture(orc, golden):
    """THE PIN.  checkpoint/checkpointdata.json in the reference holds 42 identities of a LabelsPerUnit = 1024,
    N = 8192 network with their VRF nonces.  A VRF nonce is the index of the smallest label32 of the identity's POST,
    so label32(nonce) * numLabels / 2^256 is Exp(1)-distributed for the right label function (and ~numLabels/2 for a
    wrong one).  Checks the C oracle bit for bit against the committed values, and the statistics of the real data."""
    items = golden["checkpoint_vrf"]["items"]
    assert len(items) == 42
    below = 0
    for it in items:
        c = orc.c_commitment(bytes.fromhex(it["node_id"]), bytes.fromhex(it["commitment_atx"]))
        assert c.hex() == it["commitment"]
        l32 = orc.c_label32(c, it["vrf_nonce"], it["N"])
        assert l32.hex() == it["label32"]
        num_labels = it["num_units"] * it["labels_per_unit"]
        assert it["vrf_nonce"] < num_labels
        ratio = int.from_bytes(l32, "big") * num_labels / 2**256
        assert ratio < 8, "not an arg-min label: the label function is wrong"      # P(Exp(1) > 8) = 3e-4 per identity
        below += l32 < orc.py_vrf_difficulty(num_labels)
    assert 18 <= below <= 34          # 1 - 1/e = 63 % of 42 = 26.5 expected (observed: 26)


def test_real_vrf_nonce_is_the_minimum_of_the_whole_post(orc, golden):
    """Every label of one real identity's POST (33 units x 1024 labels, N = 8192) recomputed: the nonce recorded in the
    reference's checkpoint fixture is the index of the smallest one — although that label is ABOVE 2^256/numLabels
    (ratio 1.24), i.e. the network recorded the arg-min, not the first label under a threshold.  The committed file
    carries the same check for all 42 identities (1.9 M labels, oracle/gen_golden.py)."""
    items = golden["checkpoint_vrf"]["items"]
    assert all(it["vrf_nonce_is_argmin_of_whole_post"] for it in items)
    it = items[0]
    assert it["num_units"] == 33 and it["label32_times_num_labels_over_2p256"] > 1
    c = bytes.fromhex(it["commitment"])
    _, found, idx, l32 = orc.c_labels_range(c, it["N"], 0, it["num_units"] * it["labels_per_unit"], b"\xff" * 32,
                                            threads=orc.default_threads())
    assert found and idx == it["vrf_nonce"] and l32.hex() == it["label32"]


def test_keccak_chacha_pbkdf2_building_blocks(orc):
    """Keccak-f against hashlib's SHA3-512 (same permutation, pad byte 0x06); Keccak-512/HMAC/PBKDF2/ChaCha and the
    generic scrypt-jane against the numpy restatement."""
    rng = np.random.default_rng(21)
    for n in [0, 1, 71, 72, 73, 143, 144, 145, 500]:
        m = bytes(rng.integers(0, 256, n, dtype=np.uint8))
        assert orc.c_keccak512(m, 0x06) == hashlib.sha3_512(m).digest()
        assert orc.py_keccak512(m, 0x06) == hashlib.sha3_512(m).digest()
        assert orc.c_keccak512(m) == orc.py_keccak512(m)
        for klen in (0, 32, 72, 73, 200):
            k = bytes(rng.integers(0, 256, klen, dtype=np.uint8))
            assert orc.c_hmac_keccak512(k, m) == orc.py_hmac_keccak512(k, m)
        assert orc.c_pbkdf2_keccak512(m, m[::-1], 130) == orc.py_pbkdf2_keccak512(m, m[::-1], 130)
    for _ in range(8):
        blk = rng.integers(0, 2**32, 16, dtype=np.uint32)
        assert orc.c_chacha20_8(blk.astype("<u4").tobytes()) == orc.py_chacha20_8(blk[None, :])[0].astype("<u4").tobytes()
    for n in (2, 16, 256):
        pws = [bytes(rng.integers(0, 256, k, dtype=np.uint8)) for k in (0, 8, 72, 100)]
        salts = [bytes(rng.integers(0, 256, k, dtype=np.uint8)) for k in (0, 4, 64, 9)]
        exp = orc.py_scrypt_jane_batch(pws, salts, n, dklen=48)
        assert [orc.c_scrypt_jane(p, s, n, 1, 1, 48) for p, s in zip(pws, salts)] == exp


def test_survey_candidate_vectors(orc):
    """SURVEY.md §8c candidate inputs (activation/validation_test.go:35-36: zero node id and commitment ATX)."""
    c = orc.c_commitment(bytes(32), bytes(32))
    assert c.hex() == "4d006976636a8696d909a630a4081aad4d7c50f81afdee04020bf05086ab6a55"
    assert orc.c_label32(c, 0, 2).hex() == "502009eefb489466fd46f63685e0d1cec99c7821c0a92eb013efba9f2e805abc"
    assert orc.c_label32(c, 0, 8192).hex() == "13f053790cc908fd17c1ed054ad849d63a3abb394d07bb54872fe91b24c56f46"


def test_label_golden_vectors(orc, golden):
    for case in golden["labels"]["cases"]:
        c = orc.c_commitment(bytes.fromhex(case["node_id"]), bytes.fromhex(case["commitment_atx"]))
        assert c.hex() == case["commitment"], case["name"]
        diff = bytes.fromhex(case["vrf_difficulty"]) if "vrf_difficulty" in case else None
        labels, found, idx, l32 = orc.c_labels_range(c, case["N"], case["start"], case["count"], diff, threads=4)
        assert hashlib.sha256(labels.tobytes()).hexdigest() == case["labels_sha256"], case["name"]
        if "labels_hex" in case:
            assert labels.tobytes().hex() == case["labels_hex"], case["name"]
        if diff is not None:
            if case["vrf_index"] is None:
                assert not found
            else:
                assert found and idx == case["vrf_index"] and l32.hex() == case["vrf_label32"], case["name"]


def test_gather_golden_vectors(orc, golden):
    items = golden["gather"]["items"]
    for n in (2, 8192):
        sel = [it for it in items if it["N"] == n]
        comms = np.frombuffer(b"".join(bytes.fromhex(it["commitment"]) for it in sel), dtype=np.uint8).reshape(-1, 32)
        idx = np.array([it["index"] for it in sel], dtype=np.uint64)
        got = orc.c_labels_gather(comms, idx, n, threads=4)
        for row, it in zip(got, sel):
            assert row.tobytes().hex() == it["label32"][:32]


def test_threads_do_not_change_results(orc):
    c = orc.c_commitment(b"\x01" * 32, b"\x02" * 32)
    d = orc.py_vrf_difficulty(8)
    a = orc.c_labels_range(c, 16, 7, 301, d, threads=1)
    b = orc.c_labels_range(c, 16, 7, 301, d, threads=7)
    assert (a[0] == b[0]).all() and a[1:] == b[1:]


def test_vrf_scan_matches_python(orc):
    c = orc.c_commitment(b"\x07" * 32, b"\x09" * 32)
    for num_labels in (4, 64, 4096):
        d = orc.py_vrf_difficulty(num_labels)
        _, found, idx, l32 = orc.c_labels_range(c, 4, 100, 500, d, threads=3)
        pidx, pl32 = orc.py_vrf_scan(c, 4, 100, 500, d)
        assert (idx if found else None) == pidx and (l32 if found else None) == pl32


def test_bad_parameters_rejected(orc):
    c = bytes(32)
    for n in (0, 1, 3, 12):
        with pytest.raises(ValueError):
            orc.c_labels_range(c, n, 0, 4)
    labels, found, _, _ = orc.c_labels_range(c, 2, 0, 0)
    assert labels.shape == (0, 16) and not found


# (labels, nonces, k1, num_labels, k2, first_index, proof expected): difficulty MSB noted per row
PROVE_REGIMES = {
    "msb0-lsb":    (400, 64, 4000, 1 << 20, 2, 0, True),           # 0x00, lsb != 0: every hit is a lazy-cipher hit
    "round":       (300, 16, 1 << 15, 1 << 20, 4, 0, True),        # 0x08, lsb == 0: a byte equal to the MSB never passes
    "mid-lsb":     (300, 32, 100003, 1 << 20, 6, 0, True),         # 0x18, lsb != 0
    "saturated":   (64, 16, 300, 300, 5, 0, True),                 # 0xff: k1 >= num_labels
    "no-proof":    (300, 16, 4000, 1 << 20, 10, 0, False),
    "k2-1-ties":   (40, 256, 1 << 19, 1 << 20, 1, 0, True),        # 0x80: ~128 nonces tie at the first label
    "first-index": (600, 64, 2**32 - 1, 1 << 41, 2, 2**40 + 3, True),   # 0x00, lsb != 0, 42-bit indices
}


@pytest.mark.parametrize("regime", PROVE_REGIMES)
def test_vectorised_prove_oracle_matches_scalar(orc, regime):
    """np_prove_multi (the GPU prove tests' oracle) is the scalar py_prove_multi: same winner, same indices, at every
    difficulty regime, ties and an offset first index included."""
    count, nonces, k1, num_labels, k2, first, found = PROVE_REGIMES[regime]
    rng = np.random.default_rng(sorted(PROVE_REGIMES).index(regime) + 100)
    labels = rng.integers(0, 256, (count, 16), dtype=np.uint8)
    challenge = bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    pows = [int(p) for p in rng.integers(0, 2**56, nonces // 16)]
    exp_nonce, exp_hits = orc.py_prove_multi(labels, challenge, nonces, pows, k1, k2, num_labels)
    assert (exp_nonce is not None) == found
    want = (exp_nonce, None if exp_hits is None else [first + i for i in exp_hits])
    assert orc.np_prove_multi(labels, challenge, nonces, pows, k1, k2, num_labels, first_index=first) == want
    if regime == "k2-1-ties":
        hits = orc.np_prove_hits(labels, challenge, nonces, pows, k1, k2, num_labels)
        assert exp_hits == [0] and sum(1 for h in hits.values() if list(h) == [0]) > 1


def _plain_subset(values, msg: bytes, stream_len: int):
    """Partial Fisher-Yates over one fixed XOF stream, read with bounds checks: the whole shuffle, and the bytes used."""
    import blake3
    stream = blake3.blake3(msg).digest(stream_len)
    vals, where, pos, out = list(values), list(range(len(values))), 0, []
    for idx in range(len(vals)):
        remaining = len(vals) - idx
        while True:
            assert pos + 2 <= len(stream), "fixed reference stream too short"
            r = int.from_bytes(stream[pos:pos + 2], "little")
            pos += 2
            if r < 0xFFFF - 0xFFFF % remaining:
                break
        j = idx + r % remaining
        vals[idx], vals[j] = vals[j], vals[idx]
        where[idx], where[j] = where[j], where[idx]
        out.append((vals[idx], where[idx]))
    return out, pos


def test_subset_positions_grow_the_stream(orc):
    """Subset selection with up to k2 = 65535 draws: the stream py_subset_positions grows on demand gives the same
    selections as one drawn 64 KiB up front and as a plain shuffle over a fixed 1 MiB stream, every prefix of the
    selection order is the selection for a smaller k3, and no position is selected twice."""
    rng = np.random.default_rng(41)
    k2 = 65535
    values = [int(v) for v in rng.integers(0, 2**34, k2)]
    seed, nonce, packed, pow_ = b"peer", 77, bytes(rng.integers(0, 256, 40, dtype=np.uint8)), 2**50 + 9
    full = orc.py_subset_positions(values, seed, nonce, packed, pow_, k2, with_positions=True)
    assert len(full) == k2 and len({w for _, w in full}) == k2
    assert all(values[w] == v for v, w in full)
    assert orc.py_subset_positions(values, seed, nonce, packed, pow_, k2, with_positions=True, stream_bytes=1 << 16) == full
    plain, used = _plain_subset(values, seed + nonce.to_bytes(4, "little") + packed + pow_.to_bytes(8, "little"), 1 << 20)
    assert plain == full
    assert used > 2 * 8192          # well past the fixed 8 KiB stream the oracle used to stop at
    for k in (1, 127, 128, 129, 300, 4095, 4096, 4097, 20000, 40000, 65534):
        assert orc.py_subset_positions(values, seed, nonce, packed, pow_, k, with_positions=True) == full[:k], k


def test_simd_and_scalar_romix_agree(orc):
    """The vectorised ROMix paths used for the timed CPU baseline (1 = SSE2, 2 = AVX2 with two labels per thread in
    lock-step, 3 = AVX-512 with four, where the CPU has it) are the same function as the scalar restatement, ragged
    counts and the VRF scan included."""
    L = orc.lib()
    default = L.oracle_get_impl()
    try:
        rng = np.random.default_rng(31)
        for n in (2, 4, 64, 1024, 8192):
            c = bytes(rng.integers(0, 256, 32, dtype=np.uint8))
            d = orc.py_vrf_difficulty(8)
            L.oracle_set_impl(0)
            a = orc.c_labels_range(c, n, 2**32 - 3, 27, d, threads=2)
            comms = rng.integers(0, 256, (11, 32), dtype=np.uint8); idx = rng.integers(0, 2**40, 11, dtype=np.uint64)
            ga = orc.c_labels_gather(comms, idx, n, threads=2)
            for impl in (1, 2, 3):
                if L.oracle_set_impl(impl) != 0:
                    continue
                b = orc.c_labels_range(c, n, 2**32 - 3, 27, d, threads=2)
                assert (a[0] == b[0]).all() and a[1:] == b[1:], (n, impl)
                assert (orc.c_labels_gather(comms, idx, n, threads=2) == ga).all(), (n, impl)
    finally:
        L.oracle_set_impl(default)
