"""GPU tier: the proving scan (K6a prove_scan_kernel + K6b prove_lazy_kernel) and the verifier's AES verdict (K5
verify_judge_kernel) against the vectorised oracle (oracle/pyoracle.py np_prove_multi), exactly: nonce, indices, pow.

Difficulty regimes, by the top byte (MSB) of the proving difficulty:
* MSB 0 with a non-zero lsb, the mainnet regime (K1 = 26 over >= 2^32 labels): no byte is below the MSB, so every
  hit is a byte equal to it and goes through the candidate queue and the nonce's lazy cipher;
* round (lsb 0): a byte equal to the MSB never passes;
* mid, with a non-zero lsb;
* saturated (K1 >= num_labels, MSB 0xff): every byte is at or below the MSB.

`b200post_prove_scan` runs over synthetic labels in host memory (the scan does not care where labels come from),
`b200post_generate_proof` over a real POST whose files hold an odd number of labels, at chunk sizes that put chunk
seams everywhere.  Every oracle proof is then checked by the GPU verifier, tampered and untampered."""
import importlib
import re
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NL22, NL41 = 1 << 22, 1 << 41                  # 23- and 42-bit indices
DIFF = {                                       # regime: (k1, num_labels)
    # MSB 0 with lsb ~ 2^55: half of the labels whose byte is 0 pass the lazy cipher, so a wrong lazy key shows
    "msb0": (2**13 + 5, NL22),                 # 0x00, lsb != 0: a label passes with p ~ 1/512
    "msb0-42": (2**32 - 1, NL41),              # 0x00, lsb != 0: p ~ 1/512
    "round": (1 << 17, NL22),                  # 0x08, lsb 0
    "mid": (1234567, NL22),                    # 0x4b, lsb != 0
    "sat": (NL22, NL22),                       # 0xff
}
# (id, count, first_index, nonces, regime, k2).  Saturated runs only at small counts with <= 32 nonces, and hits per
# call stay under the 4 M-entry hit buffer.  Every case has a proof; the seed of a case is its position here.
SCAN_CASES = [
    ("1-sat", 1, 0, 16, "sat", 1),
    ("1-mid", 1, 0, 32, "mid", 1),
    ("31-sat", 31, 0, 32, "sat", 31),
    ("31-mid", 31, 0, 288, "mid", 12),
    ("33-sat", 33, 0, 16, "sat", 20),
    ("33-round", 33, 0, 4096, "round", 3),
    ("33-msb0", 33, 0, 4096, "msb0", 1),
    ("33-across-2^32", 33, 2**32 - 7, 288, "msb0-42", 1),
    ("4095-msb0", 4095, 0, 288, "msb0", 15),
    ("4095-round", 4095, 0, 32, "round", 140),
    ("4095-mid", 4095, 0, 16, "mid", 200),
    ("4095-msb0-4096n", 4095, 0, 4096, "msb0", 19),
    ("4095-across-2^32", 4095, 2**32 - 7, 16, "msb0-42", 9),
    ("4095-at-2^40", 4095, 2**40, 288, "msb0-42", 14),
    ("2^18-at-2^40-4096n", 1 << 18, 2**40, 4096, "msb0-42", 150),
    ("2^18-round", 1 << 18, 0, 288, "round", 278),
]


@pytest.fixture(scope="module")
def mods(b2, gpu_ready):
    return importlib.import_module("go-spacemesh_b200.prove"), importlib.import_module("go-spacemesh_b200.verify")


@pytest.fixture(scope="module")
def host_labels():
    return np.random.default_rng(2026).integers(0, 256, (NL22 + 4097, 16), dtype=np.uint8)


def _inputs(seed: int, nonces: int):
    """A challenge and one random 56-bit pow per nonce group, so that every group key differs."""
    r = np.random.default_rng(seed)
    return bytes(r.integers(0, 256, 32, dtype=np.uint8)), [int(p) for p in r.integers(0, 2**56, nonces // 16)]


def _scanned_total(b2) -> int:
    return int(re.search(r"^b200post_prove_labels_scanned_total (\S+)$", b2.metrics_text(), re.M).group(1))


def _check_scan(b2, mods, labels, first, challenge, nonces, pows, k1, k2, num_labels, expect):
    """prove_scan must return the oracle's (nonce, indices) with the pow of the nonce's group; labels_scanned and the
    metric count labels streamed from first_index, not an absolute position."""
    pr, vf = mods
    before = _scanned_total(b2)
    nonce, packed, pow_, scanned = pr.prove_scan(labels, challenge, nonces, pows, k1, k2, num_labels, first_index=first)
    bits = vf.bits_per_index(num_labels)
    assert len(packed) == (k2 * bits + 7) // 8
    assert (nonce, vf.unpack_indices(packed, bits, k2)) == expect
    assert pow_ == pows[nonce // 16]
    assert expect[1][-1] - first < scanned <= len(labels)
    assert _scanned_total(b2) - before == scanned
    return packed


@pytest.mark.parametrize("case", SCAN_CASES, ids=[c[0] for c in SCAN_CASES])
def test_prove_scan_matches_oracle(mods, b2, orc, host_labels, case):
    _, count, first, nonces, regime, k2 = case
    k1, num_labels = DIFF[regime]
    challenge, pows = _inputs(SCAN_CASES.index(case), nonces)
    labels = host_labels[:count]
    expect = orc.np_prove_multi(labels, challenge, nonces, pows, k1, k2, num_labels, first_index=first)
    assert expect[0] is not None
    _check_scan(b2, mods, labels, first, challenge, nonces, pows, k1, k2, num_labels, expect)


def test_two_chunk_scan_decided_in_the_ragged_chunk(mods, b2, orc, host_labels):
    """2^22 + 4097 labels are two chunks, so both streams run and share the candidate queue.  Mainnet K1 = 26 (MSB 0).
    One hit label of the nonce with the most first-chunk hits is copied into the second chunk, and K2 is one more
    than that count: no nonce completes in the first chunk, and the proof needs hits from both."""
    count, nonces, k1 = NL22 + 4097, 16, 26
    labels = host_labels[:count].copy()
    challenge, pows = _inputs(100, nonces)
    first_chunk = orc.np_prove_hits(labels[:NL22], challenge, nonces, pows, k1, NL22, NL22)
    lead = max(first_chunk, key=lambda n: len(first_chunk[n]))
    k2 = len(first_chunk[lead]) + 1
    labels[NL22 + 4000] = labels[first_chunk[lead][0]]
    expect = orc.np_prove_multi(labels, challenge, nonces, pows, k1, k2, NL22)
    assert expect[0] is not None and expect[1][0] < NL22 <= expect[1][-1]
    _check_scan(b2, mods, labels, 0, challenge, nonces, pows, k1, k2, NL22, expect)


@pytest.mark.parametrize("k2", [1, 2])
def test_ties_go_to_the_lower_nonce(mods, b2, orc, host_labels, k2):
    """MSB 0x4b and 4096 nonces over 64 labels: many nonces reach their K2-th hit at the same label."""
    count, nonces = 64, 4096
    k1, num_labels = DIFF["mid"]
    challenge, pows = _inputs(200 + k2, nonces)
    labels = host_labels[:count]
    hits = orc.np_prove_hits(labels, challenge, nonces, pows, k1, k2, num_labels)
    expect = orc.np_prove_multi(labels, challenge, nonces, pows, k1, k2, num_labels)
    tied = [n for n, h in hits.items() if len(h) == k2 and h[-1] == expect[1][-1]]
    assert len(tied) > 1 and expect[0] == tied[0]
    _check_scan(b2, mods, labels, 0, challenge, nonces, pows, k1, k2, num_labels, expect)


def test_wire_cap(mods, b2, orc, host_labels):
    """With 23-bit indices, 278 of them pack to exactly 800 bytes; 279 need 803 and must be refused, not truncated."""
    pr, _ = mods
    count, nonces = 4095, 16
    k1, num_labels = DIFF["mid"]
    challenge, pows = _inputs(300, nonces)
    labels = host_labels[:count]
    expect = orc.np_prove_multi(labels, challenge, nonces, pows, k1, 278, num_labels)
    assert expect[0] is not None
    assert len(_check_scan(b2, mods, labels, 0, challenge, nonces, pows, k1, 278, num_labels, expect)) == 800
    assert orc.np_prove_multi(labels, challenge, nonces, pows, k1, 279, num_labels)[0] is not None
    with pytest.raises(b2.B200PostError) as e:
        pr.prove_scan(labels, challenge, nonces, pows, k1, 279, num_labels)
    assert e.value.code == b2.ERR_INVALID_ARGUMENT and "wire cap" in str(e.value)


def test_no_proof(mods, b2, orc, host_labels):
    pr, _ = mods
    count, nonces, k2 = 4095, 16, 278
    k1, num_labels = DIFF["msb0"]
    challenge, pows = _inputs(400, nonces)
    labels = host_labels[:count]
    assert orc.np_prove_multi(labels, challenge, nonces, pows, k1, k2, num_labels) == (None, None)
    with pytest.raises(b2.B200PostError) as e:
        pr.prove_scan(labels, challenge, nonces, pows, k1, k2, num_labels)
    assert e.value.code == b2.ERR_INVALID_PROOF and "no proof found" in str(e.value)


def test_hit_buffer_overflow_is_an_error_return(mods, b2, orc, host_labels):
    """Saturated difficulty, 2^20 labels, 64 nonces: 2^26 hits against a buffer of at most 2^22 entries.  The call must
    fail cleanly, never return a proof built from a truncated hit list, and leave the device usable."""
    pr, _ = mods
    k1, num_labels = DIFF["sat"]
    challenge, pows = _inputs(500, 64)
    with pytest.raises(b2.B200PostError) as e:
        pr.prove_scan(host_labels[:1 << 20], challenge, 64, pows, k1, 37, num_labels)
    assert e.value.code == b2.ERR_OUT_OF_MEMORY and "hit buffer overflow" in str(e.value)
    challenge, pows = _inputs(501, 16)
    expect = orc.np_prove_multi(host_labels[:33], challenge, 16, pows, k1, 20, num_labels)
    _check_scan(b2, mods, host_labels[:33], 0, challenge, 16, pows, k1, 20, num_labels, expect)


# ------------------------------------------------------------------------------------- generate_proof over a real POST
NODE, ATX = bytes(range(50, 82)), bytes(range(150, 182))
UNITS, LPU = 4, 1 << 20
NUM_LABELS = UNITS * LPU
PER_FILE = 1_000_003                         # labels per postdata_N.bin: odd, and the fifth file is partial
PROOF_REGIMES = {                            # regime: (k1, k2, nonces, challenge)
    "mainnet": (26, 37, 288, bytes(range(90, 122))),     # MSB 0, lsb != 0; the winner's 37th hit is past 3 M
    "round": (1 << 17, 200, 16, bytes(range(1, 33))),    # MSB 0x08, lsb 0
    "mid": (100003, 200, 16, bytes(range(2, 34))),       # MSB 0x06, lsb != 0
}
CHUNKS = (0, (1 << 20) + 13, 4099)           # 0 = one 2^22-label chunk; 4099 crosses every file seam mid-chunk


def _pow_of(group: int) -> int:
    return 2**55 + 977 * group


def _pow_callback(ctx, nonce_group, challenge8, difficulty, node_id, pow_out):
    pow_out[0] = _pow_of(nonce_group)
    return 0


@pytest.fixture(scope="module")
def post(b2, gpu_ready, tmp_path_factory):
    """4 units x 2^20 labels at N = 2, in five files; returns (setup module, data dir, the labels read back)."""
    su = importlib.import_module("go-spacemesh_b200.setup")
    mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=LPU, k1=26, k2=37, k3=37, max_num_units=8))
    o = su.PostSetupOpts(data_dir=str(tmp_path_factory.mktemp("post")), num_units=UNITS, max_file_size=16 * PER_FILE,
                         provider_id=0, scrypt_n=2, compute_batch_size=1 << 20)
    mgr.prepare_initializer(o, NODE, ATX)
    mgr.start_session()
    assert mgr.status().state == su.STATE_COMPLETE
    files = [Path(o.data_dir) / f"postdata_{i}.bin" for i in range(5)]
    assert [f.stat().st_size for f in files] == [16 * PER_FILE] * 4 + [16 * (NUM_LABELS - 4 * PER_FILE)]
    assert not (Path(o.data_dir) / "postdata_5.bin").exists()
    labels = np.concatenate([np.fromfile(f, dtype=np.uint8) for f in files]).reshape(-1, 16)
    return su, o.data_dir, labels


@pytest.fixture(scope="module")
def oracle_proof(post, orc, mods):
    """regime -> the oracle's proof (vf.Proof, indices), computed once: the answer does not depend on the chunk size."""
    _, vf = mods
    labels, cache = post[2], {}

    def get(regime):
        if regime not in cache:
            k1, k2, nonces, challenge = PROOF_REGIMES[regime]
            nonce, idx = orc.np_prove_multi(labels, challenge, nonces, [_pow_of(g) for g in range(nonces // 16)], k1, k2,
                                            NUM_LABELS)
            assert nonce is not None
            cache[regime] = (vf.Proof(nonce, vf.pack_indices(idx, vf.bits_per_index(NUM_LABELS)), _pow_of(nonce // 16)), idx)
        return cache[regime]
    return get


@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("regime", PROOF_REGIMES)
def test_generate_proof_matches_oracle(mods, post, oracle_proof, regime, chunk):
    pr, vf = mods
    su, data_dir, _ = post
    k1, k2, nonces, challenge = PROOF_REGIMES[regime]
    cfg = su.PostConfig(labels_per_unit=LPU, k1=k1, k2=k2, k3=k2, max_num_units=8)
    proof, meta, scanned = pr.generate_proof(data_dir, challenge, cfg, nonces=nonces, chunk_labels=chunk, pow=_pow_callback)
    want, idx = oracle_proof(regime)
    assert proof == want
    assert idx[-1] < scanned <= NUM_LABELS
    assert meta == vf.ProofMetadata(NODE, ATX, challenge, UNITS, LPU)


def _verify_args(vf, regime):
    k1, k2, _, challenge = PROOF_REGIMES[regime]
    return vf.ProofMetadata(NODE, ATX, challenge, UNITS, LPU), vf.VerifyParams(k1=k1, k2=k2, scrypt_n=2)


def _py_verdict(orc, proof, meta, params, **kw):
    return orc.py_verify(proof.nonce, proof.indices, proof.pow, NODE, ATX, meta.challenge, UNITS, LPU, params.k1, params.k2,
                         params.scrypt_n, **kw)


@pytest.mark.parametrize("regime", PROOF_REGIMES)
def test_gpu_verifier_accepts_the_oracle_proof(mods, b2, orc, oracle_proof, regime):
    _, vf = mods
    proof, _ = oracle_proof(regime)
    meta, params = _verify_args(vf, regime)
    k2 = params.k2
    assert _py_verdict(orc, proof, meta, params) == (True, None)
    v = vf.PostVerifier(pow="skip")
    try:
        v.verify(proof, meta, params)
        for k3, seed in ((1, b""), (5, b"peer-A"), (k2, b"peer-B" * 3)):
            v.verify(proof, meta, params, mode=vf.MODE_SUBSET, k3=k3, seed=seed)
        for pos in range(k2):
            v.verify(proof, meta, params, mode=vf.MODE_SELECTED_INDEX, selected_index=pos)
    finally:
        v.close()
    options = [{}] + [dict(mode=vf.MODE_SELECTED_INDEX, selected_index=pos) for pos in range(k2)]
    st, _ = vf.verify_batch([proof] * len(options), [meta] * len(options), params, options=options, pow="skip")
    assert st == [b2.OK] * len(options)


@pytest.mark.parametrize("regime", PROOF_REGIMES)
def test_tampered_proof_verdicts_match_oracle(mods, b2, orc, oracle_proof, regime):
    """Indices[pos] += 1 at several positions (and at two at once): in ALL mode, and in SELECTED_INDEX mode at the
    tampered and an untouched position, the GPU verdict and failing position equal py_verify's, through verify_batch
    and through PostVerifier."""
    _, vf = mods
    proof, idx = oracle_proof(regime)
    meta, params = _verify_args(vf, regime)
    k2, bits = params.k2, vf.bits_per_index(NUM_LABELS)
    positions = [[0], [1], [k2 // 2], [k2 - 2], [k2 - 1], [3, k2 - 3]]
    calls = []                                           # (proof, options, oracle keyword arguments)
    for bumped in positions:
        bad = list(idx)
        for pos in bumped:
            bad[pos] = (bad[pos] + 1) % NUM_LABELS
        t = vf.Proof(proof.nonce, vf.pack_indices(bad, bits), proof.pow)
        calls.append((t, {}, {}))
        for pos in (bumped[-1], (bumped[-1] + 1) % k2):
            calls.append((t, dict(mode=vf.MODE_SELECTED_INDEX, selected_index=pos), dict(mode="selected", selected=pos)))
    expect = [_py_verdict(orc, t, meta, params, **kw) for t, _, kw in calls]
    assert any(ok for ok, _ in expect) and sum(not ok for ok, _ in expect) >= len(positions)

    st, bad_pos = vf.verify_batch([t for t, _, _ in calls], [meta] * len(calls), params, options=[o for _, o, _ in calls],
                                  pow="skip")
    assert set(st) <= {b2.OK, b2.ERR_INVALID_PROOF}
    assert [(s == b2.OK, None if s == b2.OK else b) for s, b in zip(st, bad_pos)] == expect

    v = vf.PostVerifier(pow="skip")
    try:
        got = []
        for t, o, _ in calls:
            try:
                v.verify(t, meta, params, **o)
                got.append((True, None))
            except vf.ErrInvalidIndex as e:
                got.append((False, e.index))
    finally:
        v.close()
    assert got == expect
