"""GPU tier: PoET registration PoW search (SURVEY.md §8f.4) against a hashlib restatement of
shared.FindSubmitPowNonce (ASSUMED: SHA-256(powChallenge || nodeID || poetChallenge || LE64(nonce)), leading zero bits)."""
import hashlib
import importlib
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _leading_zero_bits(h: bytes) -> int:
    v = int.from_bytes(h, "big")
    return 256 - v.bit_length()


def _cpu_find(pc, ch, nid, difficulty, start=0, limit=1 << 22):
    for nonce in range(start, start + limit):
        if _leading_zero_bits(hashlib.sha256(pc + nid + ch + nonce.to_bytes(8, "little")).digest()) >= difficulty:
            return nonce
    return None


def _layouts():
    """(pc_len, ch_len) for every prefix length pc_len + 32 + ch_len that is 0, 4, ..., 60 modulo 64, each with the
    smallest prefix that leaves the tail without a full block ahead of it (none below 64 for residues under 32) and one
    block longer.  The kernel hashes a host midstate over the full blocks, then 1 or 2 tail blocks with the nonce at
    word (prefix mod 64) / 4; residue 0 puts the nonce at the start of the tail, residues 48..60 push the padding into
    a second tail block, and residue 60 splits the nonce across the two."""
    out = []
    for r in range(0, 64, 4):
        lo = r if r >= 32 else r + 64
        for prefix in (lo, lo + 64):
            rest = prefix - 32
            pc_len = (rest // 3) | 1 if rest else 0        # odd, so that neither half alone is word aligned
            out.append((pc_len, rest - pc_len))
    return out


def test_lowest_nonce_matches_sequential_search(b2, gpu_ready):
    poet = importlib.import_module("go-spacemesh_b200.poet")
    rng = np.random.default_rng(4)
    cases = [(32, 32, 12), (32, 32, 16), (16, 4, 10), (0, 0, 8), (32, 60, 14)]
    cases += [(pc_len, ch_len, d) for pc_len, ch_len in _layouts() for d in (0, 9)]
    for pc_len, ch_len, difficulty in cases:
        pc, ch, nid = (bytes(rng.integers(0, 256, n, dtype=np.uint8)) for n in (pc_len, ch_len, 32))
        for start in (0, 2**32 - 1000, 2**60):
            nonce, hashes = poet.find_submit_pow_nonce(pc, ch, nid, difficulty, start_nonce=start)
            assert nonce == _cpu_find(pc, ch, nid, difficulty, start), (pc_len, ch_len, difficulty, start)
            if difficulty == 0:
                assert nonce == start
            assert _leading_zero_bits(poet.pow_hash(pc, ch, nid, nonce)) >= difficulty
            assert poet.pow_hash(pc, ch, nid, nonce) == hashlib.sha256(pc + nid + ch + nonce.to_bytes(8, "little")).digest()


def test_prefix_not_word_aligned_is_refused(b2, gpu_ready):
    """The nonce must start on a 32-bit word of the SHA-256 block: pc_len + ch_len must be a multiple of 4."""
    poet = importlib.import_module("go-spacemesh_b200.poet")
    for pc_len, ch_len in ((1, 0), (3, 2), (32, 31), (33, 32), (0, 62)):
        with pytest.raises(b2.B200PostError) as e:
            poet.find_submit_pow_nonce(b"\x01" * pc_len, b"\x02" * ch_len, b"\x03" * 32, 4, max_nonces=1 << 10)
        assert e.value.code == b2.ERR_INVALID_ARGUMENT


def test_window_without_solution_and_rate(b2, gpu_ready):
    poet = importlib.import_module("go-spacemesh_b200.poet")
    pc, ch, nid = b"\x01" * 32, b"\x02" * 32, b"\x03" * 32
    with pytest.raises(b2.B200PostError) as e:
        poet.find_submit_pow_nonce(pc, ch, nid, 200, max_nonces=1 << 20)
    assert e.value.code == b2.ERR_INVALID_PROOF
    t0 = time.perf_counter()
    nonce, hashes = poet.find_submit_pow_nonce(pc, ch, nid, 34)            # ~2^34 candidates expected
    dt = time.perf_counter() - t0
    assert _leading_zero_bits(poet.pow_hash(pc, ch, nid, nonce)) >= 34
    print(f"poet pow: difficulty 34 solved at nonce {nonce} after {hashes} candidates in {dt:.2f} s = {hashes / dt / 1e9:.2f} GH/s")
