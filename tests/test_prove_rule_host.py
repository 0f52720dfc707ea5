"""CPU tier: the proving rule (csrc/prove_rule.cpp) driven chunk by chunk through tests/prove_rule_emul.cpp, no device.

* One shard: every pass gives window_oracle.pass_model's proof and reads as many labels, for windows-per-pass 1, 2, 3,
  w and w + 1.
* Two and three shards, chunks folded round-robin in either shard order or shard by shard from the last: the one-shard
  proof, including a tie across shards (the lower nonce wins) and shards that saturate on their own.
* Checked, with a recheck that reports a chosen set of labels damaged: the brute-force proof over usable hits, winner
  rounds <= 1 + damaged hits met, and one round of K2 labels on clean data.
* Unchecked: no round and no recheck, ever."""
import ctypes
import random
import subprocess
from pathlib import Path

import numpy as np
import pytest

import window_oracle as wo

ROOT = Path(__file__).resolve().parent.parent
U64P = ctypes.POINTER(ctypes.c_uint64)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    """csrc/prove_rule.cpp (plain C++17) compiled on its own with the emulation shim."""
    out = tmp_path_factory.mktemp("prove_rule") / "prove_rule_emul.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", str(out), str(ROOT / "tests" / "prove_rule_emul.cpp"),
                    str(ROOT / "go-spacemesh_b200" / "csrc" / "prove_rule.cpp")], check=True)
    L = ctypes.CDLL(str(out))
    L.emul_pass.argtypes = [ctypes.c_uint32, U64P, ctypes.c_uint64, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32,
                            ctypes.c_uint32, ctypes.c_uint32, ctypes.POINTER(ctypes.c_uint32), U64P, ctypes.c_uint64,
                            ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_uint32), U64P, U64P]
    return L


def run_pass(L, hits, bounds, chunk, first, window, windows, k2, order=0, damaged=None):
    """One pass over the nonces [first, first + window * windows) of hits {nonce: indices}, shard s = [bounds[s],
    bounds[s + 1]).  -> (proof (nonce, indices) or None, labels scanned, labels rechecked, rounds, damaged hits met)."""
    pairs = sorted((int(i), x) for x in range(first, first + window * windows) for i in hits.get(x, ()))
    idx = np.array([p[0] for p in pairs], dtype=np.uint64)
    nonces = np.array([p[1] for p in pairs], dtype=np.uint32)
    b = np.array(bounds, dtype=np.uint64)
    dmg = None if damaged is None else np.ascontiguousarray(damaged, dtype=np.uint8)
    nonce, ind, stats = ctypes.c_uint32(), (ctypes.c_uint64 * k2)(), (ctypes.c_uint64 * 4)()
    have = L.emul_pass(len(bounds) - 1, b.ctypes.data_as(U64P), chunk, order, first, window, windows, k2,
                       nonces.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), idx.ctypes.data_as(U64P), len(pairs),
                       None if dmg is None else dmg.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), ctypes.byref(nonce), ind, stats)
    assert have in (0, 1), have
    return ((nonce.value, list(ind)) if have else None), *stats


def windowed(L, hits, n, windows, per_pass, k2, bounds, chunk, order=0, damaged=None):
    """Passes of per_pass windows from window 0 until one has a proof, as generate() runs them.
    -> ((window, proof) or None, labels read, labels rechecked, rounds, damaged hits met, passes)."""
    total, passes, a = np.zeros(4, dtype=np.int64), 0, 0
    while a < windows:
        m = min(per_pass, windows - a)
        proof, *stats = run_pass(L, hits, bounds, chunk, a * n, n, m, k2, order, damaged)
        total += stats
        passes += 1
        if proof:
            return (proof[0] // n, proof), *total.tolist(), passes
        a += m
    return None, *total.tolist(), passes


def split_shards(total, chunk, n):
    """prover.cu's split: contiguous shards of whole chunks, the earlier ones taking the odd chunks."""
    chunks = (total + chunk - 1) // chunk
    q, r = divmod(chunks, n)
    starts = [min(total, (s * q + min(s, r)) * chunk) for s in range(n)]
    return starts + [total]


def patterns(seed, trials, dense=False, hole=False):
    """test_prove_windows_host's random hit patterns.  dense: enough hits that shards saturate; hole: the last nonce of
    every window has none, so that no shard can saturate."""
    r = random.Random(seed)
    for _ in range(trials):
        n, windows, k2 = 16 * r.choice((1, 2)), r.randint(1, 9), r.randint(1, 4)
        n_labels, chunk = r.randint(20, 300), r.randint(1, 64)
        rate = r.uniform(0.05, 0.2) if dense else r.uniform(0.002, 0.03)
        hits = {x: sorted(r.sample(range(n_labels), min(n_labels, int(rate * n_labels) + r.randint(0, 2))))
                for x in range(n * windows)}
        if hole:
            for w in range(windows):
                hits[w * n + n - 1] = []
        yield r, n, windows, k2, n_labels, chunk, hits


def saturates(hits, bounds, s, first, nonces, k2):
    return all(sum(bounds[s] <= i < bounds[s + 1] for i in hits[x]) >= k2 for x in range(first, first + nonces))


# ------------------------------------------------------------------------------------------------------------ one shard
def test_one_shard_is_the_pass_model(emul):
    for trial, (r, n, windows, k2, n_labels, chunk, hits) in enumerate(patterns(3, 300)):
        for m in (1, 2, 3, windows, windows + 1):
            a = 0
            while a < windows:
                mm = min(m, windows - a)
                proof, scanned, rechecked, rounds, _ = run_pass(emul, hits, [0, n_labels], chunk, a * n, n, mm, k2)
                assert (proof, scanned) == wo.pass_model(hits, n_labels, chunk, a, n, mm, k2), (trial, m, a)
                assert rechecked == rounds == 0
                if proof:
                    break
                a += mm


# -------------------------------------------------------------------------------------------------------- several shards
@pytest.mark.parametrize("dense", [False, True])
def test_shards_give_the_one_shard_proof(emul, dense):
    saturated = 0
    for trial, (r, n, windows, k2, n_labels, chunk, hits) in enumerate(patterns(11 + dense, 150, dense=dense)):
        m = r.choice((1, 2, windows))
        want = windowed(emul, hits, n, windows, m, k2, [0, n_labels], chunk)[0]
        for shards in (2, 3):
            bounds = split_shards(n_labels, chunk, shards)
            saturated += any(saturates(hits, bounds, s, 0, n * min(m, windows), k2) for s in range(1, shards))
            for order in (0, 1, 2):
                got, _, rechecked, rounds, _, _ = windowed(emul, hits, n, windows, m, k2, bounds, chunk, order)
                assert got == want, (trial, shards, order)
                assert rechecked == rounds == 0
    if dense:
        assert saturated > 50   # the dense patterns do make shards past the first saturate on their own


def test_tie_across_shards_goes_to_the_lower_nonce(emul):
    """Nonces 4 and 9 both have their K2-th hit at label 45, each with hits in all three shards; nonce 12's K2-th lies
    later.  Every fold order, chunk size and windows-per-pass gives nonce 4."""
    hits = {4: [15, 35, 45], 9: [5, 25, 45], 12: [1, 2, 50]}
    for chunk in (1, 5, 10, 20):
        for order in (0, 1, 2):
            for bounds in ([0, 60], [0, 20, 40, 60], [0, 40, 60]):
                proof = run_pass(emul, hits, bounds, chunk, 0, 16, 1, 3, order)[0]
                assert proof == (4, [15, 35, 45]), (chunk, order, bounds)
            assert windowed(emul, {x + 16: v for x, v in hits.items()}, 16, 2, 2, 3, [0, 20, 40, 60], chunk, order)[0] == \
                (1, (20, [15, 35, 45]))


# --------------------------------------------------------------------------------------------------------------- checked
def usable_proof(hits, damaged, n, windows, k2):
    """Brute force: the lowest window with a nonce of K2 usable hits, the lowest K2-th index, the lower nonce on ties."""
    for w in range(windows):
        best = wo.pick({x: hits[x] for x in range(w * n, (w + 1) * n)}, k2, usable=~damaged.astype(bool))
        if best:
            return w, best
    return None


@pytest.mark.parametrize("hole", [True, False])
def test_checked_proof_over_usable_hits(emul, hole):
    for trial, (r, n, windows, k2, n_labels, chunk, hits) in enumerate(patterns(21 + hole, 200, dense=not hole, hole=hole)):
        damaged = np.zeros(n_labels, dtype=np.uint8)
        damaged[r.sample(range(n_labels), int(r.uniform(0, 0.3) * n_labels))] = 1
        want = usable_proof(hits, damaged, n, windows, k2)
        m = r.choice((1, 2, windows))
        for shards in (1, 2, 3):
            bounds = split_shards(n_labels, chunk, shards)
            for order in (0, 1, 2) if shards > 1 else (0,):
                got, _, rechecked, rounds, bad, passes = windowed(emul, hits, n, windows, m, k2, bounds, chunk, order, damaged)
                assert got == want, (trial, shards, order)
                # each round ends the decision or drops a damaged hit; a shard's own saturation adds one round per pass
                assert rounds <= 1 + bad + (0 if hole else shards * passes), (trial, shards, order)
                assert rechecked >= rounds


def test_checked_on_clean_data_is_one_round_of_k2(emul):
    """No shard can saturate (a nonce of every window has no hit): one round of K2 labels when a proof exists, and the
    unchecked proof."""
    found = 0
    for trial, (r, n, windows, k2, n_labels, chunk, hits) in enumerate(patterns(31, 200, hole=True)):
        clean = np.zeros(n_labels, dtype=np.uint8)
        m = r.choice((1, 2, windows))
        for shards in (1, 2, 3):
            bounds = split_shards(n_labels, chunk, shards)
            want = windowed(emul, hits, n, windows, m, k2, bounds, chunk)[0]
            got, _, rechecked, rounds, bad, _ = windowed(emul, hits, n, windows, m, k2, bounds, chunk, 1, clean)
            assert got == want, (trial, shards)
            assert (rounds, rechecked, bad) == ((1, k2, 0) if got else (0, 0, 0)), (trial, shards)
            found += got is not None
    assert found > 100
