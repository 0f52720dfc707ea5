"""GPU tier: the batched verifier against the oracle's restatement (oracle/pyoracle.py: py_verify) on the shapes one
proof at a time never reaches: batches that mix scrypt N, (K1, K2) and label-space sizes; a gather of several layers;
Subset draws past the first 256 bytes of the XOF stream and the 1024-byte seed cap; the judge's difficulty edges
(low 56 bits zero, top byte zero, saturated, an exact lazy-cipher tie) at every ciphertext byte and nonce groups
above 255; and index widths of 10 to 64 bits, indices past the end of the POST included.

Every verdict is the oracle's: the status, and the failing position when a proof is invalid.  Every test also asserts
that it reached the path it is named for, so that another random seed cannot turn it into an easy case."""
import importlib
import re
import threading
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MASK56 = (1 << 56) - 1


@pytest.fixture(scope="module")
def vf(b2, gpu_ready):
    return importlib.import_module("go-spacemesh_b200.verify")


def _rb(rng, n):
    return bytes(rng.integers(0, 256, n, dtype=np.uint8))


def _rand_bits(rng, bits):
    return int.from_bytes(rng.bytes(8), "little") & ((1 << bits) - 1)


def _expect(orc, b2, vf, proof, meta, params, opt):
    """The oracle's verdict for one verify_batch item: (status, failing position or None)."""
    if not proof.indices:
        return b2.ERR_EMPTY_PROOF, None
    if len(proof.indices) != (params.k2 * orc.py_bits_per_index(meta.num_units * meta.labels_per_unit) + 7) // 8:
        return b2.ERR_INVALID_ARGUMENT, None
    mode = opt.get("mode", vf.MODE_ALL)
    kw = {}
    if mode == vf.MODE_SELECTED_INDEX:
        if opt.get("selected_index", 0) >= params.k2:
            return b2.ERR_INVALID_ARGUMENT, None
        kw = dict(mode="selected", selected=opt.get("selected_index", 0))
    elif mode == vf.MODE_SUBSET:
        kw = dict(mode="subset", k3=opt["k3"], seed=opt.get("seed", b""))
    ok, pos = orc.py_verify(proof.nonce, proof.indices, proof.pow, meta.node_id, meta.commitment_atx_id, meta.challenge,
                            meta.num_units, meta.labels_per_unit, params.k1, params.k2, params.scrypt_n, **kw)
    return (b2.OK, None) if ok else (b2.ERR_INVALID_PROOF, pos)


def _verdicts(b2, st, bad):
    return [(s, b if s == b2.ERR_INVALID_PROOF else None) for s, b in zip(st, bad)]


def _batch(vf, b2, proofs, metas, params, opts=None):
    return _verdicts(b2, *vf.verify_batch(proofs, metas, params, options=opts, pow="skip"))


def _assert_same(got, want):
    diff = [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert len(got) == len(want) and not diff, diff[:5]


class Opt:
    """Sets engine options for a block and restores them."""

    def __init__(self, b2, **kw):
        self.b2, self.kw = b2, kw

    def __enter__(self):
        self.old = {k: self.b2.get_option(k) for k in self.kw}
        for k, v in self.kw.items():
            self.b2.set_option(k, v)

    def __exit__(self, *a):
        for k, v in self.old.items():
            self.b2.set_option(k, v)


class _Gate:
    """pow CALLBACK that counts its calls and holds the FIRST one until released: the batch it belongs to stays on the
    device while the test queues what must go into the next batch."""

    def __init__(self):
        self.calls, self.started, self.release = 0, threading.Event(), threading.Event()

    def __call__(self, ctx, pow_, nonce_group, challenge8, difficulty, node_id):
        self.calls += 1
        if self.calls == 1:
            self.started.set()
            self.release.wait(60)
        return 0


# ------------------------------------------------------------------------------------------------ mixed batches
SPACES = [(4, 256), (3, 1000), (1, 2**20), (2, 2**32)]
# (k1, k2, scrypt N, proofs): each K1 gives mixed verdicts on some of the spaces and passes or fails the others outright
MIXED_PARAMS = [(900, 8, 2, 300), (838861, 6, 16, 260), (2**32 - 1, 4, 8192, 40)]


def _mixed_set(vf, orc, rng, idents, k1, k2, n, count):
    """`count` proofs over every identity, random indices, the three modes in rotation, and every 20th item malformed
    (empty indices, one byte short, or selected_index == K2)."""
    params = vf.VerifyParams(k1=k1, k2=k2, scrypt_n=n)
    proofs, metas, opts = [], [], []
    for i in range(count):
        node, atx, units, lpu = idents[i % len(idents)]
        nl = units * lpu
        packed = orc.py_pack_indices([int(x) for x in rng.integers(0, nl, k2)], orc.py_bits_per_index(nl))
        mode = (vf.MODE_ALL, vf.MODE_SELECTED_INDEX, vf.MODE_SUBSET)[i % 3]
        opt = dict(mode=mode)
        if mode == vf.MODE_SELECTED_INDEX:
            opt["selected_index"] = int(rng.integers(0, k2))
        elif mode == vf.MODE_SUBSET:
            opt.update(k3=int(rng.integers(1, k2 + 1)), seed=_rb(rng, int(rng.integers(0, 40))))
        if i % 20 == 7:
            kind = (i // 20) % 3
            if kind == 0:
                packed = b""
            elif kind == 1:
                packed = packed[:-1]
            else:
                opt = dict(mode=vf.MODE_SELECTED_INDEX, selected_index=k2)
        proofs.append(vf.Proof(int(rng.integers(0, 4096)), packed, int(rng.integers(0, 2**56))))
        metas.append(vf.ProofMetadata(node, atx, _rb(rng, 32), units, lpu))
        opts.append(opt)
    return params, proofs, metas, opts


def _waiting(b2):
    return float(re.search(r"^b200post_post_verification_waiting_total (\S+)$", b2.metrics_text(), re.M).group(1))


def _call(vf, b2, v, proof, meta, params, opt):
    try:
        v.verify(proof, meta, params, **opt)
        return b2.OK, None
    except vf.ErrInvalidIndex as e:
        return b2.ERR_INVALID_PROOF, e.index
    except vf.ErrEmptyProof:
        return b2.ERR_EMPTY_PROOF, None
    except b2.B200PostError as e:
        return e.code, None


def test_mixed_parameters_spaces_and_n(vf, orc, b2):
    """Proofs over four label-space sizes in each verify_batch call, then ~200 proof callers with three VerifyParams
    (N = 2, 16 and 8192) and 30 VRF checks at two N, released at once into one verifier: they are coalesced into
    the batch after a held one, where process() groups them by N and rebuilds first_item, the item rows and the
    verdict order for each group, with malformed proofs dropped in between.  Then a small batch and the large ones
    again: the grow-only judge scratch is reused and nothing changes."""
    rng = np.random.default_rng(2024)
    idents = [(_rb(rng, 32), _rb(rng, 32), u, l) for u, l in SPACES]
    sets = [_mixed_set(vf, orc, rng, idents, *p) for p in MIXED_PARAMS]
    expect = [[_expect(orc, b2, vf, p, m, q, o) for p, m, o in zip(ps, ms, os_)] for q, ps, ms, os_ in sets]
    first = []
    for (q, ps, ms, os_), want in zip(sets, expect):
        got = _batch(vf, b2, ps, ms, q, os_)
        _assert_same(got, want)
        first.append(got)
        statuses = {s for s, _ in want}
        assert {b2.OK, b2.ERR_INVALID_PROOF, b2.ERR_EMPTY_PROOF, b2.ERR_INVALID_ARGUMENT} <= statuses, statuses
        assert len({b for s, b in want if s == b2.ERR_INVALID_PROOF}) > 1     # failing positions differ between proofs

    # the queueing verifier: one held proof, then every N = 8192 proof and 80 of each other set, and the VRF checks
    gate = _Gate()
    v = vf.PostVerifier(pow=gate, max_batch_proofs=1 << 16)
    held = (0, 0)
    assert sets[0][3][0] == dict(mode=vf.MODE_ALL) and sets[0][1][0].indices
    work = [(0, i) for i in range(1, 81)] + [(1, i) for i in range(80)] + [(2, i) for i in range(MIXED_PARAMS[2][3])]
    vrf = []
    for k in range(30):
        node, atx, units, lpu = idents[k % len(idents)]
        nl = units * lpu
        nonce = [int(rng.integers(0, nl)), nl + int(rng.integers(0, 1000)), 2**32 + int(rng.integers(0, 2**20))][k % 3]
        vrf.append((node, atx, nonce, units, lpu, 2 if k % 3 else 8192))
    res = {}

    def proof_call(key):
        s, i = key
        q, ps, ms, os_ = sets[s]
        res[key] = _call(vf, b2, v, ps[i], ms[i], q, os_[i])

    def vrf_call(k):
        try:
            res[("vrf", k)] = v.verify_vrf_nonce(*vrf[k])
        except Exception as e:  # noqa: BLE001
            res[("vrf", k)] = e

    t_held = threading.Thread(target=proof_call, args=(held,))
    t_held.start()
    assert gate.started.wait(60)
    threads = [threading.Thread(target=proof_call, args=(key,)) for key in work]
    threads += [threading.Thread(target=vrf_call, args=(k,)) for k in range(len(vrf))]
    for t in threads:
        t.start()
    deadline = time.monotonic() + 60
    while _waiting(b2) < 1 + len(work) and time.monotonic() < deadline:
        time.sleep(0.02)
    time.sleep(0.5)                                   # the VRF callers are not counted as waiting: let them enqueue too
    gate.release.set()
    for t in [t_held] + threads:
        t.join()
    batches, n_proofs = v.stats()
    v.close()
    assert n_proofs == 1 + len(work)
    assert batches - 1 <= 2, batches                  # the released callers went out in at most two batches
    bad = [(key, res[key], expect[key[0]][key[1]]) for key in [held] + work if res[key] != expect[key[0]][key[1]]]
    assert not bad, bad[:5]
    assert len({MIXED_PARAMS[s][2] for s, _ in work}) == 3
    for k, c in enumerate(vrf):
        label32 = orc.c_label32(orc.c_commitment(c[0], c[1]), c[2], c[5])
        assert res[("vrf", k)] == (label32 < orc.py_vrf_difficulty(c[3] * c[4]), label32), k

    # a small batch, then the large ones again
    q, ps, ms, os_ = sets[0]
    assert _batch(vf, b2, ps[:3], ms[:3], q, os_[:3]) == expect[0][:3]
    for (q, ps, ms, os_), got in zip(sets, first):
        assert _batch(vf, b2, ps, ms, q, os_) == got


# ------------------------------------------------------------------------------------------------ several layers
def test_gather_over_several_layers(vf, orc, b2):
    """64 proofs x K2 = 37 at N = 8192 with 256-slot layers and the low-latency kernel off: the 2368 labels are
    gathered in ten layers, and failing positions land in late layers."""
    rng = np.random.default_rng(8192)
    n_proofs, k2, nl = 64, 37, 2**20
    params = vf.VerifyParams(k1=int(0.98 * nl), k2=k2, scrypt_n=8192)
    bits = orc.py_bits_per_index(nl)
    proofs, metas = [], []
    for i in range(n_proofs):
        proofs.append(vf.Proof(int(rng.integers(0, 4096)), orc.py_pack_indices([int(x) for x in rng.integers(0, nl, k2)], bits),
                               int(rng.integers(0, 2**56))))
        metas.append(vf.ProofMetadata(_rb(rng, 32), _rb(rng, 32), _rb(rng, 32), 1, nl))
    with Opt(b2, max_scratch_mib=512, lowlat_max_labels=0):
        slots = b2.wave_slots(8192)
        assert slots == 256 and n_proofs * k2 >= 4 * slots
        got = _batch(vf, b2, proofs, metas, params)
    want = [_expect(orc, b2, vf, p, m, params, {}) for p, m in zip(proofs, metas)]
    _assert_same(got, want)
    assert any(s == b2.OK for s, _ in want)
    assert any(s == b2.ERR_INVALID_PROOF and (i * k2 + b) // slots >= 3 for i, (s, b) in enumerate(want))


# ------------------------------------------------------------------------------------------------ Subset at large k3
SUBSET_K3 = (1, 127, 128, 129, 200, 300, 1000)


@pytest.fixture(scope="module")
def subset_space(vf, orc):
    """A brute-forced valid proof with K2 = 300 over 2^16 labels (17-bit indices: 638 packed bytes) at N = 2."""
    rng = np.random.default_rng(300)
    node, atx, ch = _rb(rng, 32), _rb(rng, 32), _rb(rng, 32)
    nl, k2 = 2**16, 300
    params = vf.VerifyParams(k1=int(0.4 * nl), k2=k2, scrypt_n=2)
    nonce, pow_ = 4099, int(rng.integers(0, 2**56))
    packed, hits = orc.py_prove(node, atx, ch, 1, nl, params.k1, k2, 2, nonce=nonce, pow_=pow_)
    assert packed is not None and len(packed) == 638
    return vf.ProofMetadata(node, atx, ch, 1, nl), params, vf.Proof(nonce, packed, pow_), hits


def test_subset_draws_past_the_first_stream(vf, orc, b2, subset_space):
    """~1500 variants of the proof, each with 1 to 8 positions replaced by random labels (a new seed, so a new
    selection order), judged with k3 from 1 to 1000 (clamped to K2) and caller seeds of 0, 32 and 374 bytes (the
    last makes the hashed seed exactly 1024 bytes).  The Subset stream starts at 256 bytes, 128 draws: calls whose
    first failure comes after more than 128 selections read the refilled stream."""
    meta, params, proof, hits = subset_space
    rng = np.random.default_rng(301)
    seeds = (b"", _rb(rng, 32), _rb(rng, 374))
    assert len(seeds[2]) + 4 + len(proof.indices) + 8 == 1024
    bits = orc.py_bits_per_index(meta.labels_per_unit)
    proofs, opts = [], []
    for v in range(1500 + len(SUBSET_K3) * len(seeds)):
        if v < len(SUBSET_K3) * len(seeds):
            p = proof                                     # the untampered proof at every (k3, seed)
        else:
            ix = list(hits)
            for pos in rng.choice(params.k2, int(rng.integers(1, 9)), replace=False):
                ix[pos] = int(rng.integers(0, meta.labels_per_unit))
            p = vf.Proof(proof.nonce, orc.py_pack_indices(ix, bits), proof.pow)
        proofs.append(p)
        opts.append(dict(mode=vf.MODE_SUBSET, k3=SUBSET_K3[v % len(SUBSET_K3)], seed=seeds[(v // len(SUBSET_K3)) % len(seeds)]))
    got = _batch(vf, b2, proofs, [meta] * len(proofs), params, opts)
    want = [_expect(orc, b2, vf, p, meta, params, o) for p, o in zip(proofs, opts)]
    _assert_same(got, want)
    assert all(w == (b2.OK, None) for w in want[:len(SUBSET_K3) * len(seeds)])
    late = 0
    for p, o, (s, pos) in zip(proofs, opts, want):
        if s == b2.ERR_INVALID_PROOF:
            order = [w for _, w in orc.py_subset_positions(orc.py_unpack_indices(p.indices, bits, params.k2), o["seed"], p.nonce,
                                                           p.indices, p.pow, o["k3"], with_positions=True)]
            late += order.index(pos) >= 129 and len(o["seed"]) == 374
    assert late >= 10, late                           # after the refill, with the 1024-byte seed


def test_subset_seed_cap(vf, orc, b2, subset_space):
    """The Subset seed is caller seed || LE32(nonce) || packed indices || LE64(pow), hashed as one BLAKE3 chunk: at
    most 1024 bytes.  A proof on the wire carries at most 800 bytes of indices, so no network proof with a caller seed
    of up to 212 bytes reaches the cap; past it the verifier refuses the call (ERR_INVALID_ARGUMENT) instead of
    hashing a multi-chunk input.  Here 1024 bytes are judged as the oracle judges them and 1025 are refused."""
    meta, params, proof, hits = subset_space
    bits = orc.py_bits_per_index(meta.labels_per_unit)
    rng = np.random.default_rng(302)
    for _ in range(64):                               # replace position 150 with a label that fails
        ix = list(hits)
        ix[150] = int(rng.integers(0, meta.labels_per_unit))
        tampered = vf.Proof(proof.nonce, orc.py_pack_indices(ix, bits), proof.pow)
        if _expect(orc, b2, vf, tampered, meta, params, dict(mode=vf.MODE_SELECTED_INDEX, selected_index=150))[0] != b2.OK:
            break
    at_cap = 1024 - 4 - len(proof.indices) - 8
    proofs, opts, want = [], [], []
    for p in (proof, tampered):
        for seed_len in (at_cap, at_cap + 1):
            o = dict(mode=vf.MODE_SUBSET, k3=params.k2, seed=(bytes(range(256)) * 2)[:seed_len])
            proofs.append(p)
            opts.append(o)
            want.append(_expect(orc, b2, vf, p, meta, params, o) if seed_len == at_cap else (b2.ERR_INVALID_ARGUMENT, None))
    assert want[0] == (b2.OK, None) and want[2] == (b2.ERR_INVALID_PROOF, 150)
    _assert_same(_batch(vf, b2, proofs, [meta] * 4, params, opts), want)


# ------------------------------------------------------------------------------------------------ difficulty edges
# name: (num_units, labels_per_unit, k1)
REGIMES = {
    "lsb0-m1": (4, 256, 4),          # difficulty 1 * 2^56: its low 56 bits are zero
    "lsb0-m128": (4, 256, 512),      # 128 * 2^56
    "lsb0-m255": (4, 256, 1020),     # 255 * 2^56
    "msb0": (4, 2**32, 26),          # mainnet: K1 = 26 over 2^34 labels, top byte zero
    "saturated": (4, 256, 1024),     # k1 >= num_labels clamps to 2^64 - 1
    "control": (3, 1000, 2500),      # neither byte nor low bits special
}


def _nonce(rng, i):
    """nonce % 16 = i % 16 for every 16 consecutive i; nonce groups below 256, in [256, 2^16) and 2^28 - 1."""
    kind = (i // 16) % 3
    group = [int(rng.integers(0, 256)), int(rng.integers(256, 2**16)), 2**28 - 1][kind]
    return 16 * group + i % 16


@pytest.mark.parametrize("regime", REGIMES)
def test_judge_difficulty_edges(vf, orc, b2, regime):
    """~1000 proofs through one batch at one difficulty regime, nonces at all 16 ciphertext bytes and in nonce groups
    above 255 (up to nonce 2^32 - 1).  Up to two of each proof's eight labels are picked so that the selected
    ciphertext byte equals the difficulty's top byte: the lazy cipher, not the first compare, decides them."""
    units, lpu, k1 = REGIMES[regime]
    nl = units * lpu
    diff = orc.py_proving_difficulty(k1, nl)
    assert vf.proving_difficulty(k1, nl) == diff
    msb, lsb = diff >> 56, diff & MASK56
    assert {"lsb0": lsb == 0 and msb > 0, "msb0": msb == 0 and lsb > 0, "saturated": diff == 2**64 - 1,
            "control": msb not in (0, 255) and lsb != 0}[regime.split("-")[0]]
    rng = np.random.default_rng(sorted(REGIMES).index(regime) + 500)
    node, atx = _rb(rng, 32), _rb(rng, 32)
    comm = orc.py_commitment(node, atx)
    pool = np.array([int(x) for x in rng.integers(0, nl, 4096)], dtype=np.uint64)
    pool_labels = orc.c_labels_gather(np.tile(np.frombuffer(comm, dtype=np.uint8), (len(pool), 1)), pool, 2)
    k2, bits = 8, orc.py_bits_per_index(nl)
    params = vf.VerifyParams(k1=k1, k2=k2, scrypt_n=2)
    proofs, metas, opts = [], [], []
    at_msb = 0
    for i in range(1008):
        ch, nonce, pow_ = _rb(rng, 32), _nonce(rng, i), int(rng.integers(0, 2**56))
        ct = np.frombuffer(orc.py_aes128(orc.py_cipher_key(ch, nonce // 16, pow_), pool_labels.tobytes()), dtype=np.uint8)
        eq = np.flatnonzero(ct.reshape(-1, 16)[:, nonce % 16] == msb)
        pick = list(rng.choice(len(pool), k2, replace=False))
        for slot in rng.choice(k2, min(int(rng.integers(0, 3)), len(eq)), replace=False):
            pick[slot] = int(rng.choice(eq))
        ix = [int(pool[j]) for j in pick]
        at_msb += int((ct.reshape(-1, 16)[pick, nonce % 16] == msb).sum())
        proofs.append(vf.Proof(nonce, orc.py_pack_indices(ix, bits), pow_))
        metas.append(vf.ProofMetadata(node, atx, ch, units, lpu))
        opts.append(dict(mode=vf.MODE_SELECTED_INDEX, selected_index=int(rng.integers(0, k2))) if i % 3 == 2 else {})
    got = _batch(vf, b2, proofs, metas, params, opts)
    want = [_expect(orc, b2, vf, p, m, params, o) for p, m, o in zip(proofs, metas, opts)]
    _assert_same(got, want)
    assert at_msb >= 200, at_msb
    assert {p.nonce % 16 for p in proofs} == set(range(16)) and any(p.nonce >= 4096 for p in proofs)
    assert any(p.nonce == 2**32 - 1 for p in proofs)
    if regime in ("lsb0-m128", "control"):
        assert 0 < sum(s == b2.OK for s, _ in want) < len(want)


def test_lazy_cipher_tie(vf, orc, b2):
    """Top byte of the difficulty zero (mainnet's regime) and a label whose selected byte is zero: the low 56 bits of the
    lazy cipher decide, and a label passes only when they are strictly below the difficulty's.  A label whose lazy value
    X lies in [2^34, 2^47) is found by search, so that (K1, numLabels) pairs with difficulty exactly X - 1, X and X + 1
    exist; the label fails at the first two and passes at the third.  Its nonce group is above 255."""
    rng = np.random.default_rng(56)
    node, atx, ch = _rb(rng, 32), _rb(rng, 32), _rb(rng, 32)
    labels, _, _, _ = orc.c_labels_range(orc.py_commitment(node, atx), 2, 0, 1 << 16)
    pow_, found = int(rng.integers(0, 2**56)), None
    for group in range(300, 340):
        ct = np.frombuffer(orc.py_aes128(orc.py_cipher_key(ch, group, pow_), labels.tobytes()), dtype=np.uint8).reshape(-1, 16)
        for b in range(16):
            rows = np.flatnonzero(ct[:, b] == 0)
            if not len(rows):
                continue
            lazy = np.frombuffer(orc.py_aes128(orc.py_cipher_key(ch, group, pow_, 16 * group + b), labels[rows].tobytes()),
                                 dtype=np.uint8).reshape(-1, 16)
            low = lazy[:, :8].copy().view("<u8")[:, 0] & np.uint64(MASK56)
            hit = np.flatnonzero((low >= np.uint64(2**34)) & (low < np.uint64(2**47)))
            if len(hit):
                found = (16 * group + b, int(rows[hit[0]]), int(low[hit[0]]))
                break
        if found:
            break
    assert found, "no label with a small lazy value"
    nonce, index, x = found
    k1 = 2**32 - 1
    proofs, metas, want = [], [], []
    for d, ok in ((x - 1, False), (x, False), (x + 1, True)):
        nl = (k1 << 64) // d
        assert orc.py_proving_difficulty(k1, nl) == d == vf.proving_difficulty(k1, nl)
        meta = vf.ProofMetadata(node, atx, ch, 1, nl)
        proof = vf.Proof(nonce, orc.py_pack_indices([index], orc.py_bits_per_index(nl)), pow_)
        params = vf.VerifyParams(k1=k1, k2=1, scrypt_n=2)
        assert _expect(orc, b2, vf, proof, meta, params, {}) == ((b2.OK, None) if ok else (b2.ERR_INVALID_PROOF, 0))
        proofs.append(proof)
        metas.append(meta)
        want.append((b2.OK, None) if ok else (b2.ERR_INVALID_PROOF, 0))
    _assert_same(_batch(vf, b2, proofs, metas, vf.VerifyParams(k1=k1, k2=1, scrypt_n=2)), want)


# ------------------------------------------------------------------------------------------------ index width
WIDTH_SPACES = [(1, 2**k + d) for k in (10, 32, 33) for d in (-1, 0, 1)] + [(2**31, 2**32)]


@pytest.mark.parametrize("units,lpu", WIDTH_SPACES, ids=[f"{u}x{l}" for u, l in WIDTH_SPACES])
def test_index_width(vf, orc, b2, units, lpu):
    """Label spaces of 2^k - 1, 2^k and 2^k + 1 labels (k + 0 or 1 bits per index, 32-, 33- and 34-bit indices that
    straddle 64-bit words) and one of 2^63 labels (64-bit indices).  Indices are drawn over the whole width, so some
    are >= numLabels: those are recomputed and judged, not refused.  The packed length, pack and unpack round trips
    and every verdict are the oracle's."""
    nl = units * lpu
    bits = orc.py_bits_per_index(nl)
    assert vf.bits_per_index(nl) == bits
    rng = np.random.default_rng(nl % 100003)
    k2 = 7
    params = vf.VerifyParams(k1=min(int(0.9 * nl), 2**32 - 1), k2=k2, scrypt_n=2)
    node, atx = _rb(rng, 32), _rb(rng, 32)
    proofs, metas, opts, every = [], [], [], []
    for i in range(120):
        ix = [_rand_bits(rng, bits) for _ in range(k2)]
        if i == 0:
            ix[:4] = [0, nl - 1, (1 << bits) - 1, min(nl, (1 << bits) - 1)]
        packed = vf.pack_indices(ix, bits)
        assert packed == orc.py_pack_indices(ix, bits) and len(packed) == (k2 * bits + 7) // 8
        assert vf.unpack_indices(packed, bits, k2) == ix
        every += ix
        proofs.append(vf.Proof(int(rng.integers(0, 2**32)), packed, int(rng.integers(0, 2**56))))
        metas.append(vf.ProofMetadata(node, atx, _rb(rng, 32), units, lpu))
        opts.append(dict(mode=vf.MODE_SUBSET, k3=4, seed=b"w") if i % 2 else {})
    assert any(x >= nl for x in every) and max(every) >= 2**(bits - 1)
    got = _batch(vf, b2, proofs, metas, params, opts)
    want = [_expect(orc, b2, vf, p, m, params, o) for p, m, o in zip(proofs, metas, opts)]
    _assert_same(got, want)
    assert all(s in (b2.OK, b2.ERR_INVALID_PROOF) for s, _ in want)
    if nl < 2**34:
        assert len(set(want)) > 2                     # verdicts and failing positions vary
