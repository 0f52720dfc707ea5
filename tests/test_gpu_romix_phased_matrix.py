"""GPU tier: the phased ROMix layer (romix_variant 5, romix_phased_kernel) at the shapes production runs it.

test_gpu_romix_phased.py runs every phased instance at N <= 1024 with one CTA per SM.  This module runs the kernel
where init, bench.py, verify batches and repair run it: full N = 8192 layers of 2 x wave_slots labels, several CTAs per
SM, grids capped below one CTA per SM (the only way the 512-thread instance runs at N = 8192), and N up to 2^20, where
each of a warp's two scratchpad regions is exactly 4 GiB.

Every case proves that it ran the shape it names:
  - wave: b2.wave_slots(N) equals predict_wave(), a restatement of ensure()'s rule for the phased kernel (engine.cu),
    which also names the CTA size and CTAs per SM that ran;
  - launches: a call of `count` labels makes exactly ceil(count / (2 x wave)) ROMix launches, one per layer.  The
    pipelined kernel would make layers + 1, the low-latency kernel 1 (lowlat_max_labels = 0 wherever a call could fall
    under it);
  - output: labels equal the reference byte for byte, and so does the VRF candidate.

One range per N, [START, START + count), under one commitment, and one reference of it: the pipelined kernel's output
(the full oracle's at N = 64), pinned to the oracle on >= 256 labels that include slots 0, 31, 32, S - 1, S, S + 1 and
2S - 1 of every layer of every wave S the cases use, and the last label.

Options are process-global; every test restores the ones it sets.  The module starts by releasing this process's
engines (b2.shutdown()), so the HBM budget the cases predict is the card's free memory, not what earlier modules left,
and releases them again when it ends.
"""
import hashlib
import math
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PHASED, PIPELINED = 5, 4
# (rotate_mask, tpb) of every romix_phased_kernel instance; test_romix_phased_launch_table.py checks it against the table
PHASED_MATRIX = [(mw, tpb) for mw in (0, 1) for tpb in (64, 128, 256, 512)]
OPTION_KEYS = ("romix_variant", "rotate_mask", "tpb", "dr_unroll", "ctas_per_sm", "max_scratch_mib", "speculate_next",
               "lowlat_max_labels")
START = 2**34 - 40_000          # the ranges cross 2^34
TAIL = 1037                     # not a multiple of 32 or of any CTA size
FULL_N = 8192
HBM_SHARE = 0.95                # ensure(): the layer budget is 95 % of free HBM
LADDER_MIB = 24576              # section C: 384, 192 and 96 slots at N = 2^18, 2^19, 2^20
NODE, ATX = bytes(range(40, 72)), bytes(range(3, 35))


def per_slot(n):
    """HBM bytes of one phased slot: two scratchpads of 128 x N bytes"""
    return 256 * n


def predict_wave(card, n, tpb, ctas_opt, cap_mib, free=None):
    """ensure()'s layer rule for the phased kernel, restated: (wave_slots, CTA size, CTAs per SM).
    - ctas_for(t): the occupancy limit, then the ctas_per_sm option, then what the budget holds;
    - the CTA-size search goes only down from the requested tpb, and takes a smaller size only for strictly more slots;
    - if not even one CTA per SM fits, the requested size stays and the wave is what the budget holds, in whole warps;
    - the budget is 95 % of free HBM less V's alignment pad, or max_scratch_mib if that is less."""
    free = card["free"] if free is None else free
    budget = max(0, int(free * HBM_SHARE) - v_pad(n))
    if cap_mib > 0:
        budget = min(budget, cap_mib << 20)
    sms, occ, ps = card["sms"], card["occ"], per_slot(n)

    def ctas_for(t):
        c = occ[t]
        if ctas_opt > 0:
            c = min(c, ctas_opt)
        while c > 0 and ps * t * sms * c > budget:
            c -= 1
        return c
    ctas = ctas_for(tpb)
    t = tpb // 2
    while t >= 64:
        c = ctas_for(t)
        if c * t > ctas * tpb:
            ctas, tpb = c, t
        t //= 2
    ctas = max(ctas, 1)
    wave = sms * ctas * tpb
    if ps * wave > budget:
        wave = budget // ps // 32 * 32
    return wave, tpb, ctas


def v_pad(n):
    """ensure()'s alignment pad of V: the per-warp region size N x 4 KiB, at most 4 GiB"""
    return min(128 * n * 32, 1 << 32)


def need_hbm(card, nbytes, what):
    """A case whose shape needs `nbytes` of layer budget fails, rather than silently testing a smaller layer."""
    if nbytes + v_pad(FULL_N) > card["free"] * HBM_SHARE:
        import torch
        pytest.fail(f"{what} needs {nbytes / 2**30:.1f} GiB of layer budget; torch.cuda.mem_get_info() = "
                    f"{torch.cuda.mem_get_info()} with this process's engines released")


@pytest.fixture
def opts(b2, gpu_ready):
    """opts(**kw) sets options for the rest of the test; all of OPTION_KEYS are restored afterwards."""
    old = {k: b2.get_option(k) for k in OPTION_KEYS}

    def set_(**kw):
        for k, v in kw.items():
            b2.set_option(k, v)
    yield set_
    set_(**old)


def counted(b2, fn):
    """(fn(), ROMix launches it made)"""
    b2.romix_time(reset=True)
    out = fn()
    return out, b2.romix_time()[1]


def same(got, exp, what):
    """assert byte equality of label rows, naming the first differing row"""
    assert got.shape == exp.shape, what
    bad = np.flatnonzero((got != exp).any(axis=1))
    assert bad.size == 0, f"{what}: {bad.size} of {len(exp)} labels differ, first at row {bad[0]}"


def free_hbm(b2):
    """free device memory with this process's label and k2pow engines released"""
    import torch
    b2.shutdown()
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()


@pytest.fixture(scope="module")
def card(b2, gpu_ready):
    """sms, free HBM and each phased instance's occupancy limit in CTAs per SM; the engines are released before and
    after the module.

    Python cannot query occupancy, so it is read from wave_slots at N = 64, where HBM does not bind, with
    ctas_per_sm = K for K = 1, 2, ...: the requested size t keeps min(occ(t), K) CTAs as long as occ(t) >= K - 1 (a
    size t' <= t / 2 reaches at most K t' <= K t / 2 <= (K - 1) t slots), so the first K whose wave is below K CTAs
    per SM gives occ(t).  With ctas_per_sm = 0 the search could replace t by a smaller size and hide occ(t)."""
    t0 = time.time()
    free, total = free_hbm(b2)
    sms = gpu_ready[0]["sm_count"]
    keys = ("romix_variant", "rotate_mask", "tpb", "ctas_per_sm", "max_scratch_mib")
    old = {k: b2.get_option(k) for k in keys}
    occ_by = {}
    try:
        for mw, tpb in PHASED_MATRIX:
            b2.set_option("romix_variant", PHASED)
            b2.set_option("rotate_mask", mw)
            b2.set_option("tpb", tpb)
            b2.set_option("max_scratch_mib", 0)
            for k in range(1, 33):
                b2.set_option("ctas_per_sm", k)
                w = b2.wave_slots(64)
                assert w % (sms * tpb) == 0, (mw, tpb, k, w)
                c = w // (sms * tpb)
                assert c in (k, k - 1), (mw, tpb, k, c)
                if c < k:
                    break
            occ_by[mw, tpb] = c
    finally:
        for k, v in old.items():
            b2.set_option(k, v)
    occ = {}
    for (mw, tpb), c in occ_by.items():
        assert c >= 1 and occ.setdefault(tpb, c) == c, ("occupancy differs between rotate masks", tpb, occ_by)
    print(f"\n[phased matrix] {gpu_ready[0]['model']}: {sms} SMs, free HBM {free / 2**30:.2f} of "
          f"{total / 2**30:.2f} GiB, CTAs per SM by tpb {occ} ({time.time() - t0:.1f} s)")
    yield {"sms": sms, "free": free, "total": total, "occ": occ}
    b2.shutdown()   # the cases leave V at up to 68 GiB: later modules and their subprocesses get that HBM back


# ----------------------------------------------------------------------------------------------- the range per N
def waves_used(card, n):
    """every wave the cases of this module run at scrypt-N n"""
    if n == FULL_N:
        ws = {card["sms"] * 256}                                # A's pinned instances and B's default
        ws |= {cap_wave(tpb) for tpb in (64, 128, 256, 512)}    # A's capped instances
        return sorted(ws)
    return sorted({predict_wave(card, n, tpb, 0, 0)[0] for _, tpb in PHASED_MATRIX})   # D


def cap_wave(tpb):
    """A's capped wave: four CTAs and 160 slots, under one 64-thread CTA per SM"""
    return 4 * tpb + 160


def cap_mib(tpb):
    return cap_wave(tpb) * per_slot(FULL_N) >> 20


def seam_positions(count, s):
    """slots 0, 31, 32, S - 1, S, S + 1, 2S - 1 of every layer of 2S labels, and the last label"""
    pos = [base + d for base in range(0, count, 2 * s) for d in (0, 31, 32, s - 1, s, s + 1, 2 * s - 1)]
    return [p for p in pos if p < count] + [count - 1]


def argmin_pos(labels):
    """position of the smallest label (big-endian, as the VRF compares label32 words)"""
    v = labels.view(">u8")
    return int(np.lexsort((v[:, 1], v[:, 0]))[0])


class Ref:
    """One commitment and [START, START + count) at scrypt-N n with its reference labels and VRF candidate."""

    def __init__(self, b2, orc, card, n):
        t0 = time.time()
        self.n, self.waves = n, waves_used(card, n)
        wmax = max(self.waves)
        # 2 x wmax + wmax + TAIL at N = 8192 (a full layer and a ragged one at the largest wave); 3 layers and a ragged
        # fourth at the small N
        self.count = (3 if n == FULL_N else 7) * wmax + TAIL
        self.diff = orc.py_vrf_difficulty(self.count // 64)
        keys = ("romix_variant", "rotate_mask", "tpb", "dr_unroll", "ctas_per_sm", "max_scratch_mib", "lowlat_max_labels")
        old = {k: b2.get_option(k) for k in keys}
        try:
            for k, v in dict(romix_variant=PIPELINED, rotate_mask=0, tpb=256, dr_unroll=4, ctas_per_sm=1,
                             max_scratch_mib=0, lowlat_max_labels=0).items():
                b2.set_option(k, v)
            for attempt in range(32):
                self.c = hashlib.sha256(b"phased-matrix-N%d-%d" % (n, attempt)).digest()
                if n == 64:
                    self.labels, found, idx, l32 = orc.c_labels_range(self.c, n, START, self.count, self.diff)
                    assert found
                    self.vrf = (idx, l32)
                else:
                    self.labels, self.vrf = b2.labels_range(self.c, n, START, self.count, vrf_difficulty_=self.diff)
                self.m = self.vrf[0] - START
                # section B places the arg-min in the A half, the B half and the ragged last layer of sub-range calls
                # that lie inside the range: that needs 2S + 64 <= m <= count - 5000
                s = card["sms"] * 256
                if n != FULL_N or 2 * s + 64 <= self.m <= self.count - 5000:
                    break
            else:
                pytest.fail("no commitment with a usable arg-min position")
        finally:
            for k, v in old.items():
                b2.set_option(k, v)
        assert self.m == argmin_pos(self.labels), "the VRF candidate is the range's smallest label"
        assert orc.c_label32(self.c, self.vrf[0], n) == self.vrf[1]
        if n > 64:
            rng = np.random.default_rng(n)
            pick = set(rng.integers(0, self.count, 256).tolist()) | {self.m}
            for s in self.waves:
                pick |= set(seam_positions(self.count, s))
            pick = np.array(sorted(pick))
            assert len(pick) >= 256
            comms = np.tile(np.frombuffer(self.c, dtype=np.uint8), (len(pick), 1))
            same(self.labels[pick], orc.c_labels_gather(comms, (START + pick).astype(np.uint64), n),
                 f"N={n} pipelined reference vs oracle")
        print(f"\n[phased matrix] N={n}: reference of {self.count} labels, waves {self.waves}, arg-min at {self.m} "
              f"({time.time() - t0:.1f} s)")


@pytest.fixture(scope="module")
def ref(b2, orc, card):
    """ref(n): the module's range and reference at scrypt-N n, built on first use."""
    cache = {}

    def get(n):
        if n not in cache:
            cache[n] = Ref(b2, orc, card, n)
        return cache[n]
    return get


def run_range(b2, r, wave, what, start=0, count=None):
    """the phased call over [start, start + count) of the range against the reference: labels, VRF and launches"""
    count = r.count - start if count is None else count
    (got, vrf), k = counted(b2, lambda: b2.labels_range(r.c, r.n, START + start, count, vrf_difficulty_=r.diff))
    assert k == math.ceil(count / (2 * wave)), (what, "launches", k, "wave", wave)
    same(got, r.labels[start: start + count], what)
    return vrf


# --------------------------------------------------------------------------------- A: N = 8192, each instance
A_CASES = [(mw, tpb, ctas, 0) for mw in (0, 1) for tpb, ctas in ((256, 1), (128, 2), (64, 4))]
A_CASES += [(mw, tpb, 0, cap_mib(tpb)) for mw in (0, 1) for tpb in (64, 128, 256, 512)]


@pytest.mark.parametrize("mw,tpb,ctas,cap", [
    pytest.param(*c, id=f"mw{c[0]}-tpb{c[1]}-N8192-ctas{c[2]}-" + (f"cap{c[3]}" if c[3] else "uncapped")) for c in A_CASES])
def test_full_n_instance(b2, opts, card, ref, mw, tpb, ctas, cap):
    """romix_phased_kernel<mw, tpb> over full N = 8192 layers of 2S labels and a ragged last layer.

    ctas_per_sm 1/2/4 with tpb 256/128/64 all give S = sms x 256: 256 is the production instance, and 128 and 64 put
    two and four CTAs on an SM, each with its own PHASED_BUFS x (tile A, tile B) + index words of dynamic shared memory.
    Under the cap, ensure()'s `per_slot * wave > budget` branch keeps the requested tpb and rounds the wave down to whole
    warps: S = 4 tpb + 160, a grid of four CTAs and a partial fifth.  That is the only way the 512-thread instance (single
    tiles, the `bulk_wait_read<0>` path of TILE_FREE) runs at this N."""
    r = ref(FULL_N)
    what = f"phased<mw={mw}, tpb={tpb}> N=8192 ctas_per_sm={ctas} cap={cap} MiB"
    opts(romix_variant=PHASED, rotate_mask=mw, tpb=tpb, ctas_per_sm=ctas, max_scratch_mib=cap, lowlat_max_labels=0)
    exp, ran_tpb, ran_ctas = predict_wave(card, FULL_N, tpb, ctas, cap)
    if cap:
        assert cap << 20 < per_slot(FULL_N) * 64 * card["sms"], "the cap holds less than one 64-thread CTA per SM"
        assert exp == cap_wave(tpb) and exp % tpb, (what, exp)
    else:
        need_hbm(card, per_slot(FULL_N) * card["sms"] * 256, what)
        assert (exp, ran_tpb, ran_ctas) == (card["sms"] * 256, tpb, ctas), (what, exp, ran_tpb, ran_ctas)
    wave = b2.wave_slots(FULL_N)
    assert wave == exp, (what, "wave", wave, "predicted", exp)
    assert r.count >= 2 * wave + wave + TAIL and (r.count % (2 * wave)) % 32, (what, "the last layer is ragged")
    vrf = run_range(b2, r, wave, what)
    assert vrf == r.vrf, (what, "VRF")


# --------------------------------------------------------------------------------- B: default configuration
@pytest.fixture
def default_wave(b2, opts, card):
    """the default options' wave at N = 8192: ensure() takes the requested 512 threads down to 256 (one CTA per SM),
    because the budget holds no 512-thread CTA per SM and 128/64-thread CTAs give no more slots."""
    assert b2.get_option("romix_variant") == PHASED and b2.get_option("ctas_per_sm") == 0 \
        and b2.get_option("max_scratch_mib") == 0, "section B runs the default options"
    s = card["sms"] * 256
    need_hbm(card, per_slot(FULL_N) * s, "the default N = 8192 layer")
    exp = predict_wave(card, FULL_N, b2.get_option("tpb"), 0, 0)
    assert exp == (s, 256, 1), exp
    wave = b2.wave_slots(FULL_N)
    assert wave == s, ("default wave", wave)
    return wave


def test_default_range(b2, ref, default_wave):
    """What bench.py and init run: the whole range (a full layer of 2S and a ragged one) and its VRF candidate."""
    r = ref(FULL_N)
    assert run_range(b2, r, default_wave, "default N=8192 range") == r.vrf


def test_default_vrf_argmin_position(b2, ref, default_wave):
    """The range's arg-min m, reached from three sub-range calls: at position 7 (A half of layer 0), at S + 7 (B half of
    layer 0) and in the ragged second layer (position 2S + 7).  Each call's K3 candidates and K4 merge must return m."""
    r, s = ref(FULL_N), default_wave
    for name, off in (("A half", r.m - 7), ("B half", r.m - s - 7), ("ragged last layer", r.m - 2 * s - 7)):
        assert 0 <= off
        vrf = run_range(b2, r, s, f"default N=8192 sub-range, arg-min in the {name}", start=off)
        assert vrf == r.vrf, (name, vrf)


def test_default_gathers(b2, orc, ref, default_wave):
    """labels_gather (per-item commitments) and labels_gather_indexed over 2 full layers and a ragged third.  Most items
    are range labels at random positions; every 5th has its own commitment and index (drawn from a pool of 1024 pairs
    with oracle labels, the first at index 2^64 - 1)."""
    r, s = ref(FULL_N), default_wave
    g = 2 * 2 * s + s + 333
    rng = np.random.default_rng(8192)
    pos = rng.integers(0, r.count, g)
    idx = (START + pos).astype(np.uint64)
    exp = r.labels[pos]
    pool = 1024
    pool_c = rng.integers(0, 256, (pool, 32), dtype=np.uint8)
    pool_i = rng.integers(0, 2**64 - 1, pool, dtype=np.uint64)
    pool_i[0] = 2**64 - 1
    pool_l = orc.c_labels_gather(pool_c, pool_i, FULL_N)
    own = np.flatnonzero(np.arange(g) % 5 == 2)
    which = np.arange(len(own)) % pool
    idx[own] = pool_i[which]
    exp[own] = pool_l[which]
    comms = np.tile(np.frombuffer(r.c, dtype=np.uint8), (g, 1))
    comms[own] = pool_c[which]
    got, k = counted(b2, lambda: b2.labels_gather(comms, idx, FULL_N))
    assert k == 3, ("gather launches", k)
    same(got, exp, "default N=8192 gather")
    table = np.concatenate([np.frombuffer(r.c, dtype=np.uint8)[None], pool_c])
    cidx = np.zeros(g, dtype=np.uint32)
    cidx[own] = 1 + which
    got, k = counted(b2, lambda: b2.labels_gather_indexed(table, cidx, idx, FULL_N))
    assert k == 3, ("indexed gather launches", k)
    same(got, exp, "default N=8192 indexed gather")


def test_default_compare(b2, orc, default_wave, tmp_path):
    """K3c: a POST of 2 x 2S + S + 37 labels in one file, written by a setup session and checked in full by verify_pos
    (one compare job of three layers).  One label flipped at 0, S - 1, S, 2S - 1, 2S, 3S and the last: exactly those
    positions come back as bad_index."""
    import shutil
    from pathlib import Path
    import importlib
    su = importlib.import_module("go-spacemesh_b200.setup")
    s = default_wave
    total = 5 * s + 37
    d = tmp_path / "post"
    mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=total, max_num_units=10))
    mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=1, max_file_size=16 * total, provider_id=0,
                                             scrypt_n=FULL_N), NODE, ATX)
    mgr.start_session()
    assert mgr.status().state == su.STATE_COMPLETE
    stored = np.fromfile(d / "postdata_0.bin", dtype=np.uint8).reshape(-1, 16)
    assert len(stored) == total
    victims = [0, s - 1, s, 2 * s - 1, 2 * s, 3 * s, total - 1]
    comm = orc.c_commitment(NODE, ATX)
    same(stored[victims], orc.c_labels_gather(np.tile(np.frombuffer(comm, dtype=np.uint8), (len(victims), 1)),
                                              np.array(victims, dtype=np.uint64), FULL_N), "stored POST vs oracle")
    r, k = counted(b2, lambda: su.verify_pos(str(d), fraction=100))
    assert r.code == su.OK and r.labels_checked == total, r
    assert k >= 3, ("compare launches", k)
    bad = tmp_path / "bad"
    shutil.copytree(d, bad)
    with open(Path(bad) / "postdata_0.bin", "r+b") as f:
        for i in victims:
            f.seek(i * 16 + 9)
            v = f.read(1)[0]
            f.seek(-1, 1)
            f.write(bytes([v ^ 0x20]))
    r = su.verify_pos(str(bad), fraction=100)
    assert r.code == su.ERR_LABEL_MISMATCH and r.bad_index == victims, (r.code, r.bad_index)


# --------------------------------------------------------------------------------- C: N up to 2^20
LADDER = (1 << 18, 1 << 19, 1 << 20)
LARGE_INSTANCES = ((0, 512), (1, 64))
_large = {}


def large_count(s):
    """2 full layers and a ragged third in which only the first warps have a B"""
    return 4 * s + s + 37


def test_large_n_ladder(b2, orc, opts, card):
    """N = 2^18, 2^19, 2^20 in ascending order under max_scratch_mib = 24576: waves of 384, 192 and 96 slots, so
    need_v is 24 GiB at every step and only ensure()'s `128 * N * 32 > v_align_` rule reallocates V as N grows.
    Instances (mw 0, tpb 512), one partial CTA, and (mw 1, tpb 64), two CTAs at 2^20, the last partial.

    At 2^20 each of a warp's two regions is exactly 4 GiB: B's starts in the next 4 GiB window (vb_hi = va_hi + 1) and
    the fill's 32-bit row addresses ra/rb wrap to 0 after the last store, so every B label depends on that arithmetic.
    The two instances must agree over the whole range, and an oracle sample covers every layer's A/B seam, every warp's
    first label and the tail.  The re-alignment check is a tripwire, not a proof: whether a broken rule shows depends
    on where the allocator placed the 2^19 buffer."""
    for n in LADDER:
        t0 = time.time()
        s = (LADDER_MIB << 20) // per_slot(n)
        count = large_count(s)
        c = hashlib.sha256(b"phased-large-%d" % n).digest()
        diff = orc.py_vrf_difficulty(count // 16)
        runs = {}
        for mw, tpb in LARGE_INSTANCES:
            what = f"phased<mw={mw}, tpb={tpb}> N=2^{n.bit_length() - 1} cap={LADDER_MIB} MiB"
            opts(romix_variant=PHASED, rotate_mask=mw, tpb=tpb, ctas_per_sm=0, max_scratch_mib=LADDER_MIB,
                 lowlat_max_labels=0)
            need_hbm(card, (LADDER_MIB << 20) + v_pad(n), what)
            assert predict_wave(card, n, tpb, 0, LADDER_MIB) == (s, tpb, 1)
            wave = b2.wave_slots(n)
            assert wave == s == {18: 384, 19: 192, 20: 96}[n.bit_length() - 1], (what, wave)
            (got, vrf), k = counted(b2, lambda: b2.labels_range(c, n, START, count, vrf_difficulty_=diff))
            assert k == 3, (what, "launches", k)
            runs[what] = got, vrf
        (a, va), (b, vb) = runs.values()
        same(b, a, f"N={n}: {' vs '.join(runs)}")
        assert va == vb and va is not None and va[0] - START == argmin_pos(a), (va, vb)
        pick = {count - 2, count - 1}
        for base in range(0, count, 2 * s):
            pick |= {p for p in range(base, base + 2 * s, 32)} | {base + s - 1, base + s}
        pick = np.array(sorted(p for p in pick if p < count))
        if n == 1 << 20:
            assert len(pick) <= 48
        comms = np.tile(np.frombuffer(c, dtype=np.uint8), (len(pick), 1))
        threads = max(1, min(orc.default_threads(), (8 << 30) // (128 * n)))
        same(a[pick], orc.c_labels_gather(comms, (START + pick).astype(np.uint64), n, threads=threads),
             f"N={n} oracle sample")
        assert orc.c_label32(c, va[0], n) == va[1]
        _large[n] = c, count, a
        print(f"\n[phased matrix] N={n}: wave {s}, {count} labels, {len(pick)} oracle labels ({time.time() - t0:.1f} s)")


def test_largest_layer_uncapped(b2, opts, card):
    """One call at N = 2^20 with the default budget: the largest layer the card holds.  V is aligned to the 4 GiB region
    size, so its allocation carries a pad of up to 4 GiB, and ensure() takes that pad out of its 95 % share of free HBM:
    the wave is whole warps of 256 MiB slots in 0.95 x free - 4 GiB.  wave_slots() must name the layer the call then
    runs (before the pad was budgeted, holding V shrank the next call's layer from 288 to 256 slots on an 80 GB card),
    the call must complete without ERR_OUT_OF_MEMORY, and its labels equal the capped run of test_large_n_ladder."""
    n = 1 << 20
    if n not in _large:
        pytest.fail("runs after test_large_n_ladder (its 2^20 range is the reference)")
    c, count, exp = _large[n]
    free, total = free_hbm(b2)
    opts(romix_variant=PHASED, max_scratch_mib=0, ctas_per_sm=0, lowlat_max_labels=0)
    tpb = b2.get_option("tpb")
    pred, ran_tpb, _ = predict_wave({**card, "free": free}, n, tpb, 0, 0)
    wave = b2.wave_slots(n)
    print(f"\n[phased matrix] N=2^20 uncapped: free {free / 2**30:.2f} GiB, wave {wave} (predicted {pred}), "
          f"V {wave * per_slot(n) / 2**30:.0f} GiB + 4 GiB pad")
    assert wave == pred and ran_tpb == tpb and wave < card["sms"] * 64, (wave, pred)
    assert wave * per_slot(n) + v_pad(n) <= free * HBM_SHARE, "V and its pad fit in the share"
    (got, _), k = counted(b2, lambda: b2.labels_range(c, n, START, count))
    assert k == math.ceil(count / (2 * wave)), ("launches", k, "wave", wave)
    same(got, exp, "N=2^20 uncapped vs capped")
    assert b2.wave_slots(n) == wave, "the layer does not depend on the V the engine holds"


# --------------------------------------------------------------------------------- D: occupancy-chosen CTAs
@pytest.mark.parametrize("n", (64, 1024), ids=lambda v: f"N{v}-ctas0-uncapped")
@pytest.mark.parametrize("mw,tpb", [pytest.param(*c, id=f"mw{c[0]}-tpb{c[1]}") for c in PHASED_MATRIX])
def test_occupancy_chosen_ctas(b2, orc, opts, card, ref, mw, tpb, n):
    """ctas_per_sm = 0, no cap, at N where HBM does not bind: ensure() puts the occupancy limit of CTAs on each SM, and
    its search takes a smaller CTA size where that gives strictly more slots.  The wave is a whole number of CTAs per
    SM of the size that ran, more than one for 64 and 128 threads.  Three layers and a ragged fourth; at N = 64 the
    reference is the full oracle, at N = 1024 the pipelined kernel pinned to an oracle sample."""
    r = ref(n)
    what = f"phased<mw={mw}, tpb={tpb}> N={n} ctas_per_sm=0"
    opts(romix_variant=PHASED, rotate_mask=mw, tpb=tpb, ctas_per_sm=0, max_scratch_mib=0, lowlat_max_labels=0)
    exp, ran_tpb, ran_ctas = predict_wave(card, n, tpb, 0, 0)
    wave = b2.wave_slots(n)
    assert wave == exp, (what, "wave", wave, "predicted", exp)
    assert wave == card["sms"] * ran_ctas * ran_tpb and ran_ctas == card["occ"][ran_tpb], (what, ran_tpb, ran_ctas)
    if ran_tpb in (64, 128):
        assert ran_ctas > 1, (what, ran_ctas)
    assert math.ceil(r.count / (2 * wave)) >= 4 and (r.count % (2 * wave)) % 32, (what, "layers", wave)
    vrf = run_range(b2, r, wave, f"{what} (ran tpb {ran_tpb} x {ran_ctas} CTAs per SM)")
    assert vrf == r.vrf, (what, "VRF")
