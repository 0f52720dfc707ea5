"""GPU tier: every compiled ROMix (K2) instance, on the path it names, against the oracle.

The launch table in label_kernels.cu compiles the pipelined kernel for rotate mask x CTA size x double-round unroll,
the classic kernels for variant x rotate mask x CTA size, and the low-latency kernel for each rotate mask.  Which one
runs is decided at run time by the options, the job size and the HBM budget, so a test that only sets options proves
nothing about the kernel that ran.  Every case here therefore also asserts:
  - the ROMix launch count of the call (b2.romix_time): M + 1 for a fresh pipelined call over M layers, M when it
    resumes a pre-filled first layer, M for a classic variant, 1 for the low-latency kernel;
  - the CTA size, through the wave: with ctas_per_sm = 1 at an N where HBM is not the limit, ensure() keeps the
    requested CTA size and the wave is exactly sm_count x tpb.

Options are process-global; every test and fixture here restores the values it found.
"""
import hashlib
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# (rotate_mask, tpb, dr_unroll) of every romix_pipe_kernel instance, and (romix_variant, rotate_mask, tpb) of every
# romix_kernel instance that computes labels (variant 3, ROMIX_NOMEM, is an ALU probe).  test_romix_launch_table.py
# checks these lists against the launch table.
PIPE_MATRIX = [(mw, tpb, dr) for mw in (0, 1) for tpb in (64, 128, 256, 512) for dr in (1, 4)]
CLASSIC_MATRIX = [(variant, mw, tpb) for variant in (0, 1, 2) for mw in (0, 1) for tpb in (128, 256)]
LOWLAT_MASKS = (0, 1)
PIPELINED = 4
MATRIX_N = (2, 64, 1024)             # N <= 1024: the register file, not HBM, bounds the layer
OPTION_KEYS = ("romix_variant", "rotate_mask", "tpb", "dr_unroll", "ctas_per_sm", "max_scratch_mib",
               "speculate_next", "lowlat_max_labels")


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


@pytest.fixture
def opts(b2, gpu_ready):
    """opts(**kw) sets options for the rest of the test; all of OPTION_KEYS are restored afterwards."""
    old = {k: b2.get_option(k) for k in OPTION_KEYS}

    def set_(**kw):
        for k, v in kw.items():
            b2.set_option(k, v)
    yield set_
    set_(**old)


@pytest.fixture(scope="module")
def sms(gpu_ready):
    return gpu_ready[0]["sm_count"]


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


# ---------------------------------------------------------------------------------------------------- A/B: ranges
class Plan:
    """One commitment and one index range per N, shared by every configuration of matrices A and B:
    call 1 = [start, start + count1) covers >= 4 layers at the largest wave (which arms the speculative fill) and ends
    in a ragged layer; call 2 = the continuation [start + count1, start + count1 + count2); call 3 = a gather of more
    than one layer, mostly over the range's indices, every 5th item with its own commitment and index."""

    TAIL1, TAIL2, GATHER_EXTRA = 1037, 555, 333     # not multiples of 32 or of any CTA size

    def __init__(self, b2, orc, n, wmax):
        self.n, self.wmax = n, wmax
        self.c = hashlib.sha256(b"romix-matrix-%d" % n).digest()
        self.start = 2**32 + 4099
        self.count1 = 3 * wmax + self.TAIL1
        self.count2 = wmax + self.TAIL2
        # ~64 labels under each threshold: the VRF minimum is a merge over many CTAs and layers
        self.diff1 = orc.py_vrf_difficulty(self.count1 // 64)
        self.diff2 = orc.py_vrf_difficulty(self.count2 // 64)
        self.exp1 = orc.c_labels_range(self.c, n, self.start, self.count1, self.diff1)
        self.exp2 = orc.c_labels_range(self.c, n, self.start + self.count1, self.count2, self.diff2)
        assert self.exp1[1] and self.exp2[1]
        rng = np.random.default_rng(n)
        g = wmax + self.GATHER_EXTRA
        pos = rng.choice(self.count1 + self.count2, g, replace=False)
        self.g_idx = (self.start + pos).astype(np.uint64)
        self.g_comm = np.tile(np.frombuffer(self.c, dtype=np.uint8), (g, 1))
        self.g_exp = np.concatenate([self.exp1[0], self.exp2[0]])[pos]
        own = np.arange(g) % 5 == 2
        self.g_comm[own] = rng.integers(0, 256, (own.sum(), 32), dtype=np.uint8)
        self.g_idx[own] = rng.integers(0, 2**64 - 1, own.sum(), dtype=np.uint64)
        self.g_exp[own] = orc.c_labels_gather(self.g_comm[own], self.g_idx[own], n)

    def run(self, b2, what, layers_of, resumes):
        """The three calls, each checked against the oracle and for its launch count.  layers_of(count) = layers of a
        call; resumes = the continuation consumes the pre-filled first layer (pipelined kernel only)."""
        fresh = 1 if resumes else 0   # a pipelined call makes one launch more than it has layers (the drain)
        (got, vrf), k = counted(b2, lambda: b2.labels_range(self.c, self.n, self.start, self.count1, vrf_difficulty_=self.diff1))
        assert k == layers_of(self.count1) + fresh, (what, "range launches", k)
        same(got, self.exp1[0], f"{what} range")
        assert vrf == self.exp1[2:], (what, "range VRF")
        (got, vrf), k = counted(b2, lambda: b2.labels_range(self.c, self.n, self.start + self.count1, self.count2,
                                                             vrf_difficulty_=self.diff2))
        assert k == layers_of(self.count2), (what, "continuation launches", k)
        same(got, self.exp2[0], f"{what} continuation")
        assert vrf == self.exp2[2:], (what, "continuation VRF")
        got, k = counted(b2, lambda: b2.labels_gather(self.g_comm, self.g_idx, self.n))
        assert layers_of(len(self.g_idx)) >= 2
        assert k == layers_of(len(self.g_idx)) + fresh, (what, "gather launches", k)
        same(got, self.g_exp, f"{what} gather")


@pytest.fixture(scope="module")
def plan(b2, orc, gpu_ready):
    """plan(n): the shared Plan of scrypt-N n, built on first use."""
    cache = {}

    def get(n):
        if n not in cache:
            # the largest wave of any configuration the matrices run at this N
            wmax = 0
            cfgs = [dict(romix_variant=PIPELINED, rotate_mask=mw, tpb=tpb, dr_unroll=dr, ctas_per_sm=ctas)
                    for mw, tpb, dr in PIPE_MATRIX for ctas in (1, 2)]
            cfgs += [dict(romix_variant=v, rotate_mask=mw, tpb=tpb, ctas_per_sm=1) for v, mw, tpb in CLASSIC_MATRIX]
            for cfg in cfgs:
                with Opt(b2, max_scratch_mib=0, **cfg):
                    wmax = max(wmax, b2.wave_slots(n))
            cache[n] = Plan(b2, orc, n, wmax)
        return cache[n]
    return get


def _check_shape(p, wave, tpb, what):
    assert math.ceil(p.count1 / wave) >= 4, what
    for count in (p.count1, p.count2):
        tail = count % wave
        assert tail % 32 and tail % tpb, (what, "ragged last layer", tail)


@pytest.mark.parametrize("ctas", (1, 2), ids=lambda v: f"ctas{v}")
@pytest.mark.parametrize("n", MATRIX_N, ids=lambda v: f"N{v}")
@pytest.mark.parametrize("mw,tpb,dr", [pytest.param(*c, id=f"mw{c[0]}-tpb{c[1]}-dr{c[2]}") for c in PIPE_MATRIX])
def test_pipelined_instance(b2, opts, plan, sms, mw, tpb, dr, n, ctas):
    """romix_pipe_kernel<mw, tpb, dr> over a fresh multi-layer range, its continuation from the speculative fill, and a
    multi-layer gather.  ctas_per_sm = 2 puts two CTAs on an SM where the occupancy allows it."""
    p = plan(n)
    what = f"pipe<mw={mw}, tpb={tpb}, dr={dr}> N={n} ctas_per_sm={ctas}"
    opts(romix_variant=PIPELINED, rotate_mask=mw, tpb=tpb, dr_unroll=dr, ctas_per_sm=ctas, max_scratch_mib=0,
         speculate_next=1, lowlat_max_labels=0)
    wave = b2.wave_slots(n)
    if ctas == 1:
        assert wave == sms * tpb, (what, wave)
    else:
        assert wave % (sms * tpb) == 0 and wave >= sms * tpb, (what, wave)
    _check_shape(p, wave, tpb, what)
    p.run(b2, what, lambda count: math.ceil(count / wave), resumes=True)


@pytest.mark.parametrize("n", MATRIX_N, ids=lambda v: f"N{v}")
@pytest.mark.parametrize("variant,mw,tpb", [pytest.param(*c, id=f"v{c[0]}-mw{c[1]}-tpb{c[2]}") for c in CLASSIC_MATRIX])
def test_classic_variant(b2, opts, plan, sms, variant, mw, tpb, n):
    """romix_kernel<variant, mw, tpb>: one launch per layer over the same multi-layer ranges and gather."""
    p = plan(n)
    what = f"classic<variant={variant}, mw={mw}, tpb={tpb}> N={n}"
    opts(romix_variant=variant, rotate_mask=mw, tpb=tpb, ctas_per_sm=1, max_scratch_mib=0, speculate_next=1)
    wave = b2.wave_slots(n)
    assert wave == sms * tpb, (what, wave)
    _check_shape(p, wave, tpb, what)
    p.run(b2, what, lambda count: math.ceil(count / wave), resumes=False)


# ---------------------------------------------------------------------------------------------------- C: low latency
@pytest.fixture(scope="module")
def lowlat_items(orc, sms):
    """items(n): 32 W + 1 gather items (W = 4 x SMs, the kernel's warp count) with their own commitments, the first
    at index 2^64 - 1, and their oracle labels."""
    cache = {}

    def get(n):
        if n not in cache:
            m = 32 * 4 * sms + 1
            rng = np.random.default_rng(n + 7)
            comms = rng.integers(0, 256, (m, 32), dtype=np.uint8)
            idx = rng.integers(0, 2**64 - 1, m, dtype=np.uint64)
            idx[0] = 2**64 - 1
            cache[n] = comms, idx, orc.c_labels_gather(comms, idx, n)
        return cache[n]
    return get


@pytest.mark.parametrize("n", (2, 8192), ids=lambda v: f"N{v}")
@pytest.mark.parametrize("mw", LOWLAT_MASKS, ids=lambda v: f"mw{v}")
def test_low_latency_slot_mapping(b2, opts, lowlat_items, sms, mw, n):
    """romix_lowlat_kernel<mw>: slot = lane * W + warp with W = min(n, 4 x SMs); sizes around every multiple of W up
    to the kernel's capacity of 32 W, and one label more, which must take the pipelined kernel instead."""
    w = 4 * sms
    comms, idx, exp = lowlat_items(n)
    opts(romix_variant=PIPELINED, rotate_mask=mw, lowlat_max_labels=32 * w, max_scratch_mib=0)
    for m in (1, 31, 33, w - 1, w, w + 1, 2 * w + 1, 32 * w):
        got, k = counted(b2, lambda: b2.labels_gather(comms[:m], idx[:m], n))
        assert k == 1, (mw, n, m, "launches", k)
        same(got, exp[:m], f"lowlat<mw={mw}> N={n} n={m}")
    m = 32 * w + 1
    layers = math.ceil(m / b2.wave_slots(n))
    got, k = counted(b2, lambda: b2.labels_gather(comms, idx, n))
    assert k == layers + 1, (mw, n, m, "a job over 32 W labels must take the pipelined kernel", k)
    same(got, exp, f"pipelined fallback mw={mw} N={n} n={m}")


# ---------------------------------------------------------------------------------------------------- D: N = 2^20
def test_largest_n_over_several_layers(b2, orc, opts):
    """N = 2^20: each warp's scratch region is exactly 4 GiB and V is aligned to 4 GiB, which the pipelined kernel's
    32-bit {lo, hi} address arithmetic relies on.  Two pipelined instances over more than one layer and one classic
    variant agree byte for byte, and a sample (layer seams, ragged tail, random) agrees with the oracle.  The phased kernel
    (the default) at this N, where its B regions start in the next 4 GiB window, is tested by
    test_gpu_romix_phased_matrix.py::test_large_n_ladder."""
    n = 1 << 20
    c = hashlib.sha256(b"largest-n-layers").digest()
    start = 2**40 - 3
    opts(romix_variant=PIPELINED, rotate_mask=0, dr_unroll=4, lowlat_max_labels=0, max_scratch_mib=0)
    wave = b2.wave_slots(n)
    count = wave + 37
    runs = {}
    for mw, dr in ((0, 4), (1, 1)):
        opts(rotate_mask=mw, dr_unroll=dr)
        w = b2.wave_slots(n)
        layers = math.ceil(count / w)
        assert layers >= 2, (mw, dr, w)
        runs[f"pipe mw={mw} dr={dr}"], k = counted(b2, lambda: b2.labels_range(c, n, start, count)[0])
        assert k == layers + 1, (mw, dr, "launches", k)
    opts(romix_variant=1, rotate_mask=0, dr_unroll=4, tpb=128)
    w = b2.wave_slots(n)
    runs["classic variant 1"], k = counted(b2, lambda: b2.labels_range(c, n, start, count)[0])
    assert k == math.ceil(count / w), ("classic launches", k)
    names = list(runs)
    for name in names[1:]:
        same(runs[name], runs[names[0]], f"N=2^20 {name} vs {names[0]}")
    rng = np.random.default_rng(20)
    pick = np.unique(np.concatenate([[0, 1, wave - 2, wave - 1, wave, wave + 1, count - 2, count - 1],
                                     rng.integers(0, count, 32)]))
    comms = np.tile(np.frombuffer(c, dtype=np.uint8), (len(pick), 1))
    exp = orc.c_labels_gather(comms, (start + pick).astype(np.uint64), n, threads=4)   # 128 MiB per oracle thread
    same(runs[names[0]][pick], exp, "N=2^20 oracle sample")


# ---------------------------------------------------------------------------------------------------- E: N = 8192
def test_hbm_bound_cta_size_choice_at_full_n(b2, orc, opts):
    """At N = 8192 HBM bounds the layer and ensure() picks the CTA size itself.  From every requested tpb, one full
    wave plus a ragged tail equals the default configuration byte for byte, and a sample equals the oracle."""
    n = 8192
    c = hashlib.sha256(b"hbm-bound").digest()
    start = 2**34 + 5
    opts(romix_variant=PIPELINED, rotate_mask=0, dr_unroll=4, ctas_per_sm=0, max_scratch_mib=0, lowlat_max_labels=0)
    default_tpb = b2.get_option("tpb")
    waves = {}
    for tpb in (512, 256, 128, 64):
        opts(tpb=tpb)
        waves[tpb] = b2.wave_slots(n)
    count = max(waves.values()) + 1037
    opts(tpb=default_tpb)
    ref, k = counted(b2, lambda: b2.labels_range(c, n, start, count)[0])
    assert k == math.ceil(count / waves[default_tpb]) + 1
    for tpb in (512, 256, 128, 64):
        opts(tpb=tpb)
        got, k = counted(b2, lambda: b2.labels_range(c, n, start, count)[0])
        assert k == math.ceil(count / waves[tpb]) + 1 >= 3, (tpb, waves[tpb], "launches", k)
        same(got, ref, f"N=8192 requested tpb={tpb} (wave {waves[tpb]})")
    rng = np.random.default_rng(8192)
    w = waves[default_tpb]
    pick = np.unique(np.concatenate([[0, w - 1, w, count - 1], rng.integers(0, count, 196)]))
    comms = np.tile(np.frombuffer(c, dtype=np.uint8), (len(pick), 1))
    same(ref[pick], orc.c_labels_gather(comms, (start + pick).astype(np.uint64), n), "N=8192 oracle sample")


# ---------------------------------------------------------------------------------------------------- F: VRF
@pytest.mark.parametrize("path", ("pipelined", "low-latency", "classic"))
def test_vrf_threshold_at_every_word_depth(b2, orc, opts, sms, path):
    """K3 (cand_less, warp_argmin) and K4 (vrf_merge_kernel) compare label32 with the threshold word by word, strictly.
    Thresholds built from the range's minimum L make every one of the 8 words decide the comparison."""
    n, start = 2, 2**33 + 11
    opts(romix_variant=PIPELINED, rotate_mask=0, dr_unroll=4, max_scratch_mib=0, lowlat_max_labels=0)
    if path == "pipelined":
        opts(tpb=64, ctas_per_sm=1)
        count = 2 * sms * 64 + 1037
        launches = math.ceil(count / b2.wave_slots(n)) + 1
        assert launches == 4
    elif path == "low-latency":
        count = 128 * sms - 7                 # the kernel's 32 labels per warp over 4 x SMs warps, ragged
        opts(lowlat_max_labels=count)
        assert b2.wave_slots(n) >= count
        launches = 1
    else:
        opts(romix_variant=1, tpb=128, ctas_per_sm=1)
        count = 2 * sms * 128 + 1037
        launches = math.ceil(count / b2.wave_slots(n))
        assert launches == 3
    c = hashlib.sha256(path.encode()).digest()
    _, found, li, L = orc.c_labels_range(c, n, start, count, b"\xff" * 32)
    assert found

    def vrf(words):
        diff = b"".join(int(x).to_bytes(4, "big") for x in words) if not isinstance(words, bytes) else words
        (_, got), k = counted(b2, lambda: b2.labels_range(c, n, start, count, vrf_difficulty_=diff, discard=True))
        assert k == launches, (path, "launches", k)
        return got

    assert vrf(L) is None, "the comparison is strict"
    assert vrf((int.from_bytes(L, "big") + 1).to_bytes(32, "big")) == (li, L)
    lw = [int.from_bytes(L[4 * k: 4 * k + 4], "big") for k in range(8)]
    for k in range(8):
        if lw[k] < 0xFFFFFFFF:
            assert vrf(lw[:k] + [lw[k] + 1] + [0] * (7 - k)) == (li, L), (path, "word", k, "+1")
        if lw[k] > 0:
            assert vrf(lw[:k] + [lw[k] - 1] + [0xFFFFFFFF] * (7 - k)) is None, (path, "word", k, "-1")
