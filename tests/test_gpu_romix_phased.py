"""GPU tier: the phased ROMix layer (romix_variant 5, romix_phased_kernel) against the oracle.

A phased layer holds two labels per resident slot: thread t runs slot t (A) and slot t + S (B), S = wave_slots, and a warp
whose B slots lie past the layer runs A alone.  Every compiled instance runs over several layers with
a ragged tail, and the edges of the layer mapping are checked one by one: a partial layer without B, a layer of exactly
2 x wave_slots, a gather with per-item commitments and a compare job (K3c).  Each case asserts its ROMix launch count:
one per layer, so the phased kernel, not the low-latency or pipelined one, computed the labels.
"""
import hashlib
import importlib
import math
import shutil
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PHASED = 5
# (rotate_mask, tpb) of every romix_phased_kernel instance; test_romix_phased_launch_table.py checks it against the table
PHASED_MATRIX = [(mw, tpb) for mw in (0, 1) for tpb in (64, 128, 256, 512)]
OPTION_KEYS = ("romix_variant", "rotate_mask", "tpb", "ctas_per_sm", "max_scratch_mib", "lowlat_max_labels")
NODE, ATX = bytes(range(40, 72)), bytes(range(3, 35))


@pytest.fixture
def opts(b2, gpu_ready):
    old = {k: b2.get_option(k) for k in OPTION_KEYS}

    def set_(**kw):
        for k, v in kw.items():
            b2.set_option(k, v)
    yield set_
    for k, v in old.items():
        b2.set_option(k, v)


@pytest.fixture(scope="module")
def sms(gpu_ready):
    return gpu_ready[0]["sm_count"]


def counted(b2, fn):
    b2.romix_time(reset=True)
    out = fn()
    return out, b2.romix_time()[1]


def same(got, exp, what):
    assert got.shape == exp.shape, what
    bad = np.flatnonzero((got != exp).any(axis=1))
    assert bad.size == 0, f"{what}: {bad.size} of {len(exp)} labels differ, first at row {bad[0]}"


@pytest.mark.parametrize("n", (2, 1024), ids=lambda v: f"N{v}")
@pytest.mark.parametrize("mw,tpb", [pytest.param(*c, id=f"mw{c[0]}-tpb{c[1]}") for c in PHASED_MATRIX])
def test_phased_instance(b2, orc, opts, sms, mw, tpb, n):
    """romix_phased_kernel<mw, tpb> over three layers and a ragged fourth in which only the first four warps have a B,
    with the VRF candidate merged over all of them."""
    opts(romix_variant=PHASED, rotate_mask=mw, tpb=tpb, ctas_per_sm=1, max_scratch_mib=0, lowlat_max_labels=0)
    wave = b2.wave_slots(n)
    assert wave == sms * tpb, (mw, tpb, wave)
    count = 3 * 2 * wave + wave + 101             # tail: wave + 128 slots
    c = hashlib.sha256(b"phased-%d-%d-%d" % (mw, tpb, n)).digest()
    start = 2**32 + 4099
    diff = orc.py_vrf_difficulty(count // 64)
    exp, found, idx, l32 = orc.c_labels_range(c, n, start, count, diff)
    assert found
    (got, vrf), k = counted(b2, lambda: b2.labels_range(c, n, start, count, vrf_difficulty_=diff))
    assert k == 4, (mw, tpb, "launches", k)
    same(got, exp, f"phased<mw={mw}, tpb={tpb}> N={n}")
    assert vrf == (idx, l32)


@pytest.mark.parametrize("extra", (-1, 0, 37), ids=lambda v: f"wave{v:+d}" if v != -1 else "small")
def test_partial_layer_without_b(b2, orc, opts, sms, extra):
    """One partial layer: 5 labels (one warp, no B), wave_slots labels (every thread A alone), wave_slots + 37 (only the
    first two warps have a B)."""
    opts(romix_variant=PHASED, tpb=64, ctas_per_sm=1, max_scratch_mib=0, lowlat_max_labels=0)
    count = 5 if extra < 0 else b2.wave_slots(512) + extra
    c = hashlib.sha256(b"phased-partial-%d" % count).digest()
    exp = orc.c_labels_range(c, 512, 2**35 - 17, count)[0]
    (got, _), k = counted(b2, lambda: b2.labels_range(c, 512, 2**35 - 17, count))
    assert k == 1
    same(got, exp, f"partial layer of {count}")


def test_layer_of_exactly_two_waves(b2, orc, opts, sms):
    """2 x wave_slots labels are one full layer (one launch, every thread with A and B); one label more takes a second."""
    n = 64
    opts(romix_variant=PHASED, tpb=128, ctas_per_sm=1, max_scratch_mib=0, lowlat_max_labels=0)
    wave = b2.wave_slots(n)
    c = hashlib.sha256(b"phased-two-waves").digest()
    exp = orc.c_labels_range(c, n, 7, 2 * wave + 1)[0]
    (got, _), k = counted(b2, lambda: b2.labels_range(c, n, 7, 2 * wave))
    assert k == 1
    same(got, exp[:-1], "layer of exactly 2 x wave_slots")
    (got, _), k = counted(b2, lambda: b2.labels_range(c, n, 7, 2 * wave + 1))
    assert k == 2
    same(got, exp, "2 x wave_slots + 1")


def test_gather_with_per_item_commitments(b2, orc, opts, sms):
    """A gather over two layers and a ragged third, every item with its own commitment and index."""
    n = 256
    opts(romix_variant=PHASED, tpb=64, ctas_per_sm=1, max_scratch_mib=0, lowlat_max_labels=0)
    wave = b2.wave_slots(n)
    m = 2 * 2 * wave + 333
    rng = np.random.default_rng(5)
    comms = rng.integers(0, 256, (m, 32), dtype=np.uint8)
    idx = rng.integers(0, 2**64 - 1, m, dtype=np.uint64)
    idx[0] = 2**64 - 1
    got, k = counted(b2, lambda: b2.labels_gather(comms, idx, n))
    assert k == 3
    same(got, orc.c_labels_gather(comms, idx, n), "phased gather")


def test_compare_job(b2, opts, tmp_path):
    """K3c after a phased K2: a POST written by the pipelined layer, checked in full by the phased one over layers of 128
    labels (64 slots, so a layer of 65 to 127 labels has B in its first warps only).  Clean data passes; flipped labels are
    found at their positions."""
    su = importlib.import_module("go-spacemesh_b200.setup")
    opts(romix_variant=4, lowlat_max_labels=0, max_scratch_mib=0)
    d = tmp_path / "post"
    per_file = 660
    mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=per_file, max_num_units=10))
    mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=3, max_file_size=16 * per_file, provider_id=0,
                                             scrypt_n=64, compute_batch_size=1 << 16), NODE, ATX)
    mgr.start_session()
    assert mgr.status().state == su.STATE_COMPLETE
    opts(romix_variant=PHASED, max_scratch_mib=1)           # 64 slots of two 8 KiB scratchpads: 128-label layers
    assert b2.wave_slots(64) == 64
    (r, k) = counted(b2, lambda: su.verify_pos(str(d), fraction=100))
    assert r.code == su.OK and r.labels_checked == 3 * per_file
    assert k >= math.ceil(3 * per_file / 128)
    bad = tmp_path / "bad"
    shutil.copytree(d, bad)
    victims = [0, 127, 128, per_file + 659, 2 * per_file + 641]
    for i in victims:
        p = Path(bad) / f"postdata_{i // per_file}.bin"
        with open(p, "r+b") as f:
            f.seek((i % per_file) * 16 + 5)
            v = f.read(1)[0]
            f.seek(-1, 1)
            f.write(bytes([v ^ 8]))
    r = su.verify_pos(str(bad), fraction=100)
    assert r.code == su.ERR_LABEL_MISMATCH and r.bad_index == victims
