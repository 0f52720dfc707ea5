"""CPU tier: how a range job's layers are shared with queued gathers ("riders", csrc/rider_plan.cpp, plain C++ compiled
with g++ through tests/rider_plan_emul.cpp and driven layer by layer as DeviceEngine::run_job drives it).

* Riders are taken in FIFO order into at most half of a layer (whole warps), each chunk from a 32-aligned slot after
  the range segment; a gather larger than the free slots spans consecutive layers, and no later rider overtakes it.
* The range job's labels tile [0, total) in order and each layer's share drops by exactly the rider slots.
* Riders still queued when the range job has no labels left are not placed: they run as their own calls."""
import ctypes
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
U64P = ctypes.POINTER(ctypes.c_uint64)


@pytest.fixture(scope="module")
def plan_lib(tmp_path_factory):
    out = tmp_path_factory.mktemp("rider_plan") / "rider_plan_emul.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", str(out), str(ROOT / "tests" / "rider_plan_emul.cpp"),
                    str(ROOT / "go-spacemesh_b200" / "csrc" / "rider_plan.cpp")], check=True)
    L = ctypes.CDLL(str(out))
    L.emul_run.argtypes = [ctypes.c_uint32, ctypes.c_uint64, ctypes.c_uint32, U64P, U64P, ctypes.c_uint64, U64P, U64P, U64P, U64P]
    L.emul_cap.argtypes = [ctypes.c_uint32]
    L.emul_cap.restype = ctypes.c_uint32
    return L


def run(L, S, total, riders):
    """riders: list of (items, arrival layer).  Returns layers (n, 4), chunks (n, 5), placed per rider."""
    items = np.array([r[0] for r in riders] or [0], np.uint64)
    arrive = np.array([r[1] for r in riders] or [0], np.uint64)
    cap = total // 16 + sum(r[0] for r in riders) + 64
    layers, chunks = np.zeros((cap, 4), np.uint64), np.zeros((cap, 5), np.uint64)
    placed, counts = np.zeros(max(1, len(riders)), np.uint64), np.zeros(2, np.uint64)
    p = lambda a: a.ctypes.data_as(U64P)
    assert L.emul_run(S, total, len(riders), p(items), p(arrive), cap, p(layers), p(chunks), p(placed), p(counts)) == 0
    return layers[:int(counts[0])].astype(np.int64), chunks[:int(counts[1])].astype(np.int64), placed[:len(riders)].astype(np.int64)


def warps(n):
    return -(-n // 32) * 32


def check_invariants(L, S, total, riders, layers, chunks, placed):
    cap = L.emul_cap(S)
    assert cap == S // 2 // 32 * 32
    # range labels: consecutive, tiling [0, total), the rest of each layer after its rider slots
    off = 0
    for m, (range_off, n_range, range_slots, n_slots) in enumerate(layers):
        assert range_off == off and n_range > 0
        assert range_slots == warps(n_range) and n_slots % 32 == 0 and n_slots <= S
        mine = chunks[chunks[:, 0] == m]
        rider_slots = sum(warps(int(c[3])) for c in mine)
        assert rider_slots <= cap
        assert n_slots == range_slots + rider_slots
        assert n_range == min(total - off, S - rider_slots)
        # chunks: whole-warp starts, packed in order after the range segment, no overlap
        slot = range_slots
        for c in mine:
            assert c[4] == slot and c[4] % 32 == 0 and c[3] > 0
            slot += warps(int(c[3]))
        off += n_range
    assert off == total
    # riders: each item placed at most once, in item order; placed items form a prefix
    for r, (items, _) in enumerate(riders):
        mine = chunks[chunks[:, 1] == r]
        pos = 0
        for c in mine:
            assert c[2] == pos
            pos += c[3]
        assert pos == placed[r] <= items
    # FIFO: a rider's first chunk never comes before an earlier-queued rider's last chunk unless that one is placed
    order = sorted(range(len(riders)), key=lambda r: (riders[r][1], r))
    for i, a in enumerate(order):
        for b in order[i + 1:]:
            ca, cb = chunks[chunks[:, 1] == a], chunks[chunks[:, 1] == b]
            if len(cb) == 0:
                continue
            assert placed[a] == riders[a][0], "a later rider was placed while an earlier one still had items"
            # b's first chunk is in the layer of a's last chunk or later, and after it in that layer
            assert (cb[0, 0], cb[0, 4]) > (ca[-1, 0], ca[-1, 4])


@pytest.mark.parametrize("S", [64, 96, 1024, 72704])
def test_no_riders_is_todays_layering(plan_lib, S):
    total = 5 * S + 7
    layers, chunks, _ = run(plan_lib, S, total, [])
    assert len(chunks) == 0
    assert [tuple(x) for x in layers[:, :2]] == [(m * S, min(S, total - m * S)) for m in range(-(-total // S))]


def test_fifo_order_and_half_layer_cap(plan_lib):
    S = 1024   # cap 512
    riders = [(37, 0), (1, 0), (100, 0), (500, 0), (3, 0)]
    layers, chunks, placed = run(plan_lib, S, 40 * S, riders)
    check_invariants(plan_lib, S, 40 * S, riders, layers, chunks, placed)
    # layer 0: 37 (64 slots), 1 (32), 100 (128): 224 slots; 500 takes the remaining 288 and spans into layer 1
    l0 = chunks[chunks[:, 0] == 0]
    assert [tuple(c[1:4]) for c in l0] == [(0, 0, 37), (1, 0, 1), (2, 0, 100), (3, 0, 288)]
    assert layers[0, 1] == S - 512
    l1 = chunks[chunks[:, 0] == 1]
    assert [tuple(c[1:4]) for c in l1] == [(3, 288, 212), (4, 0, 3)]
    assert layers[1, 1] == S - 224 - 32
    assert layers[2, 1] == S and (placed == [r[0] for r in riders]).all()


def test_gather_spans_consecutive_layers(plan_lib):
    S = 2048   # cap 1024
    riders = [(5000, 1), (10, 2)]
    total = 30 * S
    layers, chunks, placed = run(plan_lib, S, total, riders)
    check_invariants(plan_lib, S, total, riders, layers, chunks, placed)
    big = chunks[chunks[:, 1] == 0]
    assert list(big[:, 0]) == [1, 2, 3, 4, 5] and list(big[:, 3]) == [1024] * 4 + [904]
    # the small one waits for the big one, then shares its last layer
    small = chunks[chunks[:, 1] == 1]
    assert list(small[0, [0, 2, 3, 4]]) == [5, 0, 10, layers[5, 2] + warps(904)]
    assert layers[5, 1] == S - warps(904) - 32


def test_range_positions_unchanged_under_load(plan_lib):
    rng = np.random.default_rng(7)
    for S in (64, 96, 160, 4096):
        total = int(rng.integers(3 * S, 12 * S))
        riders = [(int(rng.integers(1, 3 * S)), int(rng.integers(0, 8))) for _ in range(int(rng.integers(1, 12)))]
        layers, chunks, placed = run(plan_lib, S, total, riders)
        check_invariants(plan_lib, S, total, riders, layers, chunks, placed)


def test_leftovers_run_as_their_own_calls(plan_lib):
    S = 256   # cap 128
    # the range job has 3 layers without riders; with a 1000-item rider it lasts until its labels run out, and the rider
    # still has items then; a rider arriving after the last layer is never placed
    total = 3 * S
    riders = [(1000, 0), (7, 0), (50, 100)]
    layers, chunks, placed = run(plan_lib, S, total, riders)
    check_invariants(plan_lib, S, total, riders, layers, chunks, placed)
    assert len(layers) == -(-total // (S - 128))
    assert placed[0] == 128 * len(layers) < 1000
    assert placed[1] == 0 and placed[2] == 0


def test_tiny_layer_hosts_nothing(plan_lib):
    # a 32-slot layer has no half-layer of whole warps: riders wait for the job to end
    layers, chunks, placed = run(plan_lib, 32, 100, [(5, 0)])
    assert plan_lib.emul_cap(32) == 0 and len(chunks) == 0 and placed[0] == 0
    assert list(layers[:, 1]) == [32, 32, 32, 4]
