"""The C library's own NCCL exchange (b200post_vrf_comm_*): two PROCESSES, one GPU each, each initialises its shard and
the ranks min-reduce the VRF candidate — BASELINE.json configs[3]'s shape at world 2, with no torch in the loop.
Needs two GPUs (skipped on a single-GPU machine)."""
import ctypes
import multiprocessing as mp
import sys
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent


def _rank_main(rank, world, id_q, res_q, start, count, n):
    import importlib
    sys.path.insert(0, str(ROOT))
    b2 = importlib.import_module("go-spacemesh_b200")
    L = b2.lib()
    L.b200post_vrf_comm_init.argtypes = [ctypes.c_uint32, ctypes.c_int, ctypes.c_int, ctypes.c_char_p, ctypes.POINTER(ctypes.c_void_p)]
    L.b200post_vrf_comm_min.argtypes = [ctypes.c_void_p, ctypes.POINTER(b2.VrfNonce), ctypes.POINTER(b2.VrfNonce)]
    L.b200post_vrf_comm_free.argtypes = [ctypes.c_void_p]
    if rank == 0:
        uid = ctypes.create_string_buffer(128)
        assert L.b200post_vrf_comm_unique_id(uid) == 0, L.b200post_last_error()
        for _ in range(world - 1):
            id_q.put(uid.raw)
        ident = uid.raw
    else:
        ident = id_q.get(timeout=120)
    comm = ctypes.c_void_p()
    assert L.b200post_vrf_comm_init(rank, rank, world, ident, ctypes.byref(comm)) == 0, L.b200post_last_error()
    commitment = b2.commitment(bytes(range(32)), bytes(range(32, 64)))
    per = (count + world - 1) // world
    s, k = start + rank * per, max(0, min(per, count - rank * per))
    diff = b2.vrf_difficulty(2**20)
    _, vrf = b2.labels_range(commitment, n, s, k, provider=rank, vrf_difficulty_=diff, discard=True)
    mine = b2.VrfNonce()
    if vrf is not None:
        mine.found, mine.index = 1, vrf[0]
        ctypes.memmove(mine.label32, vrf[1], 32)
    best = b2.VrfNonce()
    assert L.b200post_vrf_comm_min(comm, ctypes.byref(mine), ctypes.byref(best)) == 0, L.b200post_last_error()
    L.b200post_vrf_comm_free(comm)
    res_q.put((rank, bool(best.found), int(best.index), bytes(best.label32)))


def test_two_processes_min_reduce_the_vrf_candidate(b2, orc, gpu_ready):
    if len(b2.providers()) < 2:
        pytest.skip("needs two GPUs")
    ctx = mp.get_context("spawn")
    id_q, res_q = ctx.Queue(), ctx.Queue()
    start, count, n = 2**32 - 700, 1500, 8192
    procs = [ctx.Process(target=_rank_main, args=(r, 2, id_q, res_q, start, count, n)) for r in range(2)]
    for p in procs:
        p.start()
    got = [res_q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    commitment = orc.py_commitment(bytes(range(32)), bytes(range(32, 64)))
    _, found, idx, l32 = orc.c_labels_range(commitment, n, start, count, orc.py_vrf_difficulty(2**20))
    for rank, f, i, lab in got:                       # every rank holds the same, correct answer
        assert f == bool(found) and (not found or (i, lab) == (idx, l32)), rank
