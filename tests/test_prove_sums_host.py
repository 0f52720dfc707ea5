"""CPU tier: proving over checksummed POST data (b200post_generate_proof_sums) without a device.

* The chunk plan (csrc/sums_plan.cpp, plain C++ compiled with g++ through tests/sums_plan_emul.cpp): over files of
  50 001, 2^16, 3·2^16 + 5 and 2^18 labels, sidecars covering all, part or none of a file, chunk_labels from 1 to more
  than the POST and 1-3 shards, the chunks tile [0, numLabels), every digest range lies in exactly one chunk and has the
  right digest, chunks respect their bound and shards are whole chunks.
* The host checks of the entry point: arguments (`sums` NULL included), missing metadata -> ERR_IO, the CPU id ->
  UNSUPPORTED, otherwise NO_DEVICE, in that order and with their texts."""
import ctypes
import importlib
import itertools
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
B = 1 << 16
U64P = ctypes.POINTER(ctypes.c_uint64)
NODE, ATX = bytes(range(32)), bytes(range(32, 64))


@pytest.fixture(scope="module")
def plan_lib(tmp_path_factory):
    out = tmp_path_factory.mktemp("sums_plan") / "sums_plan_emul.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", str(out), str(ROOT / "tests" / "sums_plan_emul.cpp"),
                    str(ROOT / "go-spacemesh_b200" / "csrc" / "sums_plan.cpp")], check=True)
    L = ctypes.CDLL(str(out))
    L.emul_plan.argtypes = [ctypes.c_uint32, U64P, U64P, U64P, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint64, U64P, U64P, U64P, U64P]
    return L


def plan(L, labels, covered, chunk, shards):
    n = len(labels)
    first_slot = np.cumsum([0] + [-(-c // B) for c in covered])[:-1].astype(np.uint64)
    lab, cov = np.array(labels, dtype=np.uint64), np.array(covered, dtype=np.uint64)
    cap = sum(-(-x // B) for x in labels) + 2 * n + 8
    ranges, chunks = np.zeros((cap, 4), np.uint64), np.zeros((cap, 4), np.uint64)
    sh, counts = np.zeros((shards, 4), np.uint64), np.zeros(4, np.uint64)
    p = lambda a: a.ctypes.data_as(U64P)
    assert L.emul_plan(n, p(lab), p(cov), p(first_slot), chunk, shards, cap, p(ranges), p(chunks), p(sh), p(counts)) == 0
    nr, nc = int(counts[0]), int(counts[1])
    return ranges[:nr].astype(np.int64), chunks[:nc].astype(np.int64), sh.astype(np.int64), int(counts[2]), int(counts[3]), first_slot


def expected_ranges(labels, covered, first_slot):
    """(first, count, covered, digest slot) of every digest range and uncovered piece, by brute force over the grid."""
    out, base = [], 0
    for f, (n, c) in enumerate(zip(labels, covered)):
        cuts = sorted({0, n, min(c, n)} | set(range(B, n, B)))
        for lo, hi in zip(cuts, cuts[1:]):
            out.append((base + lo, hi - lo, int(hi <= c), int(first_slot[f]) + lo // B if hi <= c else -1))
        base += n
    return out


FILES = [
    ([50_001] * 3 + [3 * B - 3 * 50_001], [50_001, 0, 20_000, 3 * B - 3 * 50_001]),   # the GPU tests' 3 x 2^16 POST
    ([B, B, B], [B, B, 0]),
    ([3 * B + 5, 3 * B + 5], [3 * B + 5, 2 * B + 7]),
    ([1 << 18], [(1 << 18) - 1]),
    ([1 << 18, 50_001], [B, 50_001]),
]
CHUNKS = (1, 4099, B - 1, B, B + 1, 2 * B + 3, 1 << 22)


@pytest.mark.parametrize("files", range(len(FILES)))
def test_chunk_plan_tiles_the_post_in_whole_ranges(plan_lib, files):
    labels, covered = FILES[files]
    total = sum(labels)
    for chunk, shards in itertools.product(CHUNKS, (1, 2, 3)):
        ranges, chunks, sh, max_chunk, max_ranges, first_slot = plan(plan_lib, labels, covered, chunk, shards)
        assert [tuple(int(v) for v in r[:3]) + (int(r[3]) if r[2] else -1,) for r in ranges] == expected_ranges(labels, covered, first_slot)
        bound = max(chunk, B)
        # chunks tile [0, total), each a run of whole ranges within the bound
        assert chunks[0, 0] == 0 and chunks[-1, 0] + chunks[-1, 1] == total
        assert (chunks[1:, 0] == chunks[:-1, 0] + chunks[:-1, 1]).all()
        assert (chunks[:, 1] <= bound).all() and (chunks[:, 1] > 0).all()
        assert chunks[0, 2] == 0 and chunks[-1, 3] == len(ranges) and (chunks[1:, 2] == chunks[:-1, 3]).all()
        for c in chunks:
            rs = ranges[c[2]:c[3]]
            assert rs[0, 0] == c[0] and rs[:, 1].sum() == c[1]
            # greedy: the next range would not have fitted
            if c[3] < len(ranges):
                assert c[1] + ranges[c[3], 1] > bound
        assert max_chunk == chunks[:, 1].max() and max_ranges == (chunks[:, 3] - chunks[:, 2]).max()
        # every range in exactly one chunk
        owner = np.zeros(len(ranges), int)
        for c in chunks:
            owner[c[2]:c[3]] += 1
        assert (owner == 1).all()
        # shards: whole chunks, contiguous, chunk counts within one of each other (earlier ones take the odd chunks)
        counts = sh[:, 1] - sh[:, 0]
        assert sh[0, 0] == 0 and sh[-1, 1] == len(chunks) and (sh[1:, 0] == sh[:-1, 1]).all()
        assert counts.max() - counts.min() <= 1 and list(counts) == sorted(counts, reverse=True)
        for s in sh:
            if s[1] > s[0]:
                assert s[2] == chunks[s[0], 0] and s[3] == chunks[s[1] - 1, 0] + chunks[s[1] - 1, 1]
            else:
                assert s[2] == s[3]


# ----------------------------------------------------------------------------------------------------- host errors
@pytest.fixture()
def mods(b2):
    return importlib.import_module("go-spacemesh_b200.setup"), importlib.import_module("go-spacemesh_b200.prove")


def _call(pr, su, data_dir, providers, n_providers, with_check=True, with_sums=True, with_out=True):
    """The C call itself, so that NULL pointers can be passed."""
    L = pr._bind()
    out, meta, chk, rep, c = pr._ProofOut(), pr._Meta(), pr._ProveCheck(), pr._SumsReport(), pr._c_cfg(su.PostConfig())
    rep.bad_blocks = 99
    opts = pr._ProveOpts(0, 16, 0, ctypes.cast(None, pr.POW_PROVE_FN), None, 2, None, 0)
    arr = (ctypes.c_uint32 * len(providers))(*providers) if providers is not None else None
    rc = L.b200post_generate_proof_sums(str(data_dir).encode() if data_dir is not None else None, bytes(32), ctypes.byref(c),
                                        ctypes.byref(opts), arr, n_providers, None, ctypes.byref(out) if with_out else None,
                                        ctypes.byref(meta), ctypes.byref(chk) if with_check else None,
                                        ctypes.byref(rep) if with_sums else None, None)
    return rc, rep


def _post(su, d):
    """Metadata of a 2 x 512-label POST (no label files: the device errors come before any read)."""
    o = su.PostSetupOpts(data_dir=str(d), num_units=2, max_file_size=4096, provider_id=0, scrypt_n=2)
    su.PostSetupManager().prepare_initializer(o, NODE, ATX)
    return o.data_dir


def test_argument_checks(b2, mods, tmp_path):
    su, pr = mods
    d = _post(su, tmp_path / "p")
    L = pr._bind()
    for provs, n in ((None, 1), ([0], 0), ([0, 0], -3)):
        assert _call(pr, su, d, provs, n)[0] == b2.ERR_INVALID_ARGUMENT, (provs, n)
    for kw in (dict(with_sums=False), dict(with_check=False), dict(with_out=False)):
        assert _call(pr, su, d, [0], 1, **kw)[0] == b2.ERR_INVALID_ARGUMENT, kw
        assert L.b200post_last_error() == b"invalid argument"
    assert _call(pr, su, None, [0], 1)[0] == b2.ERR_INVALID_ARGUMENT
    # the NULL check comes before the metadata is read
    assert _call(pr, su, tmp_path / "nowhere", [0], 1, with_sums=False)[0] == b2.ERR_INVALID_ARGUMENT
    with pytest.raises(b2.B200PostError) as e:
        pr.generate_proof_sums(d, bytes(32), su.PostConfig(), providers=[], pow="skip")
    assert e.value.code == b2.ERR_INVALID_ARGUMENT
    for provs in ([b2.CPU_PROVIDER_ID], [b2.CPU_PROVIDER_ID] * 3):
        for pow_ in ("skip", "builtin"):
            with pytest.raises(b2.B200PostError) as e:
                pr.generate_proof_sums(d, bytes(32), su.PostConfig(), providers=provs, pow=pow_)
            assert e.value.code == b2.ERR_UNSUPPORTED, (provs, pow_)
            assert e.value.sums.blocks_checked == 0 and e.value.sums.bad == []


def test_missing_metadata_is_an_io_error_before_the_device(b2, mods, tmp_path):
    su, pr = mods
    (tmp_path / "empty").mkdir()
    for provs in ([0], [0, 1], [b2.CPU_PROVIDER_ID, 0]):
        for pow_ in ("skip", "builtin"):
            with pytest.raises(b2.B200PostError) as e:
                pr.generate_proof_sums(str(tmp_path / "empty"), bytes(32), su.PostConfig(), providers=provs, pow=pow_)
            assert e.value.code == su.ERR_IO and "metadata" in str(e.value), (provs, pow_)
    rc, rep = _call(pr, su, tmp_path / "empty", [0], 1)
    assert rc == su.ERR_IO and rep.bad_blocks == 0   # the report is cleared past the argument checks


def test_no_device_no_cpu_path(b2, mods, tmp_path):
    su, pr = mods
    if b2.providers():
        pytest.skip("a CUDA device is present: the no-device contract is covered on CPU-only boxes")
    d = _post(su, tmp_path / "p")
    for provs in ([0], [0, 0], [0, 1, 2]):
        for pow_ in ("skip", "builtin"):
            with pytest.raises(b2.B200PostError) as e:
                pr.generate_proof_sums(d, bytes(32), su.PostConfig(), providers=provs, pow=pow_)
            assert e.value.code == b2.ERR_NO_DEVICE, (provs, pow_)
