"""GPU tier: several identities in one call (b200post_k2pow_search_jobs, b200post_generate_proofs).

* The job search gives, job by job, the pows of b200post_k2pow_search_group_range for each identity, including more
  jobs than one batch holds and a device list of [0, 0]; a few are spot-checked against the RandomX oracle.
* Sharing is real: M identities with one group each fill one device batch together, where M separate searches run M.
* Every item of generate_proofs equals its one-identity call byte for byte (proof, labels scanned, report, status and
  text), under SKIP and under BUILTIN at an easy difficulty, for parallel_scans 1 and 3, the items in either order and
  providers [0] and [0, 0].  The items: proofs in window 0 and first in window 2, one with no proof in the windows
  tried, a missing directory, an N = 8192 POST and forged hits below the winner's K2-th hit (dropped and reported when
  checked).  Every returned proof passes verify_batch.
* A preset cancel returns CANCELLED and no item reports a proof."""
import contextlib
import ctypes
import importlib
import shutil
from pathlib import Path

import numpy as np
import pytest

from oracle import pyrandomx as orx

pytestmark = pytest.mark.gpu

ATX = bytes(range(90, 122))
LPU, PER_FILE = 1 << 12, 3001
K1, K2, NONCES, WINDOWS = 26, 37, 16, 3
CHUNK = 2053
EASY = b"\x3f" + b"\xff" * 31          # BUILTIN at 1 SU: a hash passes with probability 1/4
ERR_IO = 12                            # B200POST_ERR_IO (include/b200post_setup.h)


@contextlib.contextmanager
def options(b2, **values):
    before = {k: b2.get_option(k) for k in values}
    try:
        for k, v in values.items():
            b2.set_option(k, v)
        yield
    finally:
        for k, v in before.items():
            b2.set_option(k, v)


def _rate(r: int) -> bytes:
    return (2**256 // r).to_bytes(32, "big")


def _node(i: int) -> bytes:
    return bytes((7 * i + j) % 256 for j in range(32))


@pytest.fixture(scope="module")
def mods(b2, gpu_ready):
    return (importlib.import_module("go-spacemesh_b200.setup"), importlib.import_module("go-spacemesh_b200.prove"),
            importlib.import_module("go-spacemesh_b200.verify"), importlib.import_module("go-spacemesh_b200.k2pow"))


# ------------------------------------------------------------------------------------------------- the job search
def test_job_search_equals_the_group_searches(mods, b2):
    """3 identities x 50 groups at 1 VM per SM (150 jobs, more than a batch), difficulties 1/4, 1/9 and 1/16: every
    pow is search_group_range's for its identity, with one device and with [0, 0].  Four pows are checked against the
    oracle: valid, and no lower pow is."""
    k2 = mods[3]
    ids = [(bytes(range(i, i + 8)), _node(i), _rate(r)) for i, r in ((1, 4), (2, 9), (3, 16))]
    with options(b2, rx_vms_per_sm=1):
        assert 3 * 50 > k2.batch_size()
        want = [k2.search_group_range(ch, node, diff, 100, 50)[0] for ch, node, diff in ids]
        jobs = [(node, ch, 100 + g, diff) for ch, node, diff in ids for g in range(50)]
        for plist in ([0], [0, 0]):
            pows, done = k2.search_jobs(jobs, providers=plist)
            assert [pows[50 * i:50 * (i + 1)] for i in range(3)] == want, plist
            assert done >= len(jobs)
        # a reordered job list: the same pow for each job
        rev, _ = k2.search_jobs(jobs[::-1])
        assert rev[::-1] == sum(want, [])
    cache = orx.Cache(orx.K2POW_CACHE_KEY)
    try:
        for i, g in ((0, 0), (1, 17), (2, 49), (2, 3)):
            ch, node, diff = ids[i]
            pw = want[i][g]
            _, found, _ = cache.k2pow_scan(100 + g, ch, node, 0, pw + 1, diff, want_hashes=False)
            assert found == pw, (i, g)
    finally:
        cache.close()


def test_identities_share_one_batch(mods, b2):
    """M = 4 identities, one group each, difficulty 1/4: every pow is below batch / M with near certainty, so the job
    search runs exactly one device batch (8 VM launches, M x batch/M hashes) where M group searches run one each."""
    k2 = mods[3]
    batch = k2.batch_size()
    ids = [(bytes(range(20 + i, 28 + i)), _node(20 + i)) for i in range(4)]
    diff = _rate(4)
    separate = []
    for ch, node in ids:
        pows, done = k2.search_group_range(ch, node, diff, 0, 1)
        t = k2.last_timing()
        assert (done, t["vm_launches"], t["hashes"]) == (batch, 8, batch)
        separate.append(pows[0])
    pows, done = k2.search_jobs([(node, ch, 0, diff) for ch, node in ids])
    t = k2.last_timing()
    assert pows == separate
    assert (done, t["vm_launches"], t["hashes"]) == (4 * (batch // 4), 8, 4 * (batch // 4))


# ------------------------------------------------------------------------------------------------ generate_proofs
def _write_setup(su, d: Path, node: bytes, units: int, n: int) -> np.ndarray:
    o = su.PostSetupOpts(data_dir=str(d), num_units=units, max_file_size=16 * PER_FILE, provider_id=0, scrypt_n=n,
                         compute_batch_size=1 << 12)
    mgr = su.PostSetupManager(_cfg(su))
    mgr.prepare_initializer(o, node, ATX)
    mgr.start_session()
    assert mgr.status().state == su.STATE_COMPLETE
    files = sorted(d.glob("postdata_*.bin"), key=lambda p: int(p.stem.split("_")[1]))
    return np.concatenate([np.fromfile(f, dtype=np.uint8) for f in files]).reshape(-1, 16)


def _cfg(su, **kw):
    return su.PostConfig(labels_per_unit=LPU, k1=K1, k2=K2, k3=K2, max_num_units=8, **kw)


def _single(mods, d, ch, pow_, checked, plist):
    """The one-identity call: (status, text, proof, meta, scanned, report)."""
    su, pr, _, _ = mods
    b2 = importlib.import_module("go-spacemesh_b200")
    kw = dict(providers=list(plist), nonces=NONCES, chunk_labels=CHUNK, pow=pow_, max_windows=WINDOWS)
    try:
        if checked:
            proof, meta, scanned, rep = pr.generate_proof_checked(d, ch, _cfg(su, pow_difficulty=EASY), **kw)
        else:
            (proof, meta, scanned), rep = pr.generate_proof(d, ch, _cfg(su, pow_difficulty=EASY), **kw), None
        return b2.OK, "", proof, meta, scanned, rep
    except b2.B200PostError as e:
        return e.code, str(e).split(": ", 1)[1], None, None, 0, None


def _window_of(mods, d, ch):
    st, _, proof, *_ = _single(mods, d, ch, "skip", False, [0])
    return None if proof is None else proof.nonce // NONCES


@pytest.fixture(scope="module")
def posts(mods, orc, tmp_path_factory):
    """[(data dir, challenge)]: window 0, first in window 2, no proof in windows 0..2 (N = 2, different identities and
    NumUnits), a missing directory, an N = 8192 POST, and a copy of the first with forged hits (below)."""
    su = mods[0]
    root = tmp_path_factory.mktemp("many")
    rng = np.random.default_rng(77)
    items = []
    for i, (units, want) in enumerate(((2, 0), (1, 2), (3, None))):
        d = root / f"id{i}"
        _write_setup(su, d, _node(40 + i), units, 2)
        for _ in range(300):
            ch = rng.bytes(32)
            if _window_of(mods, str(d), ch) == want:
                break
        else:
            raise AssertionError(f"no challenge with the first proof in window {want}")
        items.append((str(d), ch))
    items.append((str(root / "missing"), rng.bytes(32)))
    _write_setup(su, root / "n8192", _node(50), 1, 8192)
    items.append((str(root / "n8192"), rng.bytes(32)))
    # forged: 5 blocks that pass the first item's winning nonce (pow 0), written over the lowest rows below its K2-th hit
    # that are not its hits: the unchecked proof takes them, the checked one drops and reports them
    vf = mods[2]
    d0, ch0 = items[0]
    num = 2 * LPU
    proof = _single(mods, d0, ch0, "skip", False, [0])[2]
    idx = vf.unpack_indices(proof.indices, vf.bits_per_index(num), K2)
    rows = [r for r in range(idx[-1]) if r not in set(idx)][:5]
    blocks = np.random.default_rng(5).integers(0, 256, (200_000, 16), dtype=np.uint8)
    hits = orc.np_prove_hits(blocks, ch0, NONCES, [0], K1, len(blocks), num)
    df = root / "forged"
    shutil.copytree(d0, df)
    stored = np.fromfile(df / "postdata_0.bin", dtype=np.uint8).reshape(-1, 16)
    stored[rows] = blocks[hits[proof.nonce][:5]]
    (df / "postdata_0.bin").write_bytes(stored.tobytes())
    items.append((str(df), ch0))
    return items


def _as_tuple(r):
    return (r.status, r.error, r.proof, r.meta, r.labels_scanned, r.check)


@pytest.mark.parametrize("plist", ([0], [0, 0]), ids=["x1", "x2"])
@pytest.mark.parametrize("pow_", ("skip", "builtin"))
@pytest.mark.parametrize("checked", (True, False), ids=["checked", "unchecked"])
def test_each_item_equals_its_single_call(mods, b2, posts, plist, pow_, checked):
    su, pr, vf, _ = mods
    with options(b2, rx_vms_per_sm=1):
        alone = [_single(mods, d, ch, pow_, checked, plist) for d, ch in posts]
        statuses = [a[0] for a in alone]
        if pow_ == "skip":
            assert statuses[2] == b2.ERR_INVALID_PROOF and "no proof found" in alone[2][1]
            assert alone[1][2].nonce // NONCES == 2 and alone[0][2].nonce // NONCES == 0
        assert statuses[3] == ERR_IO
        if checked and pow_ == "skip":
            assert alone[5][0] == b2.OK and alone[5][2] == alone[0][2]       # the clean proof
            assert alone[5][5].damaged >= 5
        for scans in (1, 3):
            for order in (1, -1):
                rc, got = pr.generate_proofs(posts[::order], _cfg(su, pow_difficulty=EASY), providers=plist, checked=checked,
                                             parallel_scans=scans, nonces=NONCES, chunk_labels=CHUNK, pow=pow_,
                                             max_windows=WINDOWS)
                assert rc == b2.OK
                got = got[::order]
                for i, (g, a) in enumerate(zip(got, alone)):
                    want = (a[0], a[1], a[2], a[3], a[4], a[5] if checked else None)
                    if not checked or a[5] is None:
                        want = want[:5] + ((g.check if checked else None),)
                    assert _as_tuple(g) == want, (i, scans, order)
    # every returned proof verifies (the unchecked proof over forged hits is the one that must not)
    verified = 0
    for (d, _), r in zip(posts, got):
        if r.status != b2.OK or (d.endswith("forged") and not checked):
            continue
        q = vf.VerifyParams(k1=K1, k2=K2, scrypt_n=8192 if d.endswith("n8192") else 2, pow_difficulty=EASY)
        st, _ = vf.verify_batch([r.proof], [r.meta], q, pow=pow_)
        assert list(st) == [b2.OK], d
        verified += 1
    assert verified >= 2


def test_preset_cancel(mods, b2, posts):
    su, pr, _, _ = mods
    flag = ctypes.c_int(1)
    for pow_ in ("skip", "builtin"):
        rc, got = pr.generate_proofs(posts, _cfg(su, pow_difficulty=EASY), nonces=NONCES, chunk_labels=CHUNK, pow=pow_,
                                     max_windows=WINDOWS, cancel=flag)
        assert rc == b2.ERR_CANCELLED
        assert all(r.proof is None for r in got)
        assert got[3].status == ERR_IO
        assert all(r.status == b2.ERR_CANCELLED for i, r in enumerate(got) if i != 3)
