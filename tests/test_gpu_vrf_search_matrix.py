"""GPU tier: the stored-label VRF-nonce search (b200post_search_vrf_nonce: K8a stored_min_kernel, K8b stored_tie_kernel,
the host fold and the recompute) against oracle.pyoracle.np_stored_argmin, at the shapes a real search runs: many
grid-stride steps per thread, hundreds of CTA partials, reads split into parallel slices, chunk and file seams.

K8 trusts the stored bytes, so a POST here is random bytes under real metadata.  When the lowest stored prefix is not a
real label the search fails with ERR_LABEL_MISMATCH and names the lowest position at that prefix, so the error text is
the kernels' arg-min and is compared exactly with NumPy.  Real labels planted at their own positions check the found
path, the past-the-end path and damage next to a real minimum.  Shapes follow the device's SM count: one grid-stride
step of K8 covers 4 * SMs * 256 labels."""
import contextlib
import ctypes
import json
import os
import threading
import time
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ATX = bytes(range(40, 72))
KMAX_CHUNK = 1 << 26
PRIME_CHUNK = 1048573                      # the largest prime below 2^20
# the planted minimum and its decoys: every decoy is larger read big-endian, and each is what a wrong compare keeps
M = bytes.fromhex("00000100000000050000010000000009")
DECOYS = [
    M[:10] + b"\x02" + M[11:],                         # the same high half, a larger low half
    M[:15] + b"\x0a",                                  # the same 15 bytes, a larger last byte
    bytes.fromhex("0001000000000005") + M[8:],         # larger, but smaller read as little-endian words (high half)
    M[:8] + bytes.fromhex("0001000000000009"),         # the same in the low half
]
assert all(d > M for d in DECOYS)


@pytest.fixture(scope="module")
def su(b2, gpu_ready):
    import importlib
    return importlib.import_module("go-spacemesh_b200.setup")


@pytest.fixture(scope="module")
def stride(gpu_ready):
    return 4 * gpu_ready[0]["sm_count"] * 256


def _read_threads():
    return os.cpu_count() or 1             # std::thread::hardware_concurrency, which parallel_pread caps its slices by


class Post:
    """A POST directory: metadata from prepare_initializer, files written from `a` (uint8[n,16], kept in memory)."""

    def __init__(self, su, d, a, per_file, node, n=2):
        self.d, self.a, self.per_file, self.node = Path(d), a, per_file, node
        self.d.mkdir(parents=True)
        num = len(a)
        opts = su.PostSetupOpts(data_dir=str(self.d), num_units=1, max_file_size=16 * per_file, provider_id=0, scrypt_n=n,
                                compute_batch_size=1024)
        su.PostSetupManager(su.PostConfig(labels_per_unit=num)).prepare_initializer(opts, node, ATX)
        for f in range(self.n_files):
            (self.d / f"postdata_{f}.bin").write_bytes(a[f * per_file:(f + 1) * per_file].tobytes())
        self.meta = self.meta_path.read_bytes()

    @property
    def n(self):
        return len(self.a)

    @property
    def n_files(self):
        return -(-self.n // self.per_file)

    @property
    def meta_path(self):
        return self.d / "postdata_metadata.json"

    def mtimes(self):
        return {p.name: p.stat().st_mtime_ns for p in self.d.glob("postdata_*.bin")}

    def _put(self, p, row):
        self.a[p] = np.frombuffer(row, dtype=np.uint8)
        f, o = divmod(p, self.per_file)
        fd = os.open(self.d / f"postdata_{f}.bin", os.O_WRONLY)
        try:
            os.pwrite(fd, row, 16 * o)
        finally:
            os.close(fd)

    @contextlib.contextmanager
    def planted(self, rows: dict):
        """rows {position: 16 bytes} written into the files and `a`; restored afterwards, metadata included."""
        old = {p: self.a[p].tobytes() for p in rows}
        try:
            for p, r in rows.items():
                self._put(p, r)
            yield
        finally:
            for p, r in old.items():
                self._put(p, r)
            self.meta_path.write_bytes(self.meta)


def _random_rows(rng, n, byte0_min=1):
    a = np.frombuffer(rng.bytes(16 * n), dtype=np.uint8).reshape(n, 16).copy()
    np.maximum(a[:, 0], byte0_min, out=a[:, 0])   # above every planted prefix, which starts with 00
    return a


def _shapes(stride):
    """name -> (num_labels, labels per file)"""
    big = (1 << 24) + 4099
    return {"1": (1, 1), "255": (255, 128), "257": (257, 129), "stride-1": (stride - 1, stride // 2),
            "stride+1": (stride + 1, stride // 2 + 1), "2^22": (1 << 22, 1500007), "big": (big, 5600001)}


def _chunks(stride, n):
    """chunk_labels values worth running on n labels (the call clamps a chunk to n, so duplicates are dropped)"""
    out, seen = [], set()
    for c in (0, 256, 257, stride, stride + 1, PRIME_CHUNK, KMAX_CHUNK):
        eff = min(c or 1 << 22, n)
        if eff not in seen:
            seen.add(eff)
            out.append(c)
    return out


def _eff(chunk, n):
    return min(chunk or 1 << 22, n)


def _slice_seams(n_labels):
    """label offsets, within one read of n_labels, where parallel_pread's slices meet"""
    b = 16 * n_labels
    nt = min(8, _read_threads(), max(1, b // (4 << 20)))
    if nt <= 1:
        return []
    per = (b // nt + 15) & ~15
    return [t * per // 16 for t in (1, nt - 1)]


def _positions(n, per_file, chunk, stride):
    """Where the minimum goes: both ends, CTA lanes, grid-stride, chunk, file and read-slice seams (+-1), and inside
    the ragged last chunk."""
    c = _eff(chunk, n)
    n_chunks = -(-n // c)
    last = (n_chunks - 1) * c
    ps = {0, n - 1, 31, 32, 255, 256, 511}
    for start, count in ((0, min(c, n)), (last, n - last)):
        for k in (1, 2, (count - 1) // stride):
            if k:
                ps |= {start + k * stride + d for d in (-1, 0, 1)}
    for k in (1, n_chunks - 1):
        ps |= {k * c + d for d in (-1, 0, 1)}
    for f in range(1, -(-n // per_file)):
        ps |= {f * per_file + d for d in (-1, 0, 1)}
    for seam in _slice_seams(min(c, per_file)):
        ps |= {seam + d for d in (-1, 0, 1)}
    if n % c:
        ps.add(last + (n - last) // 2)
    return sorted(p for p in ps if 0 <= p < n)


def _with_decoys(q, chunk, n, stride):
    """M at q, decoys below it: in the same thread (one and two strides back), warp (q-1), CTA (q-32) and the chunk
    before"""
    c = _eff(chunk, n)
    rows = {}
    for j, p in enumerate((q - stride, q - 2 * stride, q - 1, q - 32, q - c, q - c - stride)):
        if p >= 0:
            rows.setdefault(p, DECOYS[j % len(DECOYS)])
    rows[q] = M
    return rows


def _expect_damage(su, b2, orc, post, q, **kw):
    want, _ = orc.np_stored_argmin(post.a)
    assert want == q                                       # the planted case is what the test means it to be
    with pytest.raises(b2.B200PostError) as e:
        su.search_vrf_nonce(str(post.d), **kw)
    assert e.value.code == su.ERR_LABEL_MISMATCH and f"index {q} " in str(e.value), (kw, q, str(e.value))
    assert post.meta_path.read_bytes() == post.meta


@pytest.fixture(scope="module")
def root(tmp_path_factory):
    return tmp_path_factory.mktemp("vrfm")


@pytest.fixture(scope="module")
def found(b2, orc, gpu_ready, stride):
    """Per shape, a node whose POST has labels below floor(2^256 / numLabels), not near the end, and the lowest of them:
    name -> (node, p, label32(p)), found with the GPU over the whole range and confirmed with the oracle."""
    out = {}
    for name, (n, _) in _shapes(stride).items():
        if n < 257:
            continue
        diff = b2.vrf_difficulty(n)
        for seed in range(64):
            node = bytes([seed, 0x5e, len(name)]) + bytes(29)
            c = b2.commitment(node, ATX)
            _, v = b2.labels_range(c, 2, 0, n, vrf_difficulty_=diff, discard=True)
            if v is not None and v[0] < n - min(n // 2, 6 * stride):
                p, l32 = v
                assert orc.c_label32(c, p, 2) == l32 and l32 < diff
                out[name] = (node, p, l32)
                break
        assert name in out, name
    return out


@pytest.fixture(scope="module")
def posts(su, root, found, stride):
    """One random POST per shape (byte 0 of every row at least 1), under the metadata of that shape's found node."""
    rng = np.random.default_rng(2024)
    out = {}
    for name, (n, per_file) in _shapes(stride).items():
        node = found[name][0] if name in found else bytes(32)
        out[name] = Post(su, root / name, _random_rows(rng, n), per_file, node)
    return out


SHAPE_NAMES = ["1", "255", "257", "stride-1", "stride+1", "2^22", "big"]


@pytest.mark.parametrize("shape", SHAPE_NAMES)
def test_damage_names_the_argmin(su, b2, orc, posts, stride, shape):
    """A fake minimum at every seam, with decoys below it: the error names np_stored_argmin's position."""
    post = posts[shape]
    at_default = set(_positions(post.n, post.per_file, 0, stride))
    for chunk in _chunks(stride, post.n):
        ps = _positions(post.n, post.per_file, chunk, stride)
        if post.n > 1 << 20 and _eff(chunk, post.n) < 1024:
            if post.n > 1 << 23:
                continue                                  # 64 K chunks per call: 2^22 labels cover these chunk sizes
            ps = [ps[len(ps) // 2], post.n - 1]           # 16 K chunks per call: two positions are enough
        elif post.n > 1 << 20 and chunk:
            ps = [q for q in ps if q not in at_default]  # a large POST: the seams this chunk size adds
        for q in ps:
            with post.planted(_with_decoys(q, chunk, post.n, stride)):
                _expect_damage(su, b2, orc, post, q, chunk_labels=chunk)
    # the base data alone: its own arg-min (byte 0 >= 1 everywhere)
    q, _ = orc.np_stored_argmin(post.a)
    _expect_damage(su, b2, orc, post, q)


def test_chunk_limit(su, b2, posts):
    post = posts["257"]
    with pytest.raises(b2.B200PostError) as e:
        su.search_vrf_nonce(str(post.d), chunk_labels=KMAX_CHUNK + 1)
    assert e.value.code == b2.ERR_INVALID_ARGUMENT
    assert post.meta_path.read_bytes() == post.meta


def _expect_found(su, post, p, l32, **kw):
    mt = post.mtimes()
    prog = ctypes.c_uint64(0)
    assert su.search_vrf_nonce(str(post.d), progress=prog, **kw) == (p, l32), kw
    md = su.load_metadata(str(post.d))
    assert (md["nonce"], md["nonce_value"], md["last_position"], md["vrf_scan_pending"]) == (p, l32, 0, 0)
    assert prog.value == post.n and post.mtimes() == mt
    post.meta_path.write_bytes(post.meta)


@pytest.mark.parametrize("shape", ["257", "stride+1", "2^22", "big"])
def test_found_real_minimum(su, posts, found, stride, shape):
    post = posts[shape]
    _, p, l32 = found[shape]
    with post.planted({p: l32[:16]}):
        for chunk in _chunks(stride, post.n):
            if post.n > 1 << 20 and _eff(chunk, post.n) < 1024:
                continue
            _expect_found(su, post, p, l32, chunk_labels=chunk)


def test_found_uses_the_metadata_n(su, b2, orc, root, stride):
    """N = 8192 metadata: the recompute must use it (an N = 2 label at the nonce would not match the stored bytes)."""
    n = 300
    diff = b2.vrf_difficulty(n)
    for seed in range(64):
        node = bytes([seed, 0x81]) + bytes(30)
        c = b2.commitment(node, ATX)
        _, v = b2.labels_range(c, 8192, 0, n, vrf_difficulty_=diff, discard=True)
        if v is not None:
            break
    p, l32 = v
    assert orc.c_label32(c, p, 8192) == l32 and orc.c_label32(c, p, 2) != l32
    post = Post(su, root / "n8192", _random_rows(np.random.default_rng(5), n), 128, node, n=8192)
    with post.planted({p: l32[:16]}):
        for chunk in (0, 64, 257):
            _expect_found(su, post, p, l32, chunk_labels=chunk)


def _spread(rng, anchor, k, n, extra):
    """k positions, the lowest at anchor: the structured ones first (same thread one and two strides on, neighbour lane,
    next warp, next CTA, ...), then random ones above anchor"""
    ps = [anchor] + [anchor + e for e in extra if anchor < anchor + e < n]
    ps = list(dict.fromkeys(ps))[:k]
    while len(ps) < k:
        p = int(rng.integers(anchor + 1, n))
        if p not in ps:
            ps.append(p)
    return ps


@pytest.mark.parametrize("k", [2, 64, 65, 5000])
def test_ties_name_the_lowest_copy(su, b2, orc, posts, stride, k):
    """k copies of a fake minimum over lanes, one thread's strides, CTAs, chunks and files: the lowest is named."""
    post = posts["big"]
    rng = np.random.default_rng(k)
    anchor = post.per_file - 3 * stride + 77
    extra = [stride, 2 * stride, 1, 32, 256, 5 * stride + 3, post.per_file, 1 << 22, 2 * post.per_file - anchor + 9]
    ps = _spread(rng, anchor, k, post.n, extra)
    with post.planted({p: M for p in ps}):
        for chunk in (0, stride + 1, KMAX_CHUNK):
            _expect_damage(su, b2, orc, post, anchor, chunk_labels=chunk)


@pytest.mark.parametrize("k", [1, 65, 5000])
def test_copies_above_a_real_minimum(su, b2, orc, posts, found, stride, k):
    """The real minimum at p and k copies of it above: p is right, so the lowest copy is the damage to name."""
    post = posts["big"]
    _, p, l32 = found["big"]
    rng = np.random.default_rng(100 + k)
    copies = _spread(rng, p + stride, k, post.n, [1, 31, 256, stride, 1 << 22, post.per_file])
    rows = {q: l32[:16] for q in copies}
    rows[p] = l32[:16]
    with post.planted(rows):
        for chunk in (0, stride + 1, KMAX_CHUNK):
            want = min(copies)
            with pytest.raises(b2.B200PostError) as e:
                su.search_vrf_nonce(str(post.d), chunk_labels=chunk)
            assert e.value.code == su.ERR_LABEL_MISMATCH and f"index {want} " in str(e.value), (chunk, want, str(e.value))
            assert post.meta_path.read_bytes() == post.meta


def test_copies_in_two_chunks(su, b2, orc, posts, stride):
    """More than 64 copies in one chunk and more in the next: the first chunk's lowest is named."""
    post = posts["2^22"]
    rng = np.random.default_rng(9)
    c = stride + 1
    first = sorted(set(int(x) for x in rng.integers(c // 3, c, 100)))
    second = sorted(set(int(x) for x in rng.integers(c, 2 * c, 100)))
    with post.planted({p: M for p in first + second}):
        for chunk in (c, 256 * 1024):
            _expect_damage(su, b2, orc, post, first[0], chunk_labels=chunk)


def test_all_ones_post(su, b2, orc, root, stride):
    """Every stored label ff..ff, more than 64 of them per chunk: position 0 is the arg-min and is named."""
    n = 3 * stride + 5
    post = Post(su, root / "ff", np.full((n, 16), 0xff, dtype=np.uint8), stride + 7, bytes(range(1, 33)))
    for chunk in (0, 256, 1000, stride):
        _expect_damage(su, b2, orc, post, 0, chunk_labels=chunk)


def test_zero_hole_in_the_last_file(su, b2, orc, posts, stride):
    """The last file cut short and extended back with truncate: its first zero row is named."""
    post = posts["stride+1"]
    last = post.d / f"postdata_{post.n_files - 1}.bin"
    size = last.stat().st_size
    cut = size // 2 & ~15
    keep = post.a.copy()
    try:
        os.truncate(last, cut)
        os.truncate(last, size)
        post.a[(post.n_files - 1) * post.per_file + cut // 16:] = 0
        hole = (post.n_files - 1) * post.per_file + cut // 16
        for chunk in (0, 256, stride):
            _expect_damage(su, b2, orc, post, hole, chunk_labels=chunk)
    finally:
        post.a[:] = keep
        last.write_bytes(keep[(post.n_files - 1) * post.per_file:].tobytes())


def test_past_the_end(su, b2, orc, root):
    """The stored minimum is a real label at or above the threshold: the nonce comes from the first batch past numLabels
    holding a label below it, as the oracle computes that batch; a stale Nonce and LastPosition are ignored."""
    n, batch = (1 << 16) + 3, 4099
    node = bytes(range(7, 39))
    c = orc.c_commitment(node, ATX)
    diff = orc.c_vrf_difficulty(n)
    head, _, _, _ = orc.c_labels_range(c, 2, 0, 64)
    r = next(i for i in range(64) if orc.c_label32(c, i, 2) >= diff and head[i, 0] < 0xff)
    post = Post(su, root / "past", _random_rows(np.random.default_rng(11), n, byte0_min=0xff), 40000, node)
    j = 0
    while True:
        _, ok, idx, l32 = orc.c_labels_range(c, 2, n + j * batch, batch, diff)
        if ok:
            break
        j += 1
    with post.planted({r: head[r].tobytes()}):
        assert orc.np_stored_argmin(post.a)[0] == r
        assert su.search_vrf_nonce(str(post.d), compute_batch_size=batch) == (idx, l32)
        md = su.load_metadata(str(post.d))
        assert (md["nonce"], md["nonce_value"], md["last_position"], md["vrf_scan_pending"]) == (idx, l32, n + (j + 1) * batch, 0)
        # a stale nonce, and a LastPosition past the batch that holds the answer
        doc = json.loads(post.meta.decode())
        doc["Nonce"], doc["NonceValue"], doc["LastPosition"] = 12, "00" * 32, n + (j + 2) * batch
        post.meta_path.write_text(json.dumps(doc))
        assert su.search_vrf_nonce(str(post.d), compute_batch_size=batch) == (idx, l32)
        assert su.load_metadata(str(post.d))["last_position"] == n + (j + 1) * batch


def test_cancel_then_search_again(su, b2, orc, posts, stride):
    post = posts["big"]
    q = 3 * stride + 17
    with post.planted(_with_decoys(q, 0, post.n, stride)):
        prog, cancel, res = ctypes.c_uint64(0), ctypes.c_int(0), {}

        def run():
            try:
                su.search_vrf_nonce(str(post.d), chunk_labels=256, progress=prog, cancel=cancel)
                res["rc"] = 0
            except b2.B200PostError as e:
                res["rc"] = e.code
        t = threading.Thread(target=run)
        t.start()
        deadline = time.time() + 60
        while prog.value == 0 and time.time() < deadline:
            time.sleep(0.001)
        cancel.value = 1
        t.join()
        assert res["rc"] == b2.ERR_CANCELLED and 0 < prog.value < post.n
        assert post.meta_path.read_bytes() == post.meta
        _expect_damage(su, b2, orc, post, q)


def test_providers(su, b2, orc, posts, found, stride, gpu_ready):
    post = posts["stride+1"]
    _, p, l32 = found["stride+1"]
    provs = [su.PROVIDER_ALL] + ([1] if len(gpu_ready) > 1 else [])
    for prov in provs:
        with post.planted({p: l32[:16]}):
            _expect_found(su, post, p, l32, provider_id=prov)
        q = post.n - stride // 3
        with post.planted(_with_decoys(q, 0, post.n, stride)):
            _expect_damage(su, b2, orc, post, q, provider_id=prov)
