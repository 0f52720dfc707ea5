"""GPU tier: init -> prove -> verify, the reference's e2e shape (activation/e2e/nipost_test.go:151-231: setup
session, PostClient.Proof, real verifier) run entirely on the GPU engine, plus parity of the proving scan with
the oracle's restatement."""
import importlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NODE, ATX = bytes(range(50, 82)), bytes(range(150, 182))


@pytest.fixture(scope="module")
def mods(b2, gpu_ready):
    return (importlib.import_module("go-spacemesh_b200.setup"), importlib.import_module("go-spacemesh_b200.prove"),
            importlib.import_module("go-spacemesh_b200.verify"))


def _init(su, tmp_path, cfg, n, num_units, max_file_size):
    mgr = su.PostSetupManager(cfg)
    o = su.PostSetupOpts(data_dir=str(tmp_path / "post"), num_units=num_units, max_file_size=max_file_size, provider_id=0,
                         scrypt_n=n, compute_batch_size=1 << 12)
    mgr.prepare_initializer(o, NODE, ATX)
    mgr.start_session()
    assert mgr.status().state == su.STATE_COMPLETE
    return o


def test_scan_matches_oracle_rule(mods, orc):
    """Multi-nonce scan over labels in memory: same (nonce, indices) as the oracle's restatement."""
    su, pr, vf = mods
    c = orc.py_commitment(NODE, ATX)
    num_labels, k1, k2 = 4096, 180, 6
    labels, _, _, _ = orc.c_labels_range(c, 2, 0, num_labels)
    rng = np.random.default_rng(8)
    for nonces, pows in ((16, [5]), (48, [1, 2**40, 77])):
        challenge = bytes(rng.integers(0, 256, 32, dtype=np.uint8))
        nonce, packed, pow_, scanned = pr.prove_scan(labels, challenge, nonces, pows, k1, k2, num_labels)
        exp_nonce, exp_hits = orc.py_prove_multi(labels[:scanned + 64], challenge, nonces, pows, k1, k2, num_labels)
        assert exp_nonce is not None
        assert (nonce, vf.unpack_indices(packed, vf.bits_per_index(num_labels), k2)) == (exp_nonce, exp_hits)
        assert pow_ == pows[nonce // 16]


@pytest.mark.parametrize("n,lpu,units,k1,k2,nonces", [(2, 512, 4, 120, 8, 16), (2, 2048, 2, 300, 12, 64), (8192, 1024, 2, 200, 10, 16)])
def test_init_prove_verify_roundtrip(mods, tmp_path, orc, n, lpu, units, k1, k2, nonces):
    su, pr, vf = mods
    cfg = su.PostConfig(labels_per_unit=lpu, k1=k1, k2=k2, k3=k2, max_num_units=8)
    o = _init(su, tmp_path, cfg, n, units, max_file_size=lpu * 16 // 2)        # data spans several files
    challenge = bytes(range(200, 232))
    pows_seen = []

    def k2pow(ctx, nonce_group, challenge8, difficulty, node_id, pow_out):
        pows_seen.append(nonce_group)
        pow_out[0] = 1000 + nonce_group
        return 0

    proof, meta, scanned = pr.generate_proof(o.data_dir, challenge, cfg, nonces=nonces, chunk_labels=700, pow=k2pow)
    assert pows_seen == list(range(nonces // 16)) and proof.pow == 1000 + proof.nonce // 16
    assert meta.node_id == NODE and meta.commitment_atx_id == ATX and meta.challenge == challenge
    assert (meta.num_units, meta.labels_per_unit) == (units, lpu) and 0 < scanned <= units * lpu
    params = vf.VerifyParams(k1=k1, k2=k2, scrypt_n=n)
    # the oracle's verifier accepts it ...
    assert orc.py_verify(proof.nonce, proof.indices, proof.pow, NODE, ATX, challenge, units, lpu, k1, k2, n) == (True, None)
    # ... and so does the batched GPU verifier, in every mode
    v = vf.PostVerifier(pow="skip")
    try:
        v.verify(proof, meta, params)
        v.verify(proof, meta, params, mode=vf.MODE_SUBSET, k3=3, seed=b"peer")
        idx = vf.unpack_indices(proof.indices, vf.bits_per_index(units * lpu), k2)
        assert idx == sorted(idx) and len(set(idx)) == k2
        # a proof for another challenge must not verify (activation/e2e/validation_test.go:23-137 spirit)
        other = vf.ProofMetadata(NODE, ATX, bytes(32), units, lpu)
        with pytest.raises(vf.ErrInvalidIndex):
            v.verify(proof, other, params)
    finally:
        v.close()


def test_no_proof_in_a_space_that_is_too_hard(mods, tmp_path, b2):
    su, pr, vf = mods
    cfg = su.PostConfig(labels_per_unit=256, k1=1, k2=30, k3=30)
    o = _init(su, tmp_path, cfg, 2, 2, max_file_size=4096)
    with pytest.raises(b2.B200PostError) as e:
        pr.generate_proof(o.data_dir, bytes(32), cfg, pow="skip")
    assert e.value.code == b2.ERR_INVALID_PROOF and "no proof found" in str(e.value)


def test_mainnet_shaped_lifecycle_at_n8192(mods, tmp_path, orc, b2):
    """The whole POST lifecycle at the mainnet scrypt cost and K2: 4 units x 2^20 labels (64 MiB of POST data),
    N = 8192, K2 = 37, 288 proving nonces — setup session -> proof over the files -> batched verification,
    with the stored labels spot-checked against the oracle."""
    su, pr, vf = mods
    units, lpu, k1, k2 = 4, 1 << 20, 1 << 9, 37
    cfg = su.PostConfig(labels_per_unit=lpu, k1=k1, k2=k2, k3=k2, max_num_units=8)
    mgr = su.PostSetupManager(cfg)
    o = su.PostSetupOpts(data_dir=str(tmp_path / "post"), num_units=units, max_file_size=16 << 20, provider_id=0, scrypt_n=8192,
                         compute_batch_size=1 << 20)
    mgr.prepare_initializer(o, NODE, ATX)
    mgr.start_session()
    assert mgr.status() == su.PostSetupStatus(su.STATE_COMPLETE, units * lpu)
    # spot-check the files
    c = orc.py_commitment(NODE, ATX)
    pick = np.unique(np.random.default_rng(2).integers(0, units * lpu, 160)).astype(np.uint64)
    comms = np.tile(np.frombuffer(c, dtype=np.uint8), (len(pick), 1))
    exp = orc.c_labels_gather(comms, pick, 8192)
    per_file = (16 << 20) // 16
    for row, i in zip(exp, pick):
        with open(f"{o.data_dir}/postdata_{int(i) // per_file}.bin", "rb") as f:
            f.seek((int(i) % per_file) * 16)
            assert f.read(16) == row.tobytes()
    md = su.load_metadata(o.data_dir)
    assert md["nonce"] is not None and orc.c_label32(c, md["nonce"], 8192) == md["nonce_value"]
    assert b2.verify_vrf_nonce(md["nonce"], NODE, ATX, units, lpu, 8192)
    # prove + verify
    challenge = bytes(range(90, 122))
    proof, meta, scanned = pr.generate_proof(o.data_dir, challenge, cfg, nonces=288, pow="skip")
    assert len(proof.indices) == (k2 * vf.bits_per_index(units * lpu) + 7) // 8 and scanned <= units * lpu
    params = vf.VerifyParams(k1=k1, k2=k2, scrypt_n=8192)
    v = vf.PostVerifier(pow="skip")
    try:
        v.verify(proof, meta, params)                                       # all K2 indices
        v.verify(proof, meta, params, mode=vf.MODE_SUBSET, k3=1, seed=b"peer")
        idx = vf.unpack_indices(proof.indices, vf.bits_per_index(units * lpu), k2)
        bad = list(idx); bad[20] = (bad[20] + 1) % (units * lpu)             # systest: Indices[i] += 1
        tampered = vf.Proof(proof.nonce, vf.pack_indices(bad, vf.bits_per_index(units * lpu)), proof.pow)
        ok, which = orc.py_verify(tampered.nonce, tampered.indices, tampered.pow, NODE, ATX, challenge, units, lpu, k1, k2, 8192)
        if not ok:
            with pytest.raises(vf.ErrInvalidIndex) as e:
                v.verify(tampered, meta, params)
            assert e.value.index == which
    finally:
        v.close()


def test_prove_and_verify_with_the_builtin_k2pow(mods, tmp_path, b2):
    """init -> generate_proof with the RandomX k2pow search on the device (one pow per nonce group, all groups sharing
    batches) -> the verifier's builtin pow check accepts it; a pow taken from another group is rejected as 'k2pow
    invalid', not as a label error.  (activation/nipost.go:171 + activation/post_verifier.go:150-160 in one process.)"""
    import importlib
    su, pr, vf = mods
    k2 = importlib.import_module("go-spacemesh_b200.k2pow")
    diff = bytes([0x08]) + b"\x00" * 31                              # 1/32 of all hashes, 1/64 after / 2 units
    cfg = su.PostConfig(labels_per_unit=512, k1=150, k2=8, k3=8, max_num_units=8, pow_difficulty=diff)
    o = _init(su, tmp_path, cfg, 2, 2, max_file_size=512 * 16)
    challenge = bytes(range(50, 82))
    proof, meta, scanned = pr.generate_proof(o.data_dir, challenge, cfg, nonces=32)          # 2 nonce groups, builtin pow
    scaled = k2.scale_difficulty(diff, 2)
    assert k2.verify(proof.pow, proof.nonce // 16, challenge[:8], NODE, scaled)
    first, _ = k2.search(proof.nonce // 16, challenge[:8], NODE, scaled, 0, 4096)
    assert first == proof.pow                                         # the smallest valid nonce of its group
    params = vf.VerifyParams(k1=150, k2=8, scrypt_n=2, pow_difficulty=diff)
    v = vf.PostVerifier()                                             # builtin pow check
    try:
        v.verify(proof, meta, params)
        v.verify(proof, meta, params, mode=vf.MODE_SUBSET, k3=3, seed=b"peer")
        other = proof.pow + 1
        while k2.verify(other, proof.nonce // 16, challenge[:8], NODE, scaled):
            other += 1
        with pytest.raises(vf.ErrInvalidIndex) as e:
            v.verify(vf.Proof(proof.nonce, proof.indices, other), meta, params)
        assert e.value.index == vf.POW_INVALID
    finally:
        v.close()
    with pytest.raises(b2.B200PostError) as e:
        pr.generate_proof(o.data_dir, challenge, cfg, nonces=16, pow="callback-missing")
    assert e.value.code == b2.ERR_UNSUPPORTED


def test_libpost_compatible_prove_and_verify_symbols(mods, tmp_path, b2):
    """include/post_compat.h: the call sequence spacemeshos/post makes through cgo — generate_proof / free_proof on the
    proving side, new_verifier / verify_proof / verify_proof_index / verify_proof_subset / free_verifier on the
    verifying side (activation/post_verifier.go:159,204) — with post.h's by-value structs."""
    import ctypes
    su, pr, vf = mods
    L = b2.lib()

    class ArrayU8(ctypes.Structure):
        _fields_ = [("ptr", ctypes.POINTER(ctypes.c_uint8)), ("len", ctypes.c_size_t), ("cap", ctypes.c_size_t)]

    class CProof(ctypes.Structure):
        _fields_ = [("nonce", ctypes.c_uint32), ("indices", ArrayU8), ("pow", ctypes.c_uint64)]

    class CMeta(ctypes.Structure):
        _fields_ = [("node_id", ctypes.c_uint8 * 32), ("commitment_atx_id", ctypes.c_uint8 * 32), ("challenge", ctypes.c_uint8 * 32),
                    ("num_units", ctypes.c_uint32), ("labels_per_unit", ctypes.c_uint64)]

    class Scrypt(ctypes.Structure):
        _fields_ = [("n", ctypes.c_size_t), ("r", ctypes.c_size_t), ("p", ctypes.c_size_t)]

    class ProofConfig(ctypes.Structure):
        _fields_ = [("k1", ctypes.c_uint32), ("k2", ctypes.c_uint32), ("pow_difficulty", ctypes.c_uint8 * 32)]

    class InitConfig(ctypes.Structure):
        _fields_ = [("min_num_units", ctypes.c_uint32), ("max_num_units", ctypes.c_uint32), ("labels_per_unit", ctypes.c_uint64), ("scrypt", Scrypt)]

    class VerifyResult(ctypes.Structure):
        _fields_ = [("tag", ctypes.c_int), ("invalid_index", ctypes.c_uint32)]

    L.generate_proof.restype = ctypes.POINTER(CProof)
    L.generate_proof.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ProofConfig, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_uint32]
    L.free_proof.argtypes = [ctypes.POINTER(CProof)]
    L.new_verifier.restype = VerifyResult
    L.new_verifier.argtypes = [ctypes.c_uint32, ctypes.POINTER(ctypes.c_void_p)]
    L.free_verifier.argtypes = [ctypes.c_void_p]
    for f in (L.verify_proof, L.verify_proof_index, L.verify_proof_subset):
        f.restype = VerifyResult
    L.verify_proof.argtypes = [ctypes.c_void_p, CProof, ctypes.POINTER(CMeta), ProofConfig, InitConfig]
    L.verify_proof_index.argtypes = L.verify_proof.argtypes + [ctypes.c_size_t]
    L.verify_proof_subset.argtypes = L.verify_proof.argtypes + [ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t]

    diff = bytes([0x10]) + b"\x00" * 31
    lpu, units, k1, k2 = 512, 2, 150, 8
    cfg = su.PostConfig(labels_per_unit=lpu, k1=k1, k2=k2, k3=k2, max_num_units=8, pow_difficulty=diff)
    o = _init(su, tmp_path, cfg, 2, units, max_file_size=lpu * 16)
    challenge = bytes(range(7, 39))
    pc = ProofConfig(k1, k2, (ctypes.c_uint8 * 32)(*diff))
    ic = InitConfig(1, 8, lpu, Scrypt(2, 1, 1))
    pp = L.generate_proof(o.data_dir.encode(), challenge, pc, 16, 1, 0)
    assert pp, b2.lib().b200post_last_error()
    proof = pp.contents
    assert proof.indices.len == (k2 * vf.bits_per_index(units * lpu) + 7) // 8
    meta = CMeta((ctypes.c_uint8 * 32)(*NODE), (ctypes.c_uint8 * 32)(*ATX), (ctypes.c_uint8 * 32)(*challenge), units, lpu)
    ver = ctypes.c_void_p()
    assert L.new_verifier(0, ctypes.byref(ver)).tag == 0 and ver
    try:
        assert L.verify_proof(ver, proof, ctypes.byref(meta), pc, ic).tag == 0
        assert L.verify_proof_subset(ver, proof, ctypes.byref(meta), pc, ic, 3, b"peer-id", 7).tag == 0
        for pos in range(k2):
            assert L.verify_proof_index(ver, proof, ctypes.byref(meta), pc, ic, pos).tag == 0
        # systest/tests/distributed_post_verification_test.go:254-256: Indices[i] += 1 for every packed byte
        raw = bytes(proof.indices.ptr[: proof.indices.len])
        broken = bytes((b + 1) & 255 for b in raw)
        buf = (ctypes.c_uint8 * len(broken))(*broken)
        bad = CProof(proof.nonce, ArrayU8(ctypes.cast(buf, ctypes.POINTER(ctypes.c_uint8)), len(broken), len(broken)), proof.pow)
        r = L.verify_proof(ver, bad, ctypes.byref(meta), pc, ic)
        assert r.tag == 1 and 0 <= r.invalid_index < k2                       # VerifyInvalidIndex + a POSITION
        # malfeasance.go:161-166: re-verifying just that position reproduces the verdict
        r2 = L.verify_proof_index(ver, bad, ctypes.byref(meta), pc, ic, r.invalid_index)
        assert (r2.tag, r2.invalid_index) == (1, r.invalid_index)
        wrong_pow = CProof(proof.nonce, proof.indices, proof.pow ^ 0x5555)
        assert L.verify_proof(ver, wrong_pow, ctypes.byref(meta), pc, ic).tag in (1, 4)   # k2pow or (re-keyed) labels fail
        assert L.verify_proof(ver, CProof(0, ArrayU8(None, 0, 0), 0), ctypes.byref(meta), pc, ic).tag == 2
    finally:
        L.free_verifier(ver)
        L.free_proof(pp)
