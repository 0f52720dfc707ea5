"""CPU tier: the host checks of proving on several devices (b200post_k2pow_search_groups_multi and
b200post_generate_proof_multi): argument checks, the order of host errors, and no CPU path without a device."""
import ctypes
import importlib

import pytest

NODE, ATX = bytes(range(32)), bytes(range(32, 64))
EASY = b"\xff" * 32


@pytest.fixture()
def mods(b2):
    return (importlib.import_module("go-spacemesh_b200.setup"), importlib.import_module("go-spacemesh_b200.prove"),
            importlib.import_module("go-spacemesh_b200.k2pow"))


def _search_groups_multi(k2, providers, n_providers, n_groups):
    """The C call itself, so that a NULL list and a count that disagrees with the list can be passed."""
    p = k2._params(0, bytes(8), bytes(32), EASY, None)
    pows = (ctypes.c_uint64 * 257)()
    done = ctypes.c_uint64(0)
    arr = (ctypes.c_uint32 * len(providers))(*providers) if providers is not None else None
    return k2._bind().b200post_k2pow_search_groups_multi(arr, n_providers, ctypes.byref(p), n_groups, 0, pows,
                                                         ctypes.byref(done), None)


def _generate_multi(pr, su, data_dir, providers, n_providers, cfg=None):
    L = pr._bind()
    out, meta, c = pr._ProofOut(), pr._Meta(), pr._c_cfg(cfg or su.PostConfig())
    opts = pr._ProveOpts(0, 16, 0, ctypes.cast(None, pr.POW_PROVE_FN), None, 2, None, 0)
    arr = (ctypes.c_uint32 * len(providers))(*providers) if providers is not None else None
    return L.b200post_generate_proof_multi(str(data_dir).encode(), bytes(32), ctypes.byref(c), ctypes.byref(opts), arr,
                                           n_providers, ctypes.byref(out), ctypes.byref(meta), None)


def _post(su, d):
    """Metadata of a 2 x 512-label POST (no label files: the device errors come before any read)."""
    o = su.PostSetupOpts(data_dir=str(d), num_units=2, max_file_size=4096, provider_id=0, scrypt_n=2)
    su.PostSetupManager().prepare_initializer(o, NODE, ATX)
    return o.data_dir


def test_search_groups_multi_argument_checks(b2, mods):
    _, _, k2 = mods
    for provs, n, groups in ((None, 2, 1), ([0, 0], 0, 1), ([0], -1, 1), ([0, 0], 2, 0), ([0, 0], 2, 257), ([0], 1, 0),
                             ([0], 1, 257)):
        assert _search_groups_multi(k2, provs, n, groups) == b2.ERR_INVALID_ARGUMENT, (provs, n, groups)
    for provs, groups in (([], 1), ([0, 0], 0), ([0, 0], 300)):
        with pytest.raises(b2.B200PostError) as e:
            k2.search_groups(bytes(8), bytes(32), EASY, groups, providers=provs)
        assert e.value.code == b2.ERR_INVALID_ARGUMENT
    for provs in ([b2.CPU_PROVIDER_ID], [b2.CPU_PROVIDER_ID, b2.CPU_PROVIDER_ID]):
        with pytest.raises(b2.B200PostError) as e:
            k2.search_groups(bytes(8), bytes(32), EASY, 2, providers=provs)
        assert e.value.code == b2.ERR_UNSUPPORTED


def test_generate_proof_multi_argument_checks(b2, mods, tmp_path):
    su, pr, _ = mods
    d = _post(su, tmp_path / "p")
    for provs, n in ((None, 1), (None, 2), ([0], 0), ([0, 0], -3)):
        assert _generate_multi(pr, su, d, provs, n) == b2.ERR_INVALID_ARGUMENT, (provs, n)
    with pytest.raises(ValueError):
        pr.generate_proof(d, bytes(32), su.PostConfig(), provider=0, providers=[0], pow="skip")
    with pytest.raises(ValueError):
        pr.generate_proof(d, bytes(32), su.PostConfig(), providers="every", pow="skip")
    with pytest.raises(b2.B200PostError) as e:
        pr.generate_proof(d, bytes(32), su.PostConfig(), providers=[], pow="skip")
    assert e.value.code == b2.ERR_INVALID_ARGUMENT
    for provs in ([b2.CPU_PROVIDER_ID], [b2.CPU_PROVIDER_ID] * 3):
        for pow_ in ("skip", "builtin"):
            with pytest.raises(b2.B200PostError) as e:
                pr.generate_proof(d, bytes(32), su.PostConfig(), providers=provs, pow=pow_)
            assert e.value.code == b2.ERR_UNSUPPORTED, (provs, pow_)


def test_missing_metadata_is_an_io_error_before_the_device(b2, mods, tmp_path):
    su, pr, _ = mods
    (tmp_path / "empty").mkdir()
    for provs in ([0], [0, 1], [b2.CPU_PROVIDER_ID, 0]):
        for pow_ in ("skip", "builtin"):
            with pytest.raises(b2.B200PostError) as e:
                pr.generate_proof(str(tmp_path / "empty"), bytes(32), su.PostConfig(), providers=provs, pow=pow_)
            assert e.value.code == su.ERR_IO, (provs, pow_)


def test_no_device_no_cpu_path(b2, mods, tmp_path):
    su, pr, k2 = mods
    if b2.providers():
        pytest.skip("a CUDA device is present: the no-device contract is covered on CPU-only boxes")
    d = _post(su, tmp_path / "p")
    for provs in ([0], [0, 0], [0, 1, 2]):
        with pytest.raises(b2.B200PostError) as e:
            k2.search_groups(bytes(8), bytes(32), EASY, 18, providers=provs)
        assert e.value.code == b2.ERR_NO_DEVICE
        for pow_ in ("skip", "builtin"):
            with pytest.raises(b2.B200PostError) as e:
                pr.generate_proof(d, bytes(32), su.PostConfig(), providers=provs, pow=pow_)
            assert e.value.code == b2.ERR_NO_DEVICE, (provs, pow_)
    with pytest.raises(b2.B200PostError) as e:
        pr.generate_proof(d, bytes(32), su.PostConfig(), providers="all", pow="skip")
    assert e.value.code == b2.ERR_NO_DEVICE
