"""CPU tier: the host checks of b200post_generate_proof_checked: argument checks, the order of host errors, and no CPU
path without a device."""
import ctypes
import importlib

import pytest

NODE, ATX = bytes(range(32)), bytes(range(32, 64))


@pytest.fixture()
def mods(b2):
    return importlib.import_module("go-spacemesh_b200.setup"), importlib.import_module("go-spacemesh_b200.prove")


def _checked(pr, su, data_dir, providers, n_providers, with_check=True, with_out=True):
    """The C call itself, so that NULL pointers and a count that disagrees with the list can be passed."""
    L = pr._bind()
    out, meta, chk, c = pr._ProofOut(), pr._Meta(), pr._ProveCheck(), pr._c_cfg(su.PostConfig())
    chk.damaged = 99
    opts = pr._ProveOpts(0, 16, 0, ctypes.cast(None, pr.POW_PROVE_FN), None, 2, None, 0)
    arr = (ctypes.c_uint32 * len(providers))(*providers) if providers is not None else None
    rc = L.b200post_generate_proof_checked(str(data_dir).encode() if data_dir is not None else None, bytes(32), ctypes.byref(c),
                                           ctypes.byref(opts), arr, n_providers, ctypes.byref(out) if with_out else None,
                                           ctypes.byref(meta), ctypes.byref(chk) if with_check else None, None)
    return rc, chk


def _post(su, d):
    """Metadata of a 2 x 512-label POST (no label files: the device errors come before any read)."""
    o = su.PostSetupOpts(data_dir=str(d), num_units=2, max_file_size=4096, provider_id=0, scrypt_n=2)
    su.PostSetupManager().prepare_initializer(o, NODE, ATX)
    return o.data_dir


def test_argument_checks(b2, mods, tmp_path):
    su, pr = mods
    d = _post(su, tmp_path / "p")
    for provs, n in ((None, 1), (None, 2), ([0], 0), ([0, 0], -3)):
        assert _checked(pr, su, d, provs, n)[0] == b2.ERR_INVALID_ARGUMENT, (provs, n)
    assert _checked(pr, su, d, [0], 1, with_check=False)[0] == b2.ERR_INVALID_ARGUMENT
    assert _checked(pr, su, d, [0], 1, with_out=False)[0] == b2.ERR_INVALID_ARGUMENT
    assert _checked(pr, su, None, [0], 1)[0] == b2.ERR_INVALID_ARGUMENT
    # the NULL check comes before the metadata is read
    assert _checked(pr, su, tmp_path / "nowhere", [0], 1, with_check=False)[0] == b2.ERR_INVALID_ARGUMENT
    with pytest.raises(b2.B200PostError) as e:
        pr.generate_proof_checked(d, bytes(32), su.PostConfig(), providers=[], pow="skip")
    assert e.value.code == b2.ERR_INVALID_ARGUMENT
    with pytest.raises(ValueError):
        pr.generate_proof_checked(d, bytes(32), su.PostConfig(), providers="every", pow="skip")
    for provs in ([b2.CPU_PROVIDER_ID], [b2.CPU_PROVIDER_ID] * 3):
        for pow_ in ("skip", "builtin"):
            with pytest.raises(b2.B200PostError) as e:
                pr.generate_proof_checked(d, bytes(32), su.PostConfig(), providers=provs, pow=pow_)
            assert e.value.code == b2.ERR_UNSUPPORTED, (provs, pow_)


def test_missing_metadata_is_an_io_error_before_the_device(b2, mods, tmp_path):
    su, pr = mods
    (tmp_path / "empty").mkdir()
    for provs in ([0], [0, 1], [b2.CPU_PROVIDER_ID, 0]):
        for pow_ in ("skip", "builtin"):
            with pytest.raises(b2.B200PostError) as e:
                pr.generate_proof_checked(str(tmp_path / "empty"), bytes(32), su.PostConfig(), providers=provs, pow=pow_)
            assert e.value.code == su.ERR_IO, (provs, pow_)


def test_the_report_is_cleared_on_every_call_past_the_argument_checks(b2, mods, tmp_path):
    su, pr = mods
    (tmp_path / "empty").mkdir()
    rc, chk = _checked(pr, su, tmp_path / "empty", [0], 1)
    assert rc == su.ERR_IO
    assert (chk.labels_rechecked, chk.damaged, chk.n_reported, chk.proof_verified) == (0, 0, 0, 0)


def test_no_device_no_cpu_path(b2, mods, tmp_path):
    su, pr = mods
    if b2.providers():
        pytest.skip("a CUDA device is present: the no-device contract is covered on CPU-only boxes")
    d = _post(su, tmp_path / "p")
    for provs in ([0], [0, 0], [0, 1, 2]):
        for pow_ in ("skip", "builtin"):
            with pytest.raises(b2.B200PostError) as e:
                pr.generate_proof_checked(d, bytes(32), su.PostConfig(), providers=provs, pow=pow_)
            assert e.value.code == b2.ERR_NO_DEVICE, (provs, pow_)
    with pytest.raises(b2.B200PostError) as e:
        pr.generate_proof_checked(d, bytes(32), su.PostConfig(), providers="all", pow="skip")
    assert e.value.code == b2.ERR_NO_DEVICE
