"""CPU tier: b200post_verify_pos's sampler and the errors it returns before any device is touched."""
import importlib
import math
from pathlib import Path

import numpy as np
import pytest

NODE, ATX = bytes(range(32)), bytes(range(32, 64))


@pytest.fixture()
def su(b2):
    return importlib.import_module("go-spacemesh_b200.setup")


def _post(su, b2, orc, d: Path):
    """A complete N = 2 POST written on the CPU: 2 x 512 labels in 4 files of 256 labels (no VRF nonce)."""
    mgr = su.PostSetupManager()
    mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=2, max_file_size=4096, provider_id=0, scrypt_n=2,
                                             compute_batch_size=1 << 10), NODE, ATX)
    labels = orc.c_labels_range(b2.commitment(NODE, ATX), 2, 0, 1024)[0]
    for f in range(4):
        (d / f"postdata_{f}.bin").write_bytes(labels[256 * f: 256 * (f + 1)].tobytes())
    return str(d)


@pytest.mark.parametrize("L,fraction", [(1, 0.2), (255, 0.2), (256, 25.0), (1000, 3.3), (4096, 50.0), (12345, 100.0),
                                        (1 << 20, 0.1), (1 << 16, 99.9), (1 << 26, 6.0), (1 << 26, 1.0)])
def test_sample_is_distinct_sorted_in_range_and_sized(su, L, fraction):
    s = su.verify_pos_sample(7, 3, L, fraction)
    assert len(s) == max(1, math.floor(L * fraction / 100))
    assert (np.diff(s.astype(np.int64)) > 0).all() and int(s[0]) >= 0 and int(s[-1]) < L
    if fraction == 100.0:
        assert (s == np.arange(L, dtype=np.uint64)).all()


def test_sample_is_a_function_of_seed_and_file(su):
    a = su.verify_pos_sample(11, 0, 100000, 1.0)
    assert (a == su.verify_pos_sample(11, 0, 100000, 1.0)).all()
    assert not np.array_equal(a, su.verify_pos_sample(11, 1, 100000, 1.0))
    assert not np.array_equal(a, su.verify_pos_sample(12, 0, 100000, 1.0))
    # both generators (streamed selection sampling, and samples of at most 1 in 64 labels drawn whole) are deterministic
    d = su.verify_pos_sample(11, 0, 100000, 40.0)
    assert (d == su.verify_pos_sample(11, 0, 100000, 40.0)).all()


@pytest.mark.parametrize("fraction", [1.0, 30.0])
def test_sample_is_uniform(su, fraction):
    """chi^2 over 64 equal bins of the positions of many files' samples (drawn whole at 1 %, streamed at 30 %)."""
    from scipy import stats
    L, bins = 1 << 16, 64
    counts = np.zeros(bins)
    for f in range(200 if fraction < 10 else 20):
        s = su.verify_pos_sample(99, f, L, fraction)
        counts += np.bincount((s // (L // bins)).astype(np.int64), minlength=bins)
    assert stats.chisquare(counts).pvalue > 1e-4


def test_sample_argument_errors(su, b2):
    for bad in (dict(labels_in_file=0), dict(fraction=0.0), dict(fraction=-1.0), dict(fraction=100.5)):
        kw = dict(seed=1, file=0, labels_in_file=100, fraction=1.0)
        kw.update(bad)
        with pytest.raises(b2.B200PostError) as e:
            su.verify_pos_sample(**kw)
        assert e.value.code == b2.ERR_INVALID_ARGUMENT, bad


def test_verify_pos_argument_errors(su, b2, orc, tmp_path):
    import ctypes
    d = _post(su, b2, orc, tmp_path / "post")
    L = b2.lib()
    r = su._VerifyPosResult()
    o = su._VerifyPosOpts(0, 1.0, 0, -1, 1, None)
    assert L.b200post_verify_pos(None, ctypes.byref(o), ctypes.byref(r), None) == b2.ERR_INVALID_ARGUMENT
    assert L.b200post_verify_pos(d.encode(), None, ctypes.byref(r), None) == b2.ERR_INVALID_ARGUMENT
    assert L.b200post_verify_pos(d.encode(), ctypes.byref(o), None, None) == b2.ERR_INVALID_ARGUMENT
    for bad in (dict(fraction=0.0), dict(fraction=-3.0), dict(fraction=100.01), dict(from_file=2, to_file=1),
                dict(to_file=4), dict(from_file=4), dict(provider_id=-7)):
        with pytest.raises(b2.B200PostError) as e:
            su.verify_pos(d, **{"fraction": 1.0, **bad})
        assert e.value.code == b2.ERR_INVALID_ARGUMENT, bad


def test_verify_pos_data_errors(su, b2, orc, tmp_path):
    with pytest.raises(b2.B200PostError) as e:
        su.verify_pos(str(tmp_path / "nowhere"))
    assert e.value.code == su.ERR_IO and "metadata file is missing" in str(e.value)
    d = _post(su, b2, orc, tmp_path / "post")
    p = Path(d) / "postdata_2.bin"
    p.write_bytes(p.read_bytes()[:-16])
    with pytest.raises(b2.B200PostError) as e:
        su.verify_pos(d, fraction=100.0)
    assert e.value.code == su.ERR_IO and "incomplete" in str(e.value)
    p.unlink()
    with pytest.raises(b2.B200PostError) as e:
        su.verify_pos(d)
    assert e.value.code == su.ERR_IO and "incomplete" in str(e.value)
    # outside the checked file range a damaged file does not matter to the host-side checks
    try:
        code = su.verify_pos(d, from_file=0, to_file=1).code      # with a GPU: the check runs
    except b2.B200PostError as e:
        code = e.code                                             # without one: ERR_NO_DEVICE
    assert code != su.ERR_IO


def test_valid_post_without_gpu_is_no_device(su, b2, orc, tmp_path):
    if b2.providers():
        pytest.skip("a CUDA device is present")
    d = _post(su, b2, orc, tmp_path / "post")
    for fraction in (100.0, 0.2):
        with pytest.raises(b2.B200PostError) as e:
            su.verify_pos(d, fraction=fraction)
        assert e.value.code == b2.ERR_NO_DEVICE
