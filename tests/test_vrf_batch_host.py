"""CPU tier: the host checks of batched VRF-nonce verification (b200post_verify_vrf_nonces[_multi] and
b200post_verifier_verify_vrf_nonce): argument checks in their documented order, no CPU path, no device without a GPU,
and the single calls (b200post_verify_vrf_nonce, b200post_vrf_nonce_label), which now run through the batch call,
keeping the codes they give before the device is involved."""
import ctypes
import importlib

import pytest

NODE, ATX = bytes(range(32)), bytes(range(32, 64))


def _batch(b2, provider, n, checks=True, statuses=True, valid=True, labels=True):
    """The C call itself, so that NULL arrays can be passed."""
    L = b2.lib()
    L.b200post_verify_vrf_nonces.argtypes = [ctypes.c_uint32, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p,
                                             ctypes.c_void_p, ctypes.c_void_p]
    m = max(n, 1)
    cs = (b2.VrfCheck * m)(*[b2.vrf_check(NODE, ATX, i, 4, 1024, 2) for i in range(m)])
    st, ok, lab = (ctypes.c_int * m)(), (ctypes.c_int * m)(), ctypes.create_string_buffer(32 * m)
    return L.b200post_verify_vrf_nonces(provider, n, cs if checks else None, st if statuses else None, ok if valid else None,
                                        lab if labels else None)


def _multi(b2, providers, n_providers, n, checks=True, statuses=True, valid=True):
    L = b2.lib()
    L.b200post_verify_vrf_nonces_multi.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.c_void_p,
                                                   ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    m = max(n, 1)
    cs = (b2.VrfCheck * m)(*[b2.vrf_check(NODE, ATX, i, 4, 1024, 2) for i in range(m)])
    st, ok = (ctypes.c_int * m)(), (ctypes.c_int * m)()
    arr = (ctypes.c_uint32 * max(len(providers), 1))(*providers) if providers is not None else None
    return L.b200post_verify_vrf_nonces_multi(arr, n_providers, n, cs if checks else None, st if statuses else None,
                                              ok if valid else None, None)


def _single(b2, provider, nonce=5, node=NODE, atx=ATX, units=4, lpu=1024, n=8192):
    L = b2.lib()
    L.b200post_verify_vrf_nonce.argtypes = [ctypes.c_uint32, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint32,
                                            ctypes.c_uint64, ctypes.c_uint64, ctypes.POINTER(ctypes.c_int)]
    valid = ctypes.c_int(7)
    rc = L.b200post_verify_vrf_nonce(provider, nonce, node, atx, units, lpu, n, ctypes.byref(valid))
    return rc, valid.value


def _label(b2, provider, nonce=5, node=NODE, atx=ATX, n=8192, out=True):
    L = b2.lib()
    L.b200post_vrf_nonce_label.argtypes = [ctypes.c_uint32, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint64,
                                           ctypes.c_void_p]
    return L.b200post_vrf_nonce_label(provider, nonce, node, atx, n, ctypes.create_string_buffer(32) if out else None)


def test_check_struct_layout(b2):
    """b200post_vrf_check as include/b200post_verify.h declares it (the Go and C callers build it natively)."""
    C = b2.VrfCheck
    assert ctypes.sizeof(C) == 96
    assert [(f, getattr(C, f).offset) for f, _ in C._fields_] == [
        ("node_id", 0), ("commitment_atx_id", 32), ("nonce", 64), ("labels_per_unit", 72), ("scrypt_n", 80),
        ("num_units", 88), ("prioritized", 92)]


def test_batch_argument_checks(b2):
    """NULL arrays with n > 0 are refused before anything else, also on the CPU provider id; labels32 may be NULL."""
    for provider in (0, b2.CPU_PROVIDER_ID):
        for kw in (dict(checks=False), dict(statuses=False), dict(valid=False)):
            assert _batch(b2, provider, 3, **kw) == b2.ERR_INVALID_ARGUMENT, (provider, kw)
    for provs, n_prov, kw in ((None, 1, {}), (None, 2, {}), ([0], 0, {}), ([0, 0], -1, {}), ([0, 0], 2, dict(checks=False)),
                              ([0], 1, dict(statuses=False)), ([0, 0], 2, dict(valid=False))):
        assert _multi(b2, provs, n_prov, 3, **kw) == b2.ERR_INVALID_ARGUMENT, (provs, n_prov, kw)
    with pytest.raises(b2.B200PostError) as e:
        b2.verify_vrf_nonces([(NODE, ATX, 1, 4, 1024, 2)], providers=[])
    assert e.value.code == b2.ERR_INVALID_ARGUMENT


def test_verifier_call_argument_checks(b2):
    vf = importlib.import_module("go-spacemesh_b200.verify")
    L = vf._bind()
    ok = ctypes.c_int(0)
    c = b2.vrf_check(NODE, ATX, 1, 4, 1024, 2)
    assert L.b200post_verifier_verify_vrf_nonce(None, ctypes.byref(c), ctypes.byref(ok), None) == b2.ERR_INVALID_ARGUMENT


def test_cpu_provider_is_unsupported(b2):
    """There is no CPU path: the CPU provider id is refused before the n == 0 shortcut, by every entry point."""
    for n in (0, 2):
        assert _batch(b2, b2.CPU_PROVIDER_ID, n) == b2.ERR_UNSUPPORTED, n
        assert _batch(b2, b2.CPU_PROVIDER_ID, n, labels=False) == b2.ERR_UNSUPPORTED, n
    for provs in ([b2.CPU_PROVIDER_ID], [b2.CPU_PROVIDER_ID] * 2):
        for n in (0, 1, 5):
            assert _multi(b2, provs, len(provs), n) == b2.ERR_UNSUPPORTED, (provs, n)
        with pytest.raises(b2.B200PostError) as e:
            b2.verify_vrf_nonces([(NODE, ATX, 1, 4, 1024, 2)] * 3, providers=provs)
        assert e.value.code == b2.ERR_UNSUPPORTED
    with pytest.raises(b2.B200PostError) as e:
        b2.verify_vrf_nonces([(NODE, ATX, 1, 4, 1024, 2)], provider=b2.CPU_PROVIDER_ID)
    assert e.value.code == b2.ERR_UNSUPPORTED
    assert _single(b2, b2.CPU_PROVIDER_ID) == (b2.ERR_UNSUPPORTED, 0)
    assert _label(b2, b2.CPU_PROVIDER_ID) == b2.ERR_UNSUPPORTED


def test_single_calls_keep_their_argument_codes(b2):
    """b200post_verify_vrf_nonce and b200post_vrf_nonce_label judge their own arguments before the provider and the
    device, as they did before they became the one-check case of the batch call: the same codes on any box."""
    for provider in (0, 7, b2.CPU_PROVIDER_ID):
        assert _single(b2, provider, units=0) == (b2.ERR_INVALID_ARGUMENT, 0)
        assert _single(b2, provider, lpu=0) == (b2.ERR_INVALID_ARGUMENT, 0)
        assert _single(b2, provider, units=2**32 - 1, lpu=2**40) == (b2.ERR_INVALID_ARGUMENT, 0)   # numLabels >= 2^64
        assert _single(b2, provider, node=None)[0] == b2.ERR_INVALID_ARGUMENT
        assert _single(b2, provider, atx=None)[0] == b2.ERR_INVALID_ARGUMENT
        assert _label(b2, provider, node=None) == b2.ERR_INVALID_ARGUMENT
        assert _label(b2, provider, out=False) == b2.ERR_INVALID_ARGUMENT
        for n in (0, 1, 3, 6144, 2**21):
            assert _single(b2, provider, n=n) == (b2.ERR_INVALID_ARGUMENT, 0), (provider, n)
            assert _label(b2, provider, n=n) == b2.ERR_INVALID_ARGUMENT, (provider, n)


def test_no_device_no_cpu_path(b2):
    if b2.providers():
        pytest.skip("a CUDA device is present: the no-device contract is covered on CPU-only boxes")
    for n in (0, 1, 3):
        assert _batch(b2, 0, n) == b2.ERR_NO_DEVICE, n
        assert _batch(b2, 0, n, labels=False) == b2.ERR_NO_DEVICE, n
    for provs in ([0], [0, 0], [0, 1, 2], [0, b2.CPU_PROVIDER_ID]):
        for n in (0, 1, 4):
            assert _multi(b2, provs, len(provs), n) == b2.ERR_NO_DEVICE, (provs, n)
    with pytest.raises(b2.B200PostError) as e:
        b2.verify_vrf_nonces([(NODE, ATX, 1, 4, 1024, 2)] * 3, providers=[0, 0])
    assert e.value.code == b2.ERR_NO_DEVICE
    # the single calls now run through the batch call: still NO_DEVICE, nonces past the end included
    for nonce in (0, 5, 4096, 2**40, 2**64 - 1):
        assert _single(b2, 0, nonce=nonce) == (b2.ERR_NO_DEVICE, 0)
        assert _label(b2, 0, nonce=nonce) == b2.ERR_NO_DEVICE
    with pytest.raises(b2.B200PostError) as e:
        b2.verify_vrf_nonce(5, NODE, ATX, 4, 1024, 2)
    assert e.value.code == b2.ERR_NO_DEVICE
