"""CPU checks of the front-end stages' C boundary (down-converter, rate converter, carrier scanner, mode identifier): every entry
point called with a null handle or a null buffer returns JAERO_E_ARG with its exact error text, and the host-only checks of
the carrier finder and the classifier fire in their stated order. None of this needs a device."""
import ctypes

import numpy as np
import pytest

E_ARG = -1


def _lib():
    import jaero_b200
    return jaero_b200, jaero_b200.lib()


def _err(L):
    return L.jaero_last_error().decode()


def _null_calls(jb, L):
    buf = np.zeros(64, dtype=np.int16)
    p = buf.ctypes.data_as(ctypes.c_void_p)
    sz, vp, i64 = ctypes.c_size_t(), ctypes.c_void_p(), ctypes.c_int64()
    frames = ctypes.c_int64()
    by = ctypes.byref
    return [
        # down-converter
        ("jaero_ddc_write", lambda h: L.jaero_ddc_write(h, p, 4, jb.IQ_CS16), "jaero_ddc_write: null argument"),
        ("jaero_ddc_write", lambda h: L.jaero_ddc_write(h, None, 4, jb.IQ_CS16), "jaero_ddc_write: null argument"),
        ("jaero_ddc_write_device", lambda h: L.jaero_ddc_write_device(h, p, 4, jb.IQ_CS16), "jaero_ddc_write_device: null argument"),
        ("jaero_ddc_write_device", lambda h: L.jaero_ddc_write_device(h, p, 4, 7), "jaero_ddc_write_device: null argument"),
        ("jaero_ddc_output", lambda h: L.jaero_ddc_output(h, by(vp), by(sz), by(sz)), "jaero_ddc_output: null argument"),
        ("jaero_ddc_read_pcm", lambda h: L.jaero_ddc_read_pcm(h, p, 64, by(sz)), "jaero_ddc_read_pcm: null argument"),
        ("jaero_ddc_set_stream", lambda h: L.jaero_ddc_set_stream(h, None), "null handle"),
        ("jaero_ddc_set_offset", lambda h: L.jaero_ddc_set_offset(h, 0, 0.0), "jaero_ddc_set_offset: bad argument"),
        ("jaero_ddc_set_audio_freq", lambda h: L.jaero_ddc_set_audio_freq(h, 0, 8000.0), "jaero_ddc_set_audio_freq: bad argument"),
        ("jaero_ddc_get_stats", lambda h: L.jaero_ddc_get_stats(h, by(i64), None), "null handle"),
        # rate converter
        ("jaero_resample_write", lambda h: L.jaero_resample_write(h, p, 4, 4), "jaero_resample_write: null argument"),
        ("jaero_resample_write", lambda h: L.jaero_resample_write(h, p, 8, 4), "jaero_resample_write: null argument"),
        ("jaero_resample_write_device", lambda h: L.jaero_resample_write_device(h, p, 4, 4), "jaero_resample_write_device: null argument"),
        ("jaero_resample_output", lambda h: L.jaero_resample_output(h, by(vp), by(sz), by(sz)), "jaero_resample_output: null argument"),
        ("jaero_resample_read_pcm", lambda h: L.jaero_resample_read_pcm(h, p, 64, by(sz)), "jaero_resample_read_pcm: null argument"),
        ("jaero_resample_set_stream", lambda h: L.jaero_resample_set_stream(h, None), "null handle"),
        ("jaero_resample_get_stats", lambda h: L.jaero_resample_get_stats(h, by(i64), None), "null handle"),
        # carrier scanner
        ("jaero_scan_write", lambda h: L.jaero_scan_write(h, p, 4, jb.IQ_CU8), "jaero_scan_write: null argument"),
        ("jaero_scan_write", lambda h: L.jaero_scan_write(h, p, 4, 7), "jaero_scan_write: null argument"),
        ("jaero_scan_write_device", lambda h: L.jaero_scan_write_device(h, p, 4, jb.IQ_CU8), "jaero_scan_write_device: null argument"),
        ("jaero_scan_set_stream", lambda h: L.jaero_scan_set_stream(h, None), "null handle"),
        ("jaero_scan_reset", lambda h: L.jaero_scan_reset(h), "null handle"),
        ("jaero_scan_read", lambda h: L.jaero_scan_read(h, None, None, by(frames)), "null handle"),
        # mode identifier
        ("jaero_ident_write", lambda h: L.jaero_ident_write(h, p, 4, 4), "jaero_ident_write: null argument"),
        ("jaero_ident_write", lambda h: L.jaero_ident_write(h, p, 8, 4), "jaero_ident_write: null argument"),
        ("jaero_ident_write_device", lambda h: L.jaero_ident_write_device(h, p, 4, 4), "jaero_ident_write_device: null argument"),
        ("jaero_ident_set_stream", lambda h: L.jaero_ident_set_stream(h, None), "null handle"),
        ("jaero_ident_reset", lambda h: L.jaero_ident_reset(h), "null handle"),
        ("jaero_ident_read", lambda h: L.jaero_ident_read(h, None, by(frames)), "null handle"),
    ]


def test_null_handle_of_every_stage_entry_point():
    jb, L = _lib()
    for name, call, msg in _null_calls(jb, L):
        L.jaero_last_error()
        assert call(None) == E_ARG, name
        assert _err(L) == msg, (name, _err(L))


def test_null_buffers_are_rejected_with_the_null_argument_text():
    """a null data pointer on a null handle: the same first check as a null handle, one message per entry point"""
    jb, L = _lib()
    sz, vp = ctypes.c_size_t(), ctypes.c_void_p()
    cases = [
        (lambda: L.jaero_ddc_write_device(None, None, 0, jb.IQ_CU8), "jaero_ddc_write_device: null argument"),
        (lambda: L.jaero_scan_write_device(None, None, 0, jb.IQ_CU8), "jaero_scan_write_device: null argument"),
        (lambda: L.jaero_resample_write_device(None, None, 0, 0), "jaero_resample_write_device: null argument"),
        (lambda: L.jaero_ident_write_device(None, None, 0, 0), "jaero_ident_write_device: null argument"),
        (lambda: L.jaero_ident_write(None, None, 0, 0), "jaero_ident_write: null argument"),
        (lambda: L.jaero_ddc_read_pcm(None, None, 0, ctypes.byref(sz)), "jaero_ddc_read_pcm: null argument"),
        (lambda: L.jaero_resample_read_pcm(None, None, 0, None), "jaero_resample_read_pcm: null argument"),
        (lambda: L.jaero_ddc_output(None, ctypes.byref(vp), None, ctypes.byref(sz)), "jaero_ddc_output: null argument"),
        (lambda: L.jaero_resample_output(None, None, ctypes.byref(sz), ctypes.byref(sz)), "jaero_resample_output: null argument"),
    ]
    for call, msg in cases:
        assert call() == E_ARG
        assert _err(L) == msg


def test_null_handle_counters_and_destroys():
    _, L = _lib()
    for stage in ("ddc", "resample", "scan", "ident"):
        assert getattr(L, "jaero_%s_launch_count" % stage)(None) == 0
        getattr(L, "jaero_%s_destroy" % stage)(None)


def _find(L, jb, psd, nfft, rate=2.4e6):
    n = ctypes.c_int(-5)
    prm = jb.ScanParams(3.0, 100e3, 0.25, 200.0, 0.0)
    p = None if psd is None else psd.ctypes.data_as(ctypes.c_void_p)
    return L.jaero_scan_find_carriers(p, nfft, rate, ctypes.byref(prm), None, 0, ctypes.byref(n)), _err(L)


def _classify(L, jb, sq, nfft, Fs=48000.0):
    prm = jb.IdentParams(5.0, 400.0, 0.5)
    r = jb.IdentResult()
    p = None if sq is None else sq.ctypes.data_as(ctypes.c_void_p)
    return L.jaero_ident_classify(p, nfft, Fs, ctypes.byref(prm), ctypes.byref(r)), _err(L)


@pytest.mark.parametrize("bad", [-1.0, np.nan, np.inf])
def test_spectrum_checks_of_the_carrier_finder_and_the_classifier(bad):
    """nfft range first, then every bin finite and >= 0; the rest of each call is unchanged by a rejected spectrum"""
    jb, L = _lib()
    for nfft in (1024, 4096, 16384):
        psd = np.ones(nfft)
        psd[nfft // 3] = bad
        assert _find(L, jb, psd, nfft) == (E_ARG, "jaero_scan_find_carriers: spectrum values must be finite and >= 0")
        assert _classify(L, jb, psd, nfft) == (E_ARG, "jaero_ident_classify: spectrum values must be finite and >= 0")
    psd = np.full(65536, bad)
    assert _find(L, jb, psd, 65536) == (E_ARG, "jaero_scan_find_carriers: spectrum values must be finite and >= 0")
    for nfft in (512, 1000, 3000, 131072, 0, -1024):
        psd = np.full(max(nfft, 1), bad)
        assert _find(L, jb, psd, nfft) == (E_ARG, "jaero_scan_find_carriers: nfft must be a power of two from 1024 to 65536")
    for nfft in (512, 1000, 32768, 65536, 0):
        psd = np.full(max(nfft, 1), bad)
        assert _classify(L, jb, psd, nfft) == (E_ARG, "jaero_ident_classify: nfft must be a power of two from 1024 to 16384")


def test_host_only_entry_points_accept_a_clean_spectrum():
    jb, L = _lib()
    for nfft in (1024, 16384):
        assert _find(L, jb, np.ones(nfft), nfft)[0] == 0
        assert _classify(L, jb, np.ones(nfft), nfft)[0] == 0
    assert _find(L, jb, np.ones(65536), 65536)[0] == 0
    assert _find(L, jb, None, 1024) == (E_ARG, "jaero_scan_find_carriers: bad argument")
    assert _classify(L, jb, None, 1024) == (E_ARG, "jaero_ident_classify: null argument")


def test_create_checks_that_come_before_the_device():
    jb, L = _lib()
    h = ctypes.c_void_p()
    by = ctypes.byref
    for nfft in (512, 1000, 131072):
        assert L.jaero_scan_create(2.4e6, nfft, 256, 0, by(h)) == E_ARG
        assert _err(L) == "jaero_scan_create: nfft must be a power of two from 1024 to 65536"
    for nfft in (512, 1000, 32768):
        assert L.jaero_ident_create(48000.0, 1, nfft, 0, by(h)) == E_ARG
        assert _err(L) == "jaero_ident_create: nfft must be a power of two from 1024 to 16384"
    assert L.jaero_ident_create(48000.5, 1, 4096, 0, by(h)) == E_ARG
    assert _err(L) == "jaero_ident_create: Fs must be whole hertz from 8000 to 192000"
    assert L.jaero_scan_create(2.4e6, 4096, 4097, 0, by(h)) == E_ARG
    assert _err(L) == "jaero_scan_create: hop must be in [1, nfft]"
