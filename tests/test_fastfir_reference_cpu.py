"""CPU tests: pin the long-double FFT-convolution reference (tests/fastfir_reference.py) to the reference's own JFastFir and
QJHilbertFilter (oracle/_ref/libjaero_ref_fastfir.so), and to the reference's JFastFir golden (oracle/_ref/libjaero_ref.so),
so that the GPU tests that measure the CUDA engine against it measure against the right thing."""
import numpy as np
import pytest

import fastfir_reference as fr
from oracle import ref

needs_ref = pytest.mark.skipif(not ref.available(), reason="oracle/_ref not built (needs /root/reference)")
needs_ref_fastfir = pytest.mark.skipif(not ref.fastfir_available(), reason="oracle/_ref/libjaero_ref_fastfir.so not built (needs /root/reference)")


def _ri(a):
    return np.ascontiguousarray(np.stack([np.real(a), np.imag(a)], axis=-1).astype(np.float64))


def _jfastfir(taps, x, nfft, writes):
    buf = _ri(x)
    h = _ri(taps)
    w = np.ascontiguousarray(writes, dtype=np.int32)
    ref.fastfir_lib().jref_jfastfir(h.ctypes.data, len(taps), nfft, buf.ctypes.data, len(x), w.ctypes.data, len(w))
    return buf[:, 0] + 1j * buf[:, 1]


@needs_ref_fastfir
def test_hilbert_taps_equal_reference():
    """the restated QJHilbertFilter kernel is the reference's, bit for bit"""
    out = np.zeros((2048, 2))
    assert ref.fastfir_lib().jref_hilbert_kernel(out.ctypes.data) == 2048
    got = fr.hilbert_taps(2048)
    assert np.array_equal(got.real, out[:, 0]) and np.array_equal(got.imag, out[:, 1])


def test_k6_taps_shape():
    h = fr.k6_taps()
    assert len(h) == 2049 and not h.imag.any() and np.argmax(np.abs(h)) == 1024


@needs_ref_fastfir
@pytest.mark.parametrize("K,nfft", fr.SIZES)
@pytest.mark.parametrize("pattern", ["whole", "piecewise"])
def test_reference_equals_jfastfir(K, nfft, pattern):
    """fastfir_reference equals the reference's JFastFir within 1e-12 of the output scale, whole-stream and piecewise writes"""
    L = fr.block_length(K, nfft)
    rng = np.random.default_rng(K + nfft)
    n = 5 * L + 77
    x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    x[:L // 3] = rng.integers(-32768, 32768, L // 3) / 32768.0          # a stretch of real full-scale samples
    taps = fr.production_taps(K, nfft)
    if pattern == "whole":
        writes = [n]
    else:
        sizes = [1, L - 2, 1, 1, L - 1, L + 1, 3 * L + 5]
        writes, left = [], n
        for s in sizes:
            s = min(s, left)
            if s > 0:
                writes.append(s); left -= s
        while left > 0:
            s = min(int(rng.integers(1, 3000)), left); writes.append(s); left -= s
    got = _jfastfir(taps, x, nfft, writes)
    want = fr.convolve(taps, x, nfft)
    scale = float(np.max(np.abs(want)))
    assert scale > 0
    assert not got[:2 * L].any() and not want[:2 * L].any()
    err = float(np.max(np.abs(got.astype(np.clongdouble) - want)))
    assert err <= 1e-12 * scale, "max error %.3g of scale %.3g" % (err, scale)


@needs_ref
def test_reference_reproduces_jfastfir_golden():
    """the reference's own 10 000-sample JFastFir golden (jfastfir_tests.cpp:31-58) through fastfir_reference"""
    L = ref.lib()
    n = L.jref_golden_jfastfir_len()
    gi = np.zeros((n, 2)); go = np.zeros((n, 2))
    L.jref_golden_jfastfir(gi.ctypes.data, go.ctypes.data)
    Fs, fb = L.jref_golden_jfastfir_Fs(), L.jref_golden_jfastfir_fb()
    taps = np.zeros(2049)
    assert L.jref_rrc_design(0.6, 2048, Fs, fb / 2, taps.ctypes.data, len(taps)) == 2049
    y = fr.convolve(taps.astype(np.complex128), gi[:, 0] + 1j * gi[:, 1], 4096).astype(np.complex128)
    assert np.abs(y.real - go[:, 0]).max() < 1e-5 and np.abs(y.imag - go[:, 1]).max() < 1e-5


def test_block_bounds_cover_every_output():
    """every output sample from 2L on belongs to exactly one bounded block"""
    for K, nfft in fr.SIZES:
        L = fr.block_length(K, nfft)
        x = np.ones(4 * L + 3, dtype=np.complex128)
        blocks = fr.block_bounds(np.ones(K), x, nfft)
        covered = np.zeros(len(x), dtype=int)
        for a, b, bound in blocks:
            covered[a:b] += 1
            assert bound > 0
        assert (covered[2 * L:] == 1).all() and (covered[:2 * L] == 0).all()
