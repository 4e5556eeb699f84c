"""Plain long-double restatement of the streaming overlap-save FFT convolution (JFastFir, jaero_b200/csrc/fastfir.cuh) and the two
kernels the library runs through it, for the tests that compare the CUDA engine with it.

Contract (JAERO/tests/jfastfir_tests.cpp; L = nfft - K + 1): out[n] = sum_k h[k] x[n - L - k] for n >= 2L, and exactly 0 before.
The sum is a direct convolution (np.convolve) on np.clongdouble (80-bit extended precision on x86-64), about three decimal digits
more accurate than any double-precision FFT it is compared with. The taps are the exact double values the kernel receives,
widened to long double: the reference measures the kernel's arithmetic, not the taps' rounding.

Error bound (standard FP64 FFT analysis with margin): for each output block and the nfft-sample window u (K-1 history samples
plus the L-sample block) that produced it, ||y - y_ref||_2 <= 4 log2(nfft) 2^-52 max_k |H_k| ||u||_2, H = FFT of the zero-padded
taps."""
import math

import numpy as np
import scipy.fft

SIZES = ((2049, 4096), (2048, 8192))             # (K, nfft) pairs the library has a block kernel for


def block_length(K, nfft):
    return nfft - K + 1


def hilbert_taps(N=2048):
    """QJHilbertFilter::setSize(N) (JAERO/DSP.cpp:759-789): -1 at N/2, 0 at the other even taps, i (2/N) / tan(pi (i/N - 1/2)) at
    the odd ones. math.tan is the C library's tan, as the reference and the library use."""
    h = np.zeros(N, dtype=np.complex128)
    for i in range(N):
        if i == N // 2:
            h[i] = -1.0
        elif i % 2 == 0:
            h[i] = 0.0
        else:
            h[i] = complex(0.0, (2.0 / float(N)) / math.tan(math.pi * (float(i) / float(N) - 0.5)))
    return h


def k6_taps():
    """The 8400 bps pre-filter's kernel: RootRaisedCosine::design(0.6, 2048, 48000, 4200) (2049 taps), from the restated oracle"""
    from oracle import restated
    out = np.zeros(2049)
    n = restated.lib().jor_rrc_design(0.6, 2048, 48000.0, 4200.0, out.ctypes.data, len(out))
    assert n == 2049
    return out.astype(np.complex128)


def production_taps(K, nfft):
    return k6_taps() if (K, nfft) == (2049, 4096) else hilbert_taps(2048)


def spectrum(taps, nfft):
    """H = FFT(taps zero-padded to nfft), long double"""
    h = np.zeros(nfft, dtype=np.clongdouble)
    h[:len(taps)] = np.asarray(taps).astype(np.clongdouble)
    return scipy.fft.fft(h)


def convolve(taps, x, nfft):
    """The JFastFir output of one channel x [n] (complex) in long double"""
    K = len(taps)
    L = block_length(K, nfft)
    x = np.asarray(x)
    n = len(x)
    y = np.zeros(n, dtype=np.clongdouble)
    if n > 2 * L:
        full = np.convolve(x[:n - L].astype(np.clongdouble), np.asarray(taps).astype(np.clongdouble))
        y[2 * L:] = full[L:n - L]
    return y


def block_bounds(taps, x, nfft):
    """Per output block b >= 2 (samples [bL, (b+1)L) of the output): (start, stop, bound) with the bound of the module docstring"""
    K = len(taps)
    L, K1 = block_length(K, nfft), K - 1
    hmax = float(np.max(np.abs(spectrum(taps, nfft))))
    c = 4.0 * math.log2(nfft) * 2.0 ** -52 * hmax
    out = []
    x = np.asarray(x)
    for b in range(2, len(x) // L + 1):
        m = b - 1                                  # input block m produced output block b
        u = x[m * L - K1:(m + 1) * L]
        stop = min((b + 1) * L, len(x))
        if stop > b * L:
            out.append((b * L, stop, c * float(np.linalg.norm(u))))
    return out
