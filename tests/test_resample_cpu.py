"""CPU checks of the PCM rate converter's planner (include/jaero_b200.h, jaero_resample_plan): the reduced L/M of every supported
rate pair, each rejection with its message, the prototype against the filter specification on a dense frequency grid, and the
two forms of the numpy reference (tests/resample_reference.py) against each other. No GPU involved."""
from fractions import Fraction

import numpy as np
import pytest

import resample_reference as rr
from conftest import has_cuda

INPUTS = [8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 88200, 96000, 192000]
OUTPUTS = [48000, 24000, 12000]
PAIRS = [(a, b) for b in OUTPUTS for a in INPUTS if a != b]


def _plan(a, b, passband=None):
    import jaero_b200
    return jaero_b200.resample_plan(a, b, 0.45 * min(a, b) if passband is None else passband)


@pytest.mark.parametrize("a,b", PAIRS)
def test_plan_reduces_the_ratio(a, b):
    p = _plan(a, b)
    q = Fraction(b, a)
    assert (p["L"], p["M"]) == (q.numerator, q.denominator)
    assert p["L"] <= 1024 and p["M"] <= 1024 and len(p["h"]) == p["K"] <= 1 << 17
    assert abs(p["h"].sum() - p["L"]) < 1e-9 * p["L"]


def test_eleven_kilohertz_needs_more_interpolation_than_the_down_converter_allows():
    p = _plan(11025, 48000)
    assert (p["L"], p["M"]) == (640, 147)


@pytest.mark.parametrize("args,msg", [
    ((44100.5, 48000, 20000), "whole hertz"),
    ((44100, 48000.25, 20000), "whole hertz"),
    ((-44100, 48000, 20000), "whole hertz"),
    ((48000, 48000, 20000), "nothing to resample"),
    ((24000, 24000, 10000), "nothing to resample"),
    ((1000, 48001, 400), "must not exceed 1024"),                # L = 48001
    ((48001, 48000, 20000), "must not exceed 1024"),             # M = 48001
    ((44100, 48000, 22049), "taps"),                             # a 1 Hz transition at 7.056 MHz
    ((44100, 48000, 22050), "passband_hz"),
    ((44100, 48000, 30000), "passband_hz"),
    ((96000, 48000, 0), "passband_hz"),
])
def test_plan_rejects(args, msg):
    import jaero_b200
    with pytest.raises(jaero_b200.JaeroError, match=msg):
        jaero_b200.resample_plan(*args)


@pytest.mark.parametrize("a,b", PAIRS)
def test_prototype_meets_the_specification(a, b):
    """+-0.1 dB over [0, passband], at least 70 dB down over [min(rates)/2, L input_rate/2], on a grid 16 times denser than 1/K"""
    p = _plan(a, b)
    L, h = p["L"], p["h"] / p["L"]
    fs = L * a
    nfft = max(1 << 16, 1 << int(np.ceil(np.log2(16 * len(h)))))
    H = np.abs(np.fft.rfft(h, nfft))
    f = np.arange(len(H)) * fs / nfft
    pb = H[f <= 0.45 * min(a, b)]
    sb = H[f >= 0.5 * min(a, b)]
    assert np.abs(20 * np.log10(pb)).max() <= 0.1
    assert 20 * np.log10(sb.max()) <= -70.0


@pytest.mark.parametrize("a,b", [(44100, 48000), (8000, 48000), (96000, 48000), (44100, 24000), (48000, 12000), (22050, 48000)])
def test_polyphase_and_direct_forms_agree(a, b):
    p = _plan(a, b)
    rng = np.random.default_rng(a + b)
    x = rng.integers(-32768, 32768, size=(3, 3001)).astype(np.int16)
    x[2] = np.clip(np.round(40000 * np.sin(2 * np.pi * 1000 / a * np.arange(3001))), -32768, 32767).astype(np.int16)
    pcm, v, clipped = rr.resample_reference(x, p["h"], p["L"], p["M"])
    d = rr.resample_direct(x, p["h"], p["L"], p["M"])
    assert v.shape == d.shape == (3, rr.n_outputs(3001, p["L"], p["M"]))
    np.testing.assert_allclose(v, d, rtol=0, atol=1e-7)
    assert clipped[2] > 0                                        # the full-scale tone overshoots after filtering


@pytest.mark.skipif(has_cuda(), reason="only meaningful on a box without a GPU")
def test_resampler_needs_a_device():
    import jaero_b200
    with pytest.raises(jaero_b200.JaeroError, match="CUDA"):
        jaero_b200.Resampler(44100, 4)
