"""CPU checks of the mode identifier: the long-double reference (tests/ident_reference.py) against closed forms and on the committed
recordings, the library's host-only classifier (jaero_ident_classify) against the reference, argument rejections, the ctypes
mirrors of the structs, and probe_carriers' host logic with the down-converter and the identifier stubbed out."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import ident_reference as ref
from conftest import ROOT, has_cuda, load_excerpt

FS_ALL = (12000, 24000, 44100, 48000)


def _two_tone(nfft, k1, k2, frames=4):
    """cos on bin k1 + cos on bin k2, int16 at half scale: its square holds lines at 2 k1, 2 k2 and, 4x stronger, k1 + k2"""
    n = np.arange((frames + 1) * nfft // 2)
    x = 0.25 * (np.cos(2 * np.pi * k1 * n / nfft) + np.cos(2 * np.pi * k2 * n / nfft))
    return np.round(x * 32768).astype(np.int16)


def _agree(got, want, what):
    assert got["mode"] == want["mode"], what
    for k in ("carrier_hz", "fb_hz", "margin_db"):
        assert abs(got[k] - want[k]) <= 1e-12 * max(1.0, abs(want[k])), (what, k, got[k], want[k])
    for a, b in zip(got["line_hz"], want["line_hz"]):
        assert abs(a - b) <= 1e-12 * max(1.0, abs(b)), (what, "line_hz", a, b)
    for m in ref.MODES:
        a, b = got["score_db"][m], want["score_db"][m]
        assert a == b or abs(a - b) <= 1e-12 * max(1.0, abs(b)), (what, m, a, b)


# ---------------------------------------------------------------- the reference against closed forms
@pytest.mark.parametrize("nfft", [1024, 4096])
def test_reference_cosine_at_a_bin_centre_gives_one_at_2f(nfft):
    """a full-scale int16 cosine: 1 at its 2f bin, within the int16 rounding of the samples"""
    k = 101
    x = np.cos(2 * np.pi * k * np.arange(3 * nfft) / nfft)
    sq, F = ref.spectrum(np.round(x * 32767)[None].astype(np.int16), nfft)
    assert F == 5
    i = 2 * k + nfft // 2
    assert np.argmax(sq[0]) == i
    assert abs(sq[0, i] * (32768 / 32767) ** 4 - 1.0) < 1e-4


def test_reference_unit_cosine_is_exactly_one():
    """without quantisation: the spectrum of the analytic signal's square of a bin-centred cosine is 1 at the 2f bin"""
    nfft, k = 2048, 300
    x = np.cos(2 * np.pi * k * np.arange(nfft, dtype=np.longdouble) / nfft)
    w = ref.hann(nfft)
    import scipy.fft
    X = scipy.fft.fft((w * x).astype(np.clongdouble))
    A = np.zeros_like(X); A[1:nfft // 2] = 2 * X[1:nfft // 2]
    a = scipy.fft.ifft(A)
    Y = scipy.fft.fft(a * a)
    p = abs(Y[2 * k]) ** 2 / np.sum(w * w) ** 2
    assert abs(float(p) - 1.0) < 1e-15


@pytest.mark.parametrize("fs,nfft", [(48000, 16384), (48000, 4096), (24000, 2048), (12000, 1024)])
def test_reference_two_tone_square_gives_its_pair_and_carrier(fs, nfft):
    """tones at fc -+ fb/4 on bin centres: the square's lines sit at 2 fc -+ fb/2, so the pair is 10.5 kbps and the carrier fc.
    A constant 1e-6 stands in for the noise floor; the lines' symmetric leakage leaves the fit's offsets at 0 within the int16
    rounding of the tones."""
    import jaero_b200
    D = int(10500 * nfft / fs)
    assert D * fs == 10500 * nfft and D % 4 == 0
    k1 = nfft // 32
    sq, _ = ref.spectrum(_two_tone(nfft, k1, k1 + D // 2)[None], nfft)
    row = sq[0] + 1e-6
    want = ref.classify(row, fs)
    _agree(jaero_b200.identify(row, fs), want, (fs, nfft))
    assert want["mode"] == "oqpsk10500" and want["bins"] == (2 * k1 + nfft // 2, 2 * k1 + D + nfft // 2)
    assert abs(want["carrier_hz"] - (k1 + D // 4) * fs / nfft) < 1e-3
    assert abs(want["fb_hz"] - 10500.0) < 1e-3


def test_reference_frames_count_once_complete():
    assert ref.frame_count(1023, 1024) == 0 and ref.frame_count(1024, 1024) == 1
    assert ref.frame_count(1535, 1024) == 1 and ref.frame_count(1536, 1024) == 2


# ---------------------------------------------------------------- the library's classifier against the reference
def _noise_row(rng, n, level=1.0):
    return level * (1.0 + 0.2 * rng.random(n))


def _put_pair(row, i, d, amp):
    n = len(row)
    for k, a in ((i, amp), (i + d, amp)):
        row[k % n] += a
        row[(k - 1) % n] += 0.3 * a
        row[(k + 1) % n] += 0.45 * a


@pytest.mark.parametrize("fs", FS_ALL)
@pytest.mark.parametrize("mode", ref.MODES)
def test_classify_matches_reference_on_constructed_pairs(fs, mode):
    import jaero_b200
    rng = np.random.default_rng(hash((fs, mode)) & 0xFFFF)
    nfft = 4096
    fb = ref.FBS[ref.MODES.index(mode)]
    d = fb * nfft / fs
    for t in range(3):
        row = _noise_row(rng, nfft)
        i = int(rng.integers(0, nfft))
        _put_pair(row, i, int(np.floor(d)) + t % 2, 20.0)
        got, want = jaero_b200.identify(row, fs), ref.classify(row, fs)
        _agree(got, want, (fs, mode, t))
        assert got["mode"] == mode


def test_classify_matches_reference_on_random_spectra():
    import jaero_b200
    rng = np.random.default_rng(5)
    for t in range(12):
        nfft = int(rng.choice([1024, 2048, 4096]))
        fs = int(rng.choice(FS_ALL))
        row = rng.exponential(size=nfft) if t % 2 else _noise_row(rng, nfft)
        _agree(jaero_b200.identify(row, fs), ref.classify(row, fs), t)
        prm = dict(threshold_db=float(rng.uniform(0, 10)), floor_window_hz=float(rng.uniform(50, 3000)), floor_quantile=float(rng.random()))
        _agree(jaero_b200.identify(row, fs, **prm), ref.classify(row, fs, **prm), (t, prm))


def test_classify_pair_wrapping_past_half_the_rate():
    """the upper line past +Fs/2 of the squared signal wraps to the bottom of the spectrum; the pair is still found"""
    import jaero_b200
    rng = np.random.default_rng(9)
    nfft, fs = 4096, 48000
    d = round(10500 * nfft / fs)
    row = _noise_row(rng, nfft)
    i = nfft - d // 3
    _put_pair(row, i, d, 30.0)
    got, want = jaero_b200.identify(row, fs), ref.classify(row, fs)
    _agree(got, want, "wrap")
    assert got["mode"] == "oqpsk10500" and want["bins"] == (i, i + d)
    assert abs(got["fb_hz"] - d * fs / nfft) < 0.5 * fs / nfft
    assert 0 <= got["carrier_hz"] < fs / 2


def test_classify_ties_take_the_first_bin_offset_and_mode():
    import jaero_b200
    nfft, fs = 1024, 48000
    row = np.ones(nfft)
    got, want = jaero_b200.identify(row, fs), ref.classify(row, fs)
    _agree(got, want, "flat")
    assert want["best"] == "msk600" and want["bins"] == (0, round(600 * nfft / fs) - 1)
    assert got["mode"] == "unknown" and got["margin_db"] == 0.0
    # two equal pairs of one mode: the lower bin wins
    row = np.ones(nfft)
    d = round(1200 * nfft / fs)
    _put_pair(row, 600, d, 50.0); _put_pair(row, 100, d, 50.0)
    got, want = jaero_b200.identify(row, fs), ref.classify(row, fs)
    _agree(got, want, "two pairs")
    assert want["bins"][0] == 100 and got["mode"] == "msk1200"


def test_classify_zeros_beside_a_line_give_no_offset():
    import jaero_b200
    nfft, fs = 2048, 48000
    d = round(8400 * nfft / fs)
    row = np.ones(nfft)
    row[500] = row[500 + d] = 100.0
    row[499] = 0.0; row[501 + d] = 3.0
    got, want = jaero_b200.identify(row, fs), ref.classify(row, fs)
    _agree(got, want, "zeros")
    assert got["mode"] == "oqpsk8400"
    assert got["line_hz"][0] == (500 - nfft // 2) * fs / nfft                 # zero neighbour: offset 0
    assert got["line_hz"][1] > (500 + d - nfft // 2) * fs / nfft              # the other line leans to its larger neighbour


def test_classify_floor_zero_gives_q_zero():
    import jaero_b200
    nfft, fs = 1024, 48000
    row = np.zeros(nfft)
    row[10] = row[10 + round(600 * nfft / fs)] = 1.0
    got, want = jaero_b200.identify(row, fs), ref.classify(row, fs)
    assert got["mode"] == want["mode"] == "unknown"
    assert all(v == -np.inf for v in got["score_db"].values()) and all(v == -np.inf for v in want["score_db"].values())


# ---------------------------------------------------------------- the committed recordings
@pytest.mark.parametrize("name,fs,fb,carriers", ref.EXCERPTS, ids=[e[0] for e in ref.EXCERPTS])
def test_reference_identifies_every_recording(name, fs, fb, carriers):
    import jaero_b200
    sq, F = ref.spectrum(load_excerpt(name)[None], 16384)
    r = ref.classify(sq[0], fs)
    assert r["mode"] == ref.MODES[ref.FBS.index(float(fb))], r
    assert r["margin_db"] >= ref.MARGINS[name], r
    assert min(abs(r["carrier_hz"] - c) for c in carriers) < 0.1, r
    assert abs(r["fb_hz"] - fb) < 1.0
    _agree(jaero_b200.identify(sq[0], fs), r, name)


# ---------------------------------------------------------------- arguments, device, layout
def test_classify_rejections():
    import jaero_b200
    row = np.ones(4096)
    for n in (512, 1000, 32768):
        with pytest.raises(jaero_b200.JaeroError, match="nfft"):
            jaero_b200.identify(np.ones(n), 48000)
    for fs in (7999, 192001, 44100.5, float("nan")):
        with pytest.raises(jaero_b200.JaeroError, match="Fs"):
            jaero_b200.identify(row, fs)
    for bad in (dict(threshold_db=float("inf")), dict(floor_window_hz=0.0), dict(floor_quantile=-0.1), dict(floor_quantile=1.5)):
        with pytest.raises(jaero_b200.JaeroError, match="parameter"):
            jaero_b200.identify(row, 48000, **bad)
    for v in (-1.0, float("nan"), float("inf")):
        p = row.copy(); p[17] = v
        with pytest.raises(jaero_b200.JaeroError, match="finite"):
            jaero_b200.identify(p, 48000)
    L = jaero_b200.lib()
    r = jaero_b200.IdentResult()
    assert L.jaero_ident_classify(None, 4096, 48000.0, None, ctypes.byref(r)) == -1
    assert L.jaero_ident_classify(row.ctypes.data_as(ctypes.c_void_p), 4096, 48000.0, None, None) == -1
    assert L.jaero_ident_classify(row.ctypes.data_as(ctypes.c_void_p), 4096, 48000.0, None, ctypes.byref(r)) == 0   # NULL params: defaults
    assert r.frames == 0


def test_ident_create_rejections():
    import jaero_b200
    for fs, c, nfft in ((48000, 1, 512), (48000, 1, 3000), (48000, 1, 32768), (48000, 0, 4096), (7000, 1, 4096), (200000, 1, 4096),
                        (44100.5, 1, 4096), (float("nan"), 1, 4096)):
        with pytest.raises(jaero_b200.JaeroError) as ei:
            jaero_b200.Identifier(fs, c, nfft)
        assert "error -1" in str(ei.value)                          # JAERO_E_ARG, checked before any device is looked for
    L = jaero_b200.lib()
    buf = np.zeros(8, dtype=np.int16)
    assert L.jaero_ident_write(None, buf.ctypes.data_as(ctypes.c_void_p), 4, 4) == -1
    assert L.jaero_ident_write_device(None, buf.ctypes.data_as(ctypes.c_void_p), 4, 4) == -1
    assert L.jaero_ident_read(None, None, None) == -1 and L.jaero_ident_reset(None) == -1
    assert L.jaero_ident_launch_count(None) == 0
    s = jaero_b200.Identifier.__new__(jaero_b200.Identifier)
    s.n = 2
    for pcm in (np.zeros((2, 8), dtype=np.int32), np.zeros((3, 8), dtype=np.int16), np.zeros(8, dtype=np.int16)):
        with pytest.raises(ValueError):
            s.write(pcm)


@pytest.mark.skipif(has_cuda(), reason="only meaningful on a box without a GPU")
def test_ident_create_fails_without_a_gpu():
    import jaero_b200
    h = ctypes.c_void_p()
    assert jaero_b200.lib().jaero_ident_create(48000.0, 4, 16384, 0, ctypes.byref(h)) == -2   # JAERO_E_CUDA: no CPU fallback
    with pytest.raises(jaero_b200.JaeroError):
        jaero_b200.Identifier(48000, 4)


def test_ident_structs_match_header_layout(tmp_path):
    """sizeof / offsetof of jaero_ident_params and jaero_ident_result as gcc sees include/jaero_b200.h == the ctypes mirrors"""
    import jaero_b200
    fields = ["carrier_hz", "fb_hz", "line_hz", "score_db", "margin_db", "frames", "mode"]
    pf = ["threshold_db", "floor_window_hz", "floor_quantile"]
    body = "".join('printf("%%zu ", offsetof(jaero_ident_result, %s));' % f for f in fields)
    body += "".join('printf("%%zu ", offsetof(jaero_ident_params, %s));' % f for f in pf)
    src = tmp_path / "ident_layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "jaero_b200.h"\nint main(void){printf("%zu %zu ",'
                   'sizeof(jaero_ident_result), sizeof(jaero_ident_params));' + body + 'printf("\\n");return 0;}\n')
    exe = str(tmp_path / "ident_layout")
    subprocess.run(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe], check=True)
    got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    R, P = jaero_b200.IdentResult, jaero_b200.IdentParams
    assert got == [ctypes.sizeof(R), ctypes.sizeof(P)] + [getattr(R, f).offset for f in fields] + [getattr(P, f).offset for f in pf]


# ---------------------------------------------------------------- probe_carriers with stubs
def test_probe_carriers_host_logic(monkeypatch):
    """probe_carriers with the down-converter and the identifier replaced by stubs: the set-up it asks for, the 0.1 s writes, and
    how it turns each channel's classification into a carrier for channel_plan"""
    import jaero_b200
    nfft, fs_in = 4096, 2.4e6
    bin_hz = 48000.0 / nfft
    d = round(10500 * nfft / 48000)
    k1 = 1028 - d // 4                                                 # carrier on bin 1028 = 12046.875 Hz: 46.875 Hz above 12 kHz
    good, _ = ref.spectrum(_two_tone(nfft, k1, k1 + d // 2, frames=6)[None], nfft)
    good = good[0] + 1e-9
    rng = np.random.default_rng(2)
    rows = np.stack([good, good, _noise_row(rng, nfft)])
    seen = {}

    class FakeDdc:
        FORMATS, _iq = jaero_b200.Ddc.FORMATS, staticmethod(jaero_b200.Ddc._iq)

        def __init__(self, input_rate, decimation, offsets_hz, audio_hz, bandwidth, transition, gain=1.0, device=0, interpolation=1):
            seen["ddc"] = dict(input_rate=input_rate, decimation=decimation, offsets=list(offsets_hz), audio=audio_hz, bw=bandwidth,
                               tr=transition, gain=gain, interpolation=interpolation)
            seen["writes"] = []
        def set_stream(self, s): seen["ddc_stream"] = s
        def write(self, iq, fmt): seen["writes"].append(iq.size // 2)
        def output(self): return 1234, 10, 16
        def close(self): seen["ddc_closed"] = True

    class FakeIdent:
        def __init__(self, Fs, n_channels, nfft=16384, device=0):
            seen["ident"] = (Fs, n_channels, nfft)
            seen["fed"] = 0
        def set_stream(self, s): seen["ident_stream"] = s
        def write_device(self, p, n, st): assert (p, n, st) == (1234, 10, 16); seen["fed"] += 1
        def read(self): return rows, 7
        def close(self): seen["ident_closed"] = True

    monkeypatch.setattr(jaero_b200, "Ddc", FakeDdc)
    monkeypatch.setattr(jaero_b200, "Identifier", FakeIdent)
    cands = [dict(center_hz=100e3, lo_hz=97e3, hi_hz=103e3, mode="oqpsk8400", power=4e-4, flags=0),
             dict(center_hz=-200e3, lo_hz=-200.5e3, hi_hz=-199.99e3, mode="oqpsk10500", power=1e-4, flags=0),
             dict(center_hz=300e3, lo_hz=299e3, hi_hz=301e3, mode="msk1200", power=1e-5, flags=0)]
    iq = np.zeros(2 * 600_000, dtype=np.int16)                       # 0.25 s at 2.4 MS/s
    out = jaero_b200.probe_carriers(cands, fs_in, iq, "cs16", nfft=nfft, stream=77)
    assert seen["ddc"] == dict(input_rate=fs_in, decimation=50, offsets=[100e3, -200e3, 300e3], audio=12000.0, bw=16000.0, tr=4000.0,
                               gain=0.2 * np.sqrt(2) / np.sqrt(4e-4), interpolation=1)
    assert seen["ident"] == (48000.0, 3, nfft) and seen["ddc_stream"] == seen["ident_stream"] == 77
    assert seen["writes"] == [240_000, 240_000, 120_000] and seen["fed"] == 3
    assert seen["ddc_closed"] and seen["ident_closed"]
    shift = (k1 + d // 4) * bin_hz - 12000.0
    assert out[0]["mode"] == "oqpsk10500" and out[0]["width_mode"] == "oqpsk8400"
    assert abs(out[0]["center_hz"] - (100e3 + shift)) < 1e-6 and abs(out[0]["fb_hz"] - 10500.0) < 1e-6
    assert out[0]["ident_score_db"] > 20
    assert out[1]["mode"] == "unknown" and out[1]["center_hz"] == -200e3      # identified centre outside the candidate's run
    assert out[2]["mode"] == "unknown" and out[2]["width_mode"] == "msk1200"  # nothing above the threshold
    assert cands[0]["mode"] == "oqpsk8400"                                     # the input list is left alone
    # seconds caps the stream; a rational radio rate takes its ratio from rate_ratio
    jaero_b200.probe_carriers(cands, 2.0e6, iq, "cs16", seconds=0.15, nfft=nfft, stream=77)
    assert (seen["ddc"]["interpolation"], seen["ddc"]["decimation"]) == jaero_b200.rate_ratio(2.0e6)
    assert seen["writes"] == [200_000, 100_000]
    assert jaero_b200.probe_carriers([], fs_in, iq, "cs16", stream=77) == []
