"""CPU checks of the carrier scanner: the float64 reference (tests/scan_reference.py) against closed forms, the library's host-only
carrier finder (jaero_scan_find_carriers) against the reference, argument rejections, and the ctypes mirrors of the structs."""
import ctypes
import os
import subprocess
import time

import numpy as np
import pytest

import scan_reference as ref
from conftest import ROOT, has_cuda

FLOAT_FIELDS = ("center_hz", "peak_hz", "lo_hz", "hi_hz", "width_hz", "power", "snr_db", "peak_db", "floor")


# ---------------------------------------------------------------- the reference against closed forms
@pytest.mark.parametrize("nfft", [1024, 4096])
def test_reference_tone_at_a_bin_centre(nfft):
    """unit-amplitude tone on bin k: mean = nfft / 1.5 there ((sum w)^2 / sum w^2 for the Hann window) and (1/nfft) sum(mean) = 1"""
    k = 37
    n = np.arange(5 * nfft)
    x = np.exp(2j * np.pi * k * n / nfft)
    mean, mx, F = ref.scan(x, nfft, nfft // 2)
    assert F == 9
    i = k + nfft // 2                                              # fftshift position of bin k
    assert np.argmax(mean) == i
    assert abs(mean[i] - nfft / 1.5) < 1e-9 * nfft
    assert abs(np.sum(mean) / nfft - 1.0) < 1e-12
    np.testing.assert_allclose(mx, mean, rtol=1e-12, atol=1e-20)
    assert abs(ref.freqs(nfft, 2.4e6)[i] - k * 2.4e6 / nfft) < 1e-9


def test_reference_white_noise_level():
    """complex white noise of variance s^2 averages to s^2 within 3/sqrt(F) relative (the per-bin standard deviation is
    1/sqrt(F), so 3 sigma holds in all but ~0.3 % of the bins); the level over all bins within 3/sqrt(F nfft)"""
    rng = np.random.default_rng(1)
    nfft, s2 = 1024, 0.37
    x = (rng.standard_normal(400 * nfft) + 1j * rng.standard_normal(400 * nfft)) * np.sqrt(s2 / 2)
    mean, _, F = ref.scan(x, nfft, nfft)
    assert F == 400
    assert np.mean(np.abs(mean / s2 - 1) < 3 / np.sqrt(F)) > 0.99
    assert abs(np.mean(mean) / s2 - 1) < 3 / np.sqrt(F * nfft)


def test_reference_fftshift_order_and_bin_frequencies():
    nfft, rate = 1024, 96000.0
    f = ref.freqs(nfft, rate)
    assert f[0] == -rate / 2 and f[nfft // 2] == 0.0 and f[-1] == rate / 2 - rate / nfft
    for k in (-300, -1, 1, 511):                                    # a tone at k bins lands at index k + nfft/2
        x = np.exp(2j * np.pi * k * np.arange(2 * nfft) / nfft)
        mean, _, _ = ref.scan(x, nfft, nfft)
        assert np.argmax(mean) == k + nfft // 2


def test_reference_frames_count_once_complete():
    x = np.ones(3000, dtype=complex)
    assert ref.scan(x, 1024, 777)[2] == 3                           # frames at 0, 777, 1554; the one at 2331 needs 3355
    assert ref.scan(x[:1023], 1024, 1)[2] == 0


# ---------------------------------------------------------------- the library's carrier finder against the reference
def _lib_find(psd, rate, **params):
    import jaero_b200
    return jaero_b200.find_carriers(psd, rate, **params)


def _assert_same(psd, rate, **params):
    got = _lib_find(psd, rate, **params)
    exp = ref.find_carriers(psd, rate, **params)
    assert len(got) == len(exp), (len(got), len(exp))
    bin_hz = rate / len(psd)
    for g, e in zip(got, exp):
        assert round(g["lo_hz"] / bin_hz) == e["lo"] - len(psd) // 2 and round(g["hi_hz"] / bin_hz) == e["hi"] - len(psd) // 2
        assert g["mode"] == e["mode"] and g["flags"] == e["flags"]
        for f in FLOAT_FIELDS:
            assert abs(g[f] - e[f]) <= 1e-12 * e["_scale"][f], (f, g[f], e[f])
    return got


def _shape(df, kind, r):
    """peak-normalised spectra: ('rc', Rs, alpha) raised cosine of symbol rate Rs (OQPSK with RRC pulses), ('msk', fb) MSK"""
    if kind == "msk":
        x = df / r[0]
        d = 1 - 16 * x * x
        safe = np.where(np.abs(d) < 1e-9, 1.0, d)
        return np.where(np.abs(d) < 1e-9, (np.pi / 4) ** 2, (np.cos(2 * np.pi * x) / safe) ** 2)
    Rs, a = r
    u = np.abs(df)
    f1, f2 = (1 - a) * Rs / 2, (1 + a) * Rs / 2
    return np.where(u <= f1, 1.0, np.where(u <= f2, 0.5 * (1 + np.cos(np.pi / (a * Rs) * (u - f1))), 0.0))


def _synthetic_psd(nfft, rate, carriers, rng, frames=64):
    """noise floor 1 (chi-square of 2*frames degrees of freedom, scaled to mean 1) plus carriers (centre, shape, level)"""
    psd = rng.chisquare(2 * frames, size=nfft) / (2 * frames)
    f = ref.freqs(nfft, rate)
    for c, (kind, *r), lv in carriers:
        psd += lv * _shape(f - c, kind, r)
    return psd


OQ10500, OQ8400, MSK1200, MSK600 = ("rc", 5250.0, 1.0), ("rc", 4200.0, 0.6), ("msk", 1200.0), ("msk", 600.0)


@pytest.mark.parametrize("seed", range(6))
def test_find_carriers_equals_reference_on_random_spectra(seed):
    rng = np.random.default_rng(seed)
    nfft = int(rng.choice([1024, 4096, 16384]))
    rate = float(rng.choice([96000.0, 2.4e6]))
    psd = rng.exponential(1.0, size=nfft) * (1 + 50 * (rng.random(nfft) < 0.05))
    params = dict(threshold_db=float(rng.uniform(1, 6)), floor_window_hz=float(rng.uniform(0.01, 0.5)) * rate,
                  floor_quantile=float(rng.uniform(0, 1)), min_width_hz=float(rng.uniform(0, 4)) * rate / nfft)
    _assert_same(psd, rate, **params)


def test_find_carriers_equals_reference_at_band_edges_and_dc():
    rng = np.random.default_rng(7)
    nfft, rate = 16384, 2.4e6
    half = rate / 2
    carriers = [(-half + 1000.0, OQ10500, 30.0), (half - 2000.0, OQ10500, 30.0), (0.0, OQ8400, 100.0), (150e3, OQ10500, 20.0),
                (-400e3, MSK1200, 15.0), (420e3, MSK600, 15.0)]
    psd = _synthetic_psd(nfft, rate, carriers, rng)
    got = _assert_same(psd, rate, dc_guard_hz=500.0)
    assert len(got) == len(carriers)
    assert got[0]["lo_hz"] == -half and got[0]["flags"] == 2
    assert got[-1]["hi_hz"] == half - rate / nfft and got[-1]["flags"] == 2
    assert [c["flags"] for c in got[1:-1]] == [0, 1, 0, 0] and abs(got[2]["center_hz"]) < rate / nfft
    _assert_same(psd, rate, floor_window_hz=rate * 2)                 # W clamped to nfft
    _assert_same(psd, rate, floor_window_hz=1.0)                      # W clamped to 3


def test_find_carriers_cap_reports_the_total():
    import jaero_b200
    rng = np.random.default_rng(8)
    nfft, rate = 4096, 2.4e6
    psd = _synthetic_psd(nfft, rate, [(-300e3, OQ10500, 30.0), (0.0, OQ10500, 30.0), (300e3, OQ10500, 30.0)], rng)
    L = jaero_b200.lib()
    arr = (jaero_b200.Carrier * 1)()
    n = ctypes.c_int()
    assert L.jaero_scan_find_carriers(psd.ctypes.data_as(ctypes.c_void_p), nfft, rate, None, ctypes.cast(arr, ctypes.c_void_p), 1,
                                      ctypes.byref(n)) == 0
    assert n.value == 3 and abs(arr[0].center_hz + 300e3) < 2 * rate / nfft
    assert [c["center_hz"] for c in _lib_find(psd, rate)] == sorted(c["center_hz"] for c in _lib_find(psd, rate))


def test_find_carriers_floor_budget():
    """2^16 bins with a 100 kHz window at 2.4 MS/s: the sliding order statistic keeps the whole search well inside 50 ms"""
    import jaero_b200
    rng = np.random.default_rng(9)
    psd = rng.exponential(1.0, size=65536)
    L, n = jaero_b200.lib(), ctypes.c_int()
    call = lambda: L.jaero_scan_find_carriers(psd.ctypes.data_as(ctypes.c_void_p), 65536, 2.4e6, None, None, 0, ctypes.byref(n))
    assert call() == 0
    t = time.perf_counter()
    for _ in range(5):
        call()
    dt = (time.perf_counter() - t) / 5
    print("find_carriers, 2^16 bins, 100 kHz floor window: %.1f ms" % (1e3 * dt))
    assert dt < 0.05


def test_mode_hints_from_nominal_widths():
    rng = np.random.default_rng(10)
    nfft, rate = 65536, 2.4e6
    carriers = [(-500e3, OQ10500, 50.0), (-200e3, OQ8400, 50.0), (100e3, MSK1200, 50.0), (400e3, MSK600, 50.0), (600e3, ("rc", 1500.0, 0.5), 50.0)]
    psd = _synthetic_psd(nfft, rate, carriers, rng, frames=10000)
    got = _assert_same(psd, rate)
    assert [c["mode"] for c in got] == ["oqpsk10500", "oqpsk8400", "msk1200", "msk600", "unknown"]


# ---------------------------------------------------------------- rejections and the boundary
def test_find_carriers_rejections():
    import jaero_b200
    psd = np.ones(4096)
    for nfft in (512, 3000, 131072):
        with pytest.raises(jaero_b200.JaeroError, match="nfft"):
            jaero_b200.find_carriers(np.ones(nfft), 2.4e6)
    for rate in (0.0, -1.0, float("nan")):
        with pytest.raises(jaero_b200.JaeroError, match="input_rate"):
            jaero_b200.find_carriers(psd, rate)
    for bad in (dict(threshold_db=0.0), dict(threshold_db=float("inf")), dict(floor_window_hz=0.0), dict(floor_quantile=-0.1),
                dict(floor_quantile=1.5), dict(min_width_hz=-1.0), dict(dc_guard_hz=float("nan"))):
        with pytest.raises(jaero_b200.JaeroError, match="parameter"):
            jaero_b200.find_carriers(psd, 2.4e6, **bad)
    for v in (-1.0, float("nan"), float("inf")):
        p = psd.copy(); p[17] = v
        with pytest.raises(jaero_b200.JaeroError, match="finite"):
            jaero_b200.find_carriers(p, 2.4e6)


def test_scan_create_rejections():
    import jaero_b200
    for nfft, hop, rate in ((512, 256, 2.4e6), (1000, 500, 2.4e6), (1 << 17, 1024, 2.4e6), (1024, 0, 2.4e6), (1024, 1025, 2.4e6),
                            (1024, 512, 0.0), (1024, 512, float("nan"))):
        with pytest.raises(jaero_b200.JaeroError) as ei:
            jaero_b200.Scanner(rate, nfft, hop)
        assert "error -1" in str(ei.value)                          # JAERO_E_ARG, checked before any device is looked for


def test_scan_write_rejects_bad_iq():
    import jaero_b200
    s = jaero_b200.Scanner.__new__(jaero_b200.Scanner)                # argument checks of the Python layer need no handle
    for iq, fmt in ((np.zeros(8, dtype=np.int16), "cu8"), (np.zeros(8, dtype=np.uint8), "cs16"), (np.zeros(7, dtype=np.uint8), "cu8"),
                    (np.zeros(8, dtype=np.uint8), "cf32")):
        with pytest.raises(ValueError):
            s.write(iq, fmt)
    with pytest.raises(ValueError):
        s.write_device(0, 4, 2)
    L = jaero_b200.lib()
    buf = np.zeros(8, dtype=np.uint8)
    assert L.jaero_scan_write(None, buf.ctypes.data_as(ctypes.c_void_p), 4, 0) == -1
    assert L.jaero_scan_write_device(None, buf.ctypes.data_as(ctypes.c_void_p), 4, 0) == -1


@pytest.mark.skipif(has_cuda(), reason="only meaningful on a box without a GPU")
def test_scan_create_fails_without_a_gpu():
    import jaero_b200
    L = jaero_b200.lib()
    h = ctypes.c_void_p()
    assert L.jaero_scan_create(2.4e6, 65536, 16384, 0, ctypes.byref(h)) == -2    # JAERO_E_CUDA: there is no CPU fallback
    with pytest.raises(jaero_b200.JaeroError):
        jaero_b200.Scanner(2.4e6, 65536)


def test_scan_structs_match_header_layout(tmp_path):
    """sizeof / offsetof of jaero_scan_params and jaero_carrier as gcc sees include/jaero_b200.h == the ctypes mirrors"""
    import jaero_b200
    fields = ["center_hz", "peak_hz", "lo_hz", "hi_hz", "width_hz", "power", "snr_db", "peak_db", "floor", "mode", "flags"]
    pf = ["threshold_db", "floor_window_hz", "floor_quantile", "min_width_hz", "dc_guard_hz"]
    body = "".join('printf("%%zu ", offsetof(jaero_carrier, %s));' % f for f in fields)
    body += "".join('printf("%%zu ", offsetof(jaero_scan_params, %s));' % f for f in pf)
    src = tmp_path / "scan_layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "jaero_b200.h"\nint main(void){printf("%zu %zu ",'
                   'sizeof(jaero_carrier), sizeof(jaero_scan_params));' + body + 'printf("\\n");return 0;}\n')
    exe = str(tmp_path / "scan_layout")
    subprocess.run(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe], check=True)
    got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    C, P = jaero_b200.Carrier, jaero_b200.ScanParams
    assert got == [ctypes.sizeof(C), ctypes.sizeof(P)] + [getattr(C, f).offset for f in fields] + [getattr(P, f).offset for f in pf]


def test_channel_plan_groups_by_mode():
    import jaero_b200
    mk = lambda c, mode, power, flags=0: dict(center_hz=c, mode=mode, power=power, flags=flags)
    cs = [mk(300e3, "oqpsk10500", 1e-4), mk(-100e3, "oqpsk10500", 1e-2), mk(50e3, "msk1200", 4e-5), mk(0.0, "oqpsk10500", 1.0, 1),
          mk(70e3, "unknown", 1.0), mk(1.199e6, "oqpsk10500", 1.0)]
    plans, unplanned = jaero_b200.channel_plan(cs, 2.4e6, 50)
    assert sorted(plans) == ["msk1200", "oqpsk10500"]
    oq = plans["oqpsk10500"]
    assert oq["ddc"]["offsets_hz"] == [-100e3, 300e3]
    assert abs(oq["ddc"]["gain"] - 0.2 * np.sqrt(2) / 0.1) < 1e-12
    assert (oq["ddc"]["audio_hz"], oq["ddc"]["bandwidth"], oq["ddc"]["transition"]) == (8000.0, 12000.0, 4000.0)
    assert oq["demod"] == dict(kind="oqpsk", n_channels=2, fb=10500, freq_center=8000.0, lockingbw=10500.0)
    assert plans["msk1200"]["demod"]["lockingbw"] == 1800.0 and plans["msk1200"]["ddc"]["bandwidth"] == 3000.0
    assert sorted(c["center_hz"] for c in unplanned) == [0.0, 70e3, 1.199e6]
