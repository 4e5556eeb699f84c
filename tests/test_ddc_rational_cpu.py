"""CPU checks of the rational-rate down-converter (include/jaero_b200.h, jaero_ddc_plan_rational / jaero_ddc_create_rational):
the stages the planner designs for the usual software-radio rates meet the filter specification (passband within +-0.1 dB,
>= 70 dB from bandwidth/2 + transition to input_rate/2, aliases of both decimations and images of the x L zero-stuffing
included), the polyphase reference equals the contract formula, L = 1 is exactly the integer down-converter, and the planner
and rate_ratio reject what they must. All of it is host code."""
import ctypes
import inspect

import numpy as np
import pytest

import ddc_reference as ref
import ddc_reference_rational as rref
from conftest import has_cuda

# the usual rates of radios that do not run at a multiple of 48 kHz: RTL-SDR 2.048, Airspy 2.5 / 10, Airspy Mini 3, HackRF 8 MS/s
RATES = [2.048e6, 2.5e6, 3e6, 8e6, 10e6]
BANDS = [(12000.0, 4000.0), (3000.0, 1000.0), (1500.0, 500.0)]


def _plan(fs, B, dT):
    import jaero_b200
    L, M = jaero_b200.rate_ratio(fs)
    return jaero_b200.ddc_plan(fs, M, B, dT, interpolation=L), L, M


def _probe_tones(fs, M, B, dT):
    """passband sweep, both transition edges, and every frequency up to fs/2 that lands on the passband: the stage-1 aliases
    (period fs/D1), the output aliases (period fs L / M) and the images of the zero-stuffing all lie on the lattice of step fs/M"""
    edge = B / 2 + dT
    pas = np.linspace(-B / 2, B / 2, 41)
    stop = [-edge, edge, fs / 2, -fs / 2 + 1.0]
    step = fs / M
    k = np.arange(1, int(fs / 2 // step) + 1)
    for fp in (-B / 2, 0.0, B / 2):
        for f in np.concatenate([k * step + fp, -k * step + fp]):
            if edge <= abs(f) <= fs / 2:
                stop.append(f)
    return pas, np.array(stop)


def _dense_response(p, L, fs):
    """(f, main-term gain |H1(f) H2(f)| / L, bound on the gain at any output phase sum_k |H1(f)| |H2(f + k fs/D1)| / L) on a
    grid of spacing fs / (D1 2^15) over [-fs/2, fs/2), from zero-padded FFTs of the taps: H1 has period fs, H2 period L fs/D1"""
    D1 = p["D1"]
    nf1 = D1 << 15
    nf2 = L << 15                                                  # H2's period in grid steps
    H1 = np.abs(np.fft.fft(p["h1"], nf1))
    H2 = np.abs(np.fft.fft(p["h2"], nf2))
    i = np.arange(-nf1 // 2, nf1 // 2)
    f = i * fs / nf1
    h1 = H1[i % nf1]
    main = h1 * H2[i % nf2] / L
    bound = np.zeros(len(i))
    for k in range(L):
        bound += H2[(i + k * (1 << 15)) % nf2]
    return f, main, h1 * bound / L


@pytest.mark.parametrize("fs", RATES)
@pytest.mark.parametrize("band", BANDS)
def test_rational_plan_meets_the_filter_specification(fs, band):
    B, dT = band
    p, L, M = _plan(fs, B, dT)
    assert p["L"] == L and p["D1"] * p["D2"] == M and len(p["h1"]) == p["K1"] and len(p["h2"]) == p["K2"]
    assert abs(p["h2"].sum() - L) < 1e-12 * L and abs(p["h1"].sum() - 1.0) < 1e-12
    pas, stop = _probe_tones(fs, M, B, dT)
    # run the reference chain on complex tones: a channel tuned to -f sees the constant input x = 1 as a tone at +f
    tones = np.concatenate([[0.0], pas, stop])
    T = [ref.tuning_word(-f, fs) for f in tones]
    f_q = -np.array([(t if t < 2 ** 31 else t - 2 ** 32) for t in T], dtype=np.float64) / 2 ** 32 * fs
    R = -(-p["K2"] // L)
    N = p["K1"] + p["D1"] * (R + 2) + 2 * M
    _, _, _, v = rref.ddc_reference_rational(np.ones(N, dtype=np.complex128), p["h1"], p["D1"], p["h2"], L, p["D2"], T, [0] * len(T))
    g = np.abs(v[:, -1])                                          # steady state: the last output's window lies inside the input
    g0 = g[0]
    db = 20 * np.log10(np.maximum(g / g0, 1e-30))
    npas = len(pas)
    assert np.all(np.abs(db[1:1 + npas]) <= 0.1), db[1:1 + npas]
    assert np.all(db[1 + npas:] <= -70.0), (f_q[1 + npas:][db[1 + npas:] > -70], db[1 + npas:].max())
    # the chain and the closed form (images included, at the last output's phase) agree on the probed tones
    m = v.shape[1] - 1
    phase = (m * p["D2"]) % L
    tr = rref.tone_response_rational(p["h1"], p["D1"], p["h2"], L, fs, f_q, phase)
    np.testing.assert_allclose(g / g0, tr / tr[0], atol=1e-9)
    # and densely, from the closed form: the passband ripple of the main term, and a bound over every output phase elsewhere
    f, main, bound = _dense_response(p, L, fs)
    norm = main[np.argmin(np.abs(f))]
    inband = np.abs(f) <= B / 2
    assert np.abs(20 * np.log10(main[inband] / norm)).max() <= 0.1
    out = np.abs(f) >= B / 2 + dT
    assert 20 * np.log10(bound[out].max() / norm) <= -70.0


@pytest.mark.parametrize("fs", [2.5e6, 10e6, 2.048e6])
def test_direct_equals_polyphase(fs):
    """zero-stuff, convolve and decimate as the contract writes it == the polyphase sum over the stage-1 rows"""
    import jaero_b200
    L, M = jaero_b200.rate_ratio(fs)
    p = jaero_b200.ddc_plan(fs, M, 12000.0, 4000.0, interpolation=L)
    rng = np.random.default_rng(6)
    n = 12_007
    x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    T = [ref.tuning_word(f, fs) for f in (0.0, 123456.7, -fs / 2 + 6000.0, 0.41 * fs)]
    S = [ref.tuning_word(f, 48000.0) for f in (8000.0, 6000.5, 12000.0, 17000.0)]
    _, val, _, v = rref.ddc_reference_rational(x, p["h1"], p["D1"], p["h2"], L, p["D2"], T, S, gain=0.5)
    val_d, v_d = rref.ddc_direct_rational(x, p["h1"], p["D1"], p["h2"], L, p["D2"], T, S, gain=0.5)
    assert v.shape == v_d.shape == (4, -(-n * L // M))
    assert np.abs(v - v_d).max() <= 1e-12 * max(1.0, np.abs(v_d).max())
    assert np.abs(val - val_d).max() <= 1e-12 * 32768 * max(1.0, np.abs(v_d).max())


def test_rational_reference_with_l1_is_the_integer_reference():
    import jaero_b200
    rng = np.random.default_rng(8)
    fs, D = 2.4e6, 50
    p = jaero_b200.ddc_plan(fs, D, 12000.0, 4000.0)
    x = rng.standard_normal(20_000) + 1j * rng.standard_normal(20_000)
    T0, T1 = [ref.tuning_word(f, fs) for f in (1e5, -3e5)], [ref.tuning_word(f, fs) for f in (-2e5, 7e5)]
    S0, S1 = [ref.tuning_word(f, fs / D) for f in (8000.0, 9000.0)], [ref.tuning_word(f, fs / D) for f in (16000.0, 7000.0)]
    Tsch, Ssch = [(0, T0), (2501, T1)], [(0, S0), (7000, S1)]
    a = ref.ddc_reference(x, p["h1"], p["D1"], p["h2"], p["D2"], Tsch, Ssch, gain=3.0)
    b = rref.ddc_reference_rational(x, p["h1"], p["D1"], p["h2"], 1, p["D2"], Tsch, Ssch, gain=3.0)
    for u, w in zip(a, b):
        np.testing.assert_array_equal(u, w)


@pytest.mark.parametrize("D", [2, 50, 64, 200])
@pytest.mark.parametrize("band", BANDS)
def test_plan_rational_with_l1_equals_plan_bit_for_bit(D, band):
    import jaero_b200
    lib = jaero_b200.lib()
    fs = 48000.0 * D
    a, b = np.zeros(4, dtype=np.int32), np.zeros(5, dtype=np.int32)
    assert lib.jaero_ddc_plan(fs, D, band[0], band[1], a.ctypes.data, None, None) == 0
    assert lib.jaero_ddc_plan_rational(fs, 1, D, band[0], band[1], b.ctypes.data, None, None) == 0
    assert b[0] == 1 and list(a) == list(b[1:])
    h1a, h2a, h1b, h2b = np.zeros(a[1]), np.zeros(a[3]), np.zeros(a[1]), np.zeros(a[3])
    assert lib.jaero_ddc_plan(fs, D, band[0], band[1], a.ctypes.data, h1a.ctypes.data, h2a.ctypes.data) == 0
    assert lib.jaero_ddc_plan_rational(fs, 1, D, band[0], band[1], b.ctypes.data, h1b.ctypes.data, h2b.ctypes.data) == 0
    assert h1a.tobytes() == h1b.tobytes() and h2a.tobytes() == h2b.tobytes()


@pytest.mark.parametrize("L,M", [(1, 50), (3, 625), (12, 625), (3, 128), (2, 125), (7, 3)])
def test_output_count(L, M):
    """output m exists once input floor(m M / L) has arrived: N inputs give ceil(N L / M) outputs"""
    for N in list(range(1, 3 * M + 2)) + [10 ** 6 + 17]:
        m = np.arange(N * L // M + 3)
        assert rref.n_outputs_rational(N, L, M) == int(np.count_nonzero(m * M // L <= N - 1))
        if L == 1:
            assert rref.n_outputs_rational(N, L, M) == (N - 1) // M + 1


@pytest.mark.parametrize("fs,ratio", [(10e6, (3, 625)), (2.5e6, (12, 625)), (3e6, (2, 125)), (2e6, (3, 125)), (8e6, (3, 500)),
                                      (20e6, (3, 1250)), (2.048e6, (3, 128)), (2.4e6, (1, 50)), (3.072e6, (1, 64)), (6e6, (1, 125)),
                                      (9.6e6, (1, 200))])
def test_rate_ratio(fs, ratio):
    import jaero_b200
    assert jaero_b200.rate_ratio(fs) == ratio
    assert jaero_b200.rate_ratio(int(fs), 48000) == ratio


@pytest.mark.parametrize("fs", [2.4e6 + 0.5, float("nan"), -2.4e6, 1_000_001.0, 0.0])
def test_rate_ratio_rejections(fs):
    import jaero_b200
    with pytest.raises(ValueError):
        jaero_b200.rate_ratio(fs)


@pytest.mark.parametrize("args,match", [
    ((10e6, 0, 625, 12000.0, 4000.0), "interpolation must be 1 to 256"),
    ((10e6, 257, 625, 12000.0, 4000.0), "interpolation must be 1 to 256"),
    ((10e6, 3, 600, 12000.0, 4000.0), "reduce the ratio"),
    ((10e6, 6, 1250, 12000.0, 4000.0), "reduce the ratio"),
    ((10e6, 3, 625, 44000.0, 4000.0), "half the output rate"),
    ((10e6, 3, 625, 12000.0, 1.0), "no two-stage split"),
    ((0.0, 3, 625, 12000.0, 4000.0), "positive"),
])
def test_rational_plan_rejections(args, match):
    import jaero_b200
    fs, L, M, B, dT = args
    with pytest.raises(jaero_b200.JaeroError, match=match):
        jaero_b200.ddc_plan(fs, M, B, dT, interpolation=L)
    st = np.zeros(5, dtype=np.int32)
    assert jaero_b200.lib().jaero_ddc_plan_rational(fs, L, M, B, dT, st.ctypes.data, None, None) == -1
    assert "jaero_ddc_plan_rational" in jaero_b200.lib().jaero_last_error().decode()


def test_rational_create_rejects_channels_outside_the_bands():
    """checked before any device is touched: the audio band is judged against the rational output rate"""
    import jaero_b200
    with pytest.raises(jaero_b200.JaeroError, match="audio passband"):
        jaero_b200.Ddc(10e6, 625, [0.0], [18000.5], 12000.0, 4000.0, interpolation=3)
    with pytest.raises(jaero_b200.JaeroError, match="offset"):
        jaero_b200.Ddc(10e6, 625, [5e6 - 5999.0], [8000.0], 12000.0, 4000.0, interpolation=3)
    with pytest.raises(jaero_b200.JaeroError, match="reduce the ratio"):
        jaero_b200.Ddc(10e6, 1250, [0.0], [8000.0], 12000.0, 4000.0, interpolation=6)


def test_channel_plan_with_interpolation():
    import jaero_b200
    mk = lambda c, mode, power, flags=0: dict(center_hz=c, mode=mode, power=power, flags=flags)
    cs = [mk(300e3, "oqpsk10500", 1e-4), mk(-100e3, "oqpsk10500", 1e-2), mk(50e3, "msk1200", 4e-5), mk(1.249e6, "oqpsk10500", 1.0)]
    fs = 2.5e6
    L, M = jaero_b200.rate_ratio(fs)
    plans, unplanned = jaero_b200.channel_plan(cs, fs, M, interpolation=L)
    assert sorted(plans) == ["msk1200", "oqpsk10500"]
    assert [c["center_hz"] for c in unplanned] == [1.249e6]
    sig = inspect.signature(jaero_b200.Ddc)
    for plan in plans.values():
        dd = plan["ddc"]
        assert (dd["input_rate"], dd["decimation"], dd["interpolation"]) == (fs, 625, 12)
        sig.bind(**dd)                                            # Ddc(**plan["ddc"]) is a complete call
        assert jaero_b200.ddc_plan(fs, dd["decimation"], dd["bandwidth"], dd["transition"], dd["interpolation"])["L"] == 12
    # the integer call keeps interpolation 1
    plans, _ = jaero_b200.channel_plan(cs, 2.4e6, 50)
    assert plans["oqpsk10500"]["ddc"]["interpolation"] == 1


@pytest.mark.skipif(has_cuda(), reason="only meaningful on a box without a GPU")
def test_create_rational_fails_without_a_gpu():
    import jaero_b200
    lib = jaero_b200.lib()
    h = ctypes.c_void_p()
    off, aud = np.zeros(2), np.full(2, 8000.0)
    assert lib.jaero_ddc_create_rational(10e6, 3, 625, 2, off.ctypes.data, aud.ctypes.data, 12000.0, 4000.0, 1.0, 0, ctypes.byref(h)) == -2
    with pytest.raises(jaero_b200.JaeroError):
        jaero_b200.Ddc(10e6, 625, off, aud, 12000.0, 4000.0, interpolation=3)
