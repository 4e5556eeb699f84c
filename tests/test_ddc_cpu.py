"""CPU checks of the wideband IQ down-converter: the filter stages jaero_ddc_plan designs meet the specification in
include/jaero_b200.h (composite passband within +-0.1 dB, >= 70 dB everywhere from bandwidth/2 + transition to input_rate/2,
aliases of both decimations included), the folded-tap reference equals the contract formula, and the planner rejects what it
must. jaero_ddc_plan is host code: none of this needs a GPU."""
import numpy as np
import pytest

import ddc_reference as ref

# (decimation, bandwidth, transition): the three decimations for 48 kHz audio from 2.4, 3.072 and 9.6 MS/s, a 96 kHz input (one
# stage), and the passbands of the 10.5 kbps OQPSK, 1200 bps and 600 bps MSK channels
RATES = [2, 50, 64, 200]
BANDS = [(12000.0, 4000.0), (3000.0, 1000.0), (1500.0, 500.0)]


def _plan(fs, D, B, dT):
    import jaero_b200
    return jaero_b200.ddc_plan(fs, D, B, dT)


def _probe_tones(fs, D1, D, B, dT):
    """passband sweep, both transition edges, and every frequency up to fs/2 that either decimation folds onto the passband"""
    edge = B / 2 + dT
    pas = np.linspace(-B / 2, B / 2, 41)
    stop = [-edge, edge, fs / 2, -fs / 2 + 1.0]
    for step in sorted({fs / D1, fs / D}):
        k = np.arange(1, int(fs / 2 // step) + 1)
        for fp in (-B / 2, 0.0, B / 2):
            for f in np.concatenate([k * step + fp, -k * step + fp]):
                if edge <= abs(f) <= fs / 2:
                    stop.append(f)
    return pas, np.array(stop)


@pytest.mark.parametrize("D", RATES)
@pytest.mark.parametrize("band", BANDS)
def test_plan_meets_the_filter_specification(D, band):
    B, dT = band
    fs = 48000.0 * D
    p = _plan(fs, D, B, dT)
    assert p["D1"] * p["D2"] == D and len(p["h1"]) == p["K1"] and len(p["h2"]) == p["K2"]
    pas, stop = _probe_tones(fs, p["D1"], D, B, dT)
    # run the reference chain on complex tones: a channel tuned to -f sees the constant input x = 1 as a tone at +f
    tones = np.concatenate([[0.0], pas, stop])
    T = [ref.tuning_word(-f, fs) for f in tones]
    f_q = -np.array([(t if t < 2 ** 31 else t - 2 ** 32) for t in T], dtype=np.float64) / 2 ** 32 * fs   # quantised tone frequency
    N = p["K1"] + p["D1"] * p["K2"] + 2 * D
    _, _, _, v = ref.ddc_reference(np.ones(N, dtype=np.complex128), p["h1"], p["D1"], p["h2"], p["D2"], T, [0] * len(T))
    g = np.abs(v[:, -1])                                          # steady state: the last output's window lies inside the input
    g0 = g[0]
    db = 20 * np.log10(np.maximum(g / g0, 1e-30))
    npas = len(pas)
    assert np.all(np.abs(db[1:1 + npas]) <= 0.1), db[1:1 + npas]
    assert np.all(db[1 + npas:] <= -70.0), (f_q[1 + npas:][db[1 + npas:] > -70], db[1 + npas:].max())
    # and densely, from the closed-form response of the same taps
    grid = np.concatenate([np.linspace(-B / 2, B / 2, 401), np.linspace(B / 2 + dT, fs / 2, 20001), -np.linspace(B / 2 + dT, fs / 2, 20001)])
    H = np.abs(ref.composite_response(p["h1"], p["D1"], p["h2"], fs, grid))
    Hdb = 20 * np.log10(H / abs(ref.composite_response(p["h1"], p["D1"], p["h2"], fs, [0.0])[0]))
    assert np.abs(Hdb[:401]).max() <= 0.1
    assert Hdb[401:].max() <= -70.0
    # the chain and the closed form agree on the probed tones
    Hq = np.abs(ref.composite_response(p["h1"], p["D1"], p["h2"], fs, f_q))
    np.testing.assert_allclose(g / g0, Hq / Hq[0], atol=1e-9)


def test_planner_prefers_two_stages_for_a_large_decimation():
    """9.6 MS/s to 48 kHz: a single 4 kHz-transition stage would need thousands of taps"""
    p = _plan(9.6e6, 200, 12000.0, 4000.0)
    assert p["D2"] > 1 and p["K1"] < 400 and p["K2"] < 400
    flop = 8 * p["D2"] * p["K1"] + 4 * p["K2"]
    assert flop < 12000


def test_folded_taps_equal_the_direct_formula():
    """mix-then-filter as the contract writes it == folded complex taps with one rotation per stage-1 output"""
    rng = np.random.default_rng(5)
    fs, D = 48000.0 * 50, 50
    p = _plan(fs, D, 12000.0, 4000.0)
    x = rng.standard_normal(6000) + 1j * rng.standard_normal(6000)
    T = [ref.tuning_word(f, fs) for f in (0.0, 123456.7, -1.19e6, 1.1e6 + 0.01)]
    S = [ref.tuning_word(f, fs / D) for f in (8000.0, 6000.5, 2000.0, 17000.0)]
    val, _, _, v = ref.ddc_reference(x, p["h1"], p["D1"], p["h2"], p["D2"], T, S, gain=0.5)
    val_d, v_d = ref.ddc_direct(x, p["h1"], p["D1"], p["h2"], p["D2"], T, S, gain=0.5)
    assert v.shape == v_d.shape == (4, (6000 - 1) // D + 1)
    assert np.abs(v - v_d).max() <= 1e-12 * max(1.0, np.abs(v_d).max())
    np.testing.assert_array_equal(val, np.clip(np.rint(val_d), -32768, 32767).astype(np.int16))


def test_reference_retune_schedule_splits_at_the_sample_the_rule_names():
    """a schedule with one entry is the fixed-word chain; a retune changes only stage-1 samples from j D1 >= the retune input on"""
    rng = np.random.default_rng(9)
    fs, D = 48000.0 * 50, 50
    p = _plan(fs, D, 12000.0, 4000.0)
    x = rng.standard_normal(20000) + 1j * rng.standard_normal(20000)
    T0, T1, S0 = [ref.tuning_word(1e5, fs)], [ref.tuning_word(-2e5, fs)], [ref.tuning_word(8000.0, fs / D)]
    a, *_ = ref.ddc_reference(x, p["h1"], p["D1"], p["h2"], p["D2"], T0, S0)
    b, *_ = ref.ddc_reference(x, p["h1"], p["D1"], p["h2"], p["D2"], [(0, T0), (2500, T1)], [(0, S0)])
    np.testing.assert_array_equal(a[:, :2500 // D], b[:, :2500 // D])
    assert not np.array_equal(a[:, 2500 // D + p["K2"] // p["D2"]:], b[:, 2500 // D + p["K2"] // p["D2"]:])


def test_tuning_word_rounds_as_the_library_does():
    assert ref.tuning_word(0.0, 1.0) == 0
    assert ref.tuning_word(-0.25, 1.0) == 3 * 2 ** 30
    assert ref.tuning_word(0.5, 1.0) == 2 ** 31
    assert ref.tuning_word(-0.5, 1.0) == 2 ** 31


@pytest.mark.parametrize("args,match", [
    ((0.0, 50, 12000.0, 4000.0), "positive"),
    ((2.4e6, 0, 12000.0, 4000.0), "positive"),
    ((2.4e6, 50, -1.0, 4000.0), "positive"),
    ((2.4e6, 50, 12000.0, 0.0), "positive"),
    ((2.4e6, 50, 44000.0, 4000.0), "half the output rate"),
    ((4.8e6, 100, 12000.0, 4000.0), None),
])
def test_plan_rejections(args, match):
    import jaero_b200
    if match is None:
        assert jaero_b200.ddc_plan(*args)["D1"] > 1
        return
    with pytest.raises(jaero_b200.JaeroError, match=match):
        jaero_b200.ddc_plan(*args)


def test_small_decimation_plans_a_single_stage():
    p = _plan(96000.0, 2, 12000.0, 4000.0)
    assert (p["D1"], p["D2"], p["K2"]) == (2, 1, 1) and list(p["h2"]) == [1.0]


@pytest.mark.parametrize("offset,audio,match", [
    (1.2e6 - 5999.0, 8000.0, "offset"),                  # |offset| > input_rate/2 - bandwidth/2
    (-1.2e6, 8000.0, "offset"),
    (float("nan"), 8000.0, "offset"),
    (0.0, 6000.0, "audio passband"),                     # passband touches 0 Hz
    (0.0, 18000.0, "audio passband"),                    # passband touches Fs_out/2
    (0.0, -8000.0, "audio passband"),
])
def test_create_rejects_channels_outside_the_bands(offset, audio, match):
    """checked before any device is touched, so this holds with or without a GPU"""
    import jaero_b200
    with pytest.raises(jaero_b200.JaeroError, match=match):
        jaero_b200.Ddc(2.4e6, 50, [0.0, offset], [8000.0, audio], 12000.0, 4000.0)


def test_ddc_write_rejects_mismatched_iq_before_the_library():
    import jaero_b200
    with pytest.raises(ValueError):
        jaero_b200.Ddc._iq(np.zeros(8, dtype=np.int16), "cu8")
    with pytest.raises(ValueError):
        jaero_b200.Ddc._iq(np.zeros(7, dtype=np.uint8), "cu8")
    with pytest.raises(ValueError):
        jaero_b200.Ddc._iq(np.zeros(8, dtype=np.float32), "cf32")
