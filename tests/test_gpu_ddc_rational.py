"""GPU checks of the rational-rate down-converter (jaero_b200.Ddc with interpolation > 1, include/jaero_b200.h
jaero_ddc_create_rational): every PCM sample against the float64 polyphase reference (tests/ddc_reference_rational.py) at 2.5 MS/s
(L/M = 12/625) and 10 MS/s (3/625), independence of how the stream is cut into writes, the retune rule, L = 1 against the integer
entry point, and a scanner-planned SDR stream at 2.5 MS/s through Ddc -> DemodBatch -> PChannelBatch on one CUDA stream."""
import ctypes

import numpy as np
import pytest

import ddc_reference as ref
import ddc_reference_rational as rref
from test_gpu_ddc import _assert_matches, _random_iq

pytestmark = pytest.mark.gpu

B, DT = 12000.0, 4000.0
RATES = [2.5e6, 10e6]


def _setup(fs):
    import jaero_b200
    L, M = jaero_b200.rate_ratio(fs)
    return L, M, jaero_b200.ddc_plan(fs, M, B, DT, interpolation=L)


def _channels(fs, C, seed):
    rng = np.random.default_rng(seed)
    edge = fs / 2 - B / 2
    off = rng.uniform(-edge, edge, size=C)
    if C > 1:
        off[0], off[1] = -edge, edge                             # both ends of the tunable range
    aud = rng.uniform(B / 2 + 1.0, 24000.0 - B / 2 - 1.0, size=C)
    return off, aud


def _ddc(fs, off, aud, gain):
    import jaero_b200
    L, M = jaero_b200.rate_ratio(fs)
    return jaero_b200.Ddc(fs, M, off, aud, B, DT, gain=gain, interpolation=L)


def _reference(fs, x, gain, T, S):
    L, M, p = _setup(fs)
    return rref.ddc_reference_rational(x, p["h1"], p["D1"], p["h2"], L, p["D2"], T, S, gain=gain)


def _words(fs, off, aud):
    L, M, _ = _setup(fs)
    return [ref.tuning_word(o, fs) for o in off], [ref.tuning_word(a, fs * L / M) for a in aud]


@pytest.mark.parametrize("fs", RATES)
@pytest.mark.parametrize("fmt", ["cu8", "cs16"])
@pytest.mark.parametrize("C,gain", [(1, 1.0), (33, 1.0), (300, 1.0), (33, 300.0)])
def test_rational_ddc_equals_reference(fs, fmt, C, gain):
    L, M, _ = _setup(fs)
    n = 150_001
    iq = _random_iq(fmt, n, seed=C + (7 if fmt == "cu8" else 0) + int(fs) % 97)
    off, aud = _channels(fs, C, seed=C)
    d = _ddc(fs, off, aud, gain)
    assert d.output_rate == fs * L / M
    d.write(iq[:2 * 70_001], fmt)
    a = d.read_pcm()
    d.write(iq[2 * 70_001:], fmt)
    got = np.concatenate([a, d.read_pcm()], axis=1)
    inputs, clipped = d.stats()
    d.close()
    T, S = _words(fs, off, aud)
    _, val, clip_ref, _ = _reference(fs, ref.iq_to_complex(iq, fmt), gain, T, S)
    assert inputs == n and got.shape == (C, -(-n * L // M)) and a.shape[1] == -(-70_001 * L // M)
    _assert_matches(got, val)
    np.testing.assert_array_equal(clipped, clip_ref)
    if gain > 1:
        assert clip_ref.min() > 0                                # the high-gain case does clip, on every channel


@pytest.mark.parametrize("fs", RATES)
def test_rational_output_does_not_depend_on_how_the_stream_is_cut(fs):
    import torch
    L, M, p = _setup(fs)
    fmt, n = "cs16", 400_009
    iq = _random_iq(fmt, n, seed=3)
    off, aud = _channels(fs, 40, seed=4)
    d = _ddc(fs, off, aud, 4.0)
    d.write(iq, fmt)
    whole = d.read_pcm()
    d.close()
    assert whole.shape[1] == -(-n * L // M)
    rng = np.random.default_rng(11)
    D1 = p["D1"]
    pieces = [1, L, M - 1, M, M + 1, D1 - 1, D1 + 1, 7, 101, 997, 2, 3, 65_537, 50_021]
    cuts = []
    while sum(cuts) < n:
        cuts.append(min(int(pieces[len(cuts)] if len(cuts) < len(pieces) else rng.choice(pieces)), n - sum(cuts)))
    dev = torch.from_numpy(iq).cuda()
    torch.cuda.synchronize()
    for path in ("host", "device"):
        d = _ddc(fs, off, aud, 4.0)
        parts, a = [], 0
        for c in cuts:
            if path == "host":
                d.write(iq[2 * a:2 * (a + c)], fmt)
            else:
                d.write_device(dev.data_ptr() + 4 * a, c, fmt)
            part = d.read_pcm()
            assert part.shape[1] == -(-(a + c) * L // M) - (-(-a * L // M))
            parts.append(part)
            a += c
        d.close()
        got = np.concatenate(parts, axis=1)
        assert got.shape == whole.shape
        assert np.array_equal(got, whole), path


@pytest.mark.parametrize("fs", RATES)
def test_rational_retune_follows_the_rule(fs):
    """set_offset between writes applies to stage-1 samples whose input j*D1 arrives later; set_audio_freq to outputs m whose
    input floor(m M / L) arrives later"""
    fmt = "cu8"
    iq = _random_iq(fmt, 300_000, seed=21)
    off, aud = _channels(fs, 9, seed=22)
    d = _ddc(fs, off, aud, 8.0)
    a, b = 60_013, 190_001
    d.write(iq[:2 * a], fmt); p0 = d.read_pcm()
    off2 = off.copy(); off2[3] = 123_456.78; off2[5] = -1_000_000.0
    aud2 = aud.copy(); aud2[4] = 15_000.0
    d.set_offset(off2[3], channel=3); d.set_offset(off2[5], channel=5); d.set_audio_freq(aud2[4], channel=4)
    d.write(iq[2 * a:2 * b], fmt); p1 = d.read_pcm()
    aud3 = np.full(9, 17_000.0)
    d.set_audio_freq(17_000.0)
    off3 = np.full(9, -250_000.0)
    d.set_offset(-250_000.0)
    d.write(iq[2 * b:], fmt); p2 = d.read_pcm()
    d.close()
    T1, S1 = _words(fs, off, aud)
    T2, S2 = _words(fs, off2, aud2)
    T3, S3 = _words(fs, off3, aud3)
    _, val, _, _ = _reference(fs, ref.iq_to_complex(iq, fmt), 8.0, [(0, T1), (a, T2), (b, T3)], [(0, S1), (a, S2), (b, S3)])
    _assert_matches(np.concatenate([p0, p1, p2], axis=1), val)


def test_interpolation_one_is_the_integer_ddc():
    """Ddc(fs, D), Ddc(fs, D, interpolation=1) and a handle from the integer entry point jaero_ddc_create give the same bytes"""
    import jaero_b200
    fs, D = 2.4e6, 50
    iq = _random_iq("cs16", 200_003, seed=51)
    off, aud = _channels(fs, 37, seed=52)
    h = ctypes.c_void_p()
    offc, audc = np.ascontiguousarray(off), np.ascontiguousarray(aud)
    assert jaero_b200.lib().jaero_ddc_create(fs, D, len(off), offc.ctypes.data, audc.ctypes.data, B, DT, 4.0, 0, ctypes.byref(h)) == 0
    legacy = jaero_b200.Ddc.__new__(jaero_b200.Ddc)
    legacy.n, legacy.h = len(off), h
    outs = []
    for d in (jaero_b200.Ddc(fs, D, off, aud, B, DT, gain=4.0), jaero_b200.Ddc(fs, D, off, aud, B, DT, gain=4.0, interpolation=1), legacy):
        parts = []
        for a, c in ((0, 1), (1, 49), (50, 99_999), (100_049, 100_003 - 49)):
            d.write(iq[2 * a:2 * (a + c)], "cs16"); parts.append(d.read_pcm())
        outs.append(np.concatenate(parts, axis=1))
        d.close()
    assert outs[0].shape == (37, (200_003 - 1) // D + 1)
    assert outs[0].tobytes() == outs[1].tobytes() == outs[2].tobytes()


def _run_plan(iq, fmt, dd, dm, stream, chunk):
    """Ddc(**plan) -> DemodBatch.write_device -> PChannelBatch.process_batch on one CUDA stream, no host copy of the PCM"""
    import torch
    import jaero_b200
    dev = torch.from_numpy(iq).cuda()
    torch.cuda.synchronize()
    d = jaero_b200.Ddc(**dd)
    b = jaero_b200.DemodBatch(dm["kind"], dm["n_channels"], fb=dm["fb"], freq_center=dm["freq_center"], lockingbw=dm["lockingbw"])
    pc = jaero_b200.PChannelBatch(dm["n_channels"], dm["fb"])
    d.set_stream(stream.cuda_stream); b.set_stream(stream.cuda_stream)
    bytes_per = 2 if fmt == "cu8" else 4
    n = iq.size // 2
    got = [[] for _ in range(dm["n_channels"])]
    for k, a in enumerate(range(0, n, chunk)):
        d.write_device(dev.data_ptr() + bytes_per * a, min(chunk, n - a), fmt)
        ptr, m, stride = d.output()
        b.write_device(ptr, m, stride)
        pc.process_batch(b)
        if k % 10 == 9:
            for ch, r in enumerate(pc.read_sus()):
                got[ch].append((r[0], r[1]))
    for ch, r in enumerate(pc.read_sus()):
        got[ch].append((r[0], r[1]))
    _, clipped = d.stats()
    assert clipped.sum() == 0
    d.close(); b.close(); pc.close()
    return got


def test_scan_driven_2_5_msps_stream_through_ddc_demod_and_pchannel():
    """The signal set of test_gpu_ddc's end-to-end run at an Airspy's 2.5 MS/s, which no integer decimation reaches: Scanner ->
    find_carriers -> channel_plan(rate_ratio) -> Ddc (L/M = 12/625) -> DemodBatch -> PChannelBatch, all on one CUDA stream.
    Every planned carrier (the 20 dB stronger neighbour too) decodes a contiguous run of its transmitted signal units, judged as
    test_gpu_scan judges it against the same demodulator fed the same envelope as 48 kHz PCM."""
    import torch
    import jaero_b200
    from jaero_b200 import synth
    from test_gpu_ddc import _decoded, _run_direct
    fs = 2.5e6
    oq_off = [-700_123.0, -150_000.0, 260_500.0, 810_000.0]
    msk_off = [-420_000.0, 530_250.0]
    neighbour = oq_off[1] + B / 2 + DT + 5250.0 + 1000.0
    envs, sus, offs, ebn0, fbs = [], [], [], [], []
    for i, f in enumerate(oq_off):
        bits, s = synth.pchannel_bits(10500, 16, seed=300 + i, return_sus=True)
        envs.append(synth.oqpsk_envelope(bits, 10500.0)); sus.append(s); offs.append(f); ebn0.append(11.0); fbs.append(10500.0)
    for i, f in enumerate(msk_off):
        bits, s = synth.pchannel_bits(1200, 8, seed=400 + i, return_sus=True, loop=True, even_parity=True)
        envs.append(synth.msk_envelope(bits, 1200.0)); sus.append(s); offs.append(f); ebn0.append(12.0); fbs.append(1200.0)
    nb, s = synth.pchannel_bits(10500, 16, seed=999, return_sus=True)
    envs.append(synth.oqpsk_envelope(nb, 10500.0)); sus.append(s); offs.append(neighbour); ebn0.append(31.0); fbs.append(10500.0)
    sent = [[bytes(x) for x in s_.reshape(-1, 12)] for s_ in sus]
    oq_idx, msk_idx = [0, 1, 2, 3, 6], [4, 5]
    direct = {}
    pcm = np.stack([synth.to_passband_int16(envs[i], 8000.0, ebn0_db=ebn0[i], fb=10500.0, rng=np.random.default_rng(70 + i)) for i in oq_idx])
    for ch, g in enumerate(_run_direct(pcm, "oqpsk", 10500, 8000.0, 10500)):
        direct[oq_idx[ch]] = _decoded(sent[oq_idx[ch]], g)
    pcm = np.stack([synth.to_passband_int16(envs[i], 2000.0, ebn0_db=12.0, fb=1200.0, rng=np.random.default_rng(80 + i)) for i in msk_idx])
    for ch, g in enumerate(_run_direct(pcm, "msk", 1200, 2000.0, 1800)):
        direct[msk_idx[ch]] = _decoded(sent[msk_idx[ch]], g)
    for i, (dk0, dn, drun) in direct.items():
        assert dk0 >= 0 and drun, "the direct path did not lock on carrier %d" % i
    slowest = {"oqpsk10500": max(direct[i][0] for i in oq_idx[:4]), "msk1200": max(direct[i][0] for i in msk_idx)}
    frame = {"oqpsk10500": 26, "msk1200": 6}

    iq = synth.wideband_iq(envs, offs, fs, ebn0, fmt="cs16", seed=5, fb=fbs)
    stream = torch.cuda.Stream()
    dev = torch.from_numpy(iq).cuda()
    torch.cuda.synchronize()
    chunk = 250_000                                              # 0.1 s of IQ, 4800 PCM samples per channel
    sc = jaero_b200.Scanner(fs, 1 << 16, 1 << 15)
    sc.set_stream(stream.cuda_stream)
    for a in range(0, iq.size // 2, chunk):
        sc.write_device(dev.data_ptr() + 4 * a, min(chunk, iq.size // 2 - a), "cs16")
    mean, _, _ = sc.read()
    sc.close()
    del dev
    L, M = jaero_b200.rate_ratio(fs)
    assert (L, M) == (12, 625)
    plans, unplanned = jaero_b200.channel_plan(jaero_b200.find_carriers(mean, fs), fs, M, interpolation=L)
    assert not unplanned, unplanned
    assert sorted(plans) == ["msk1200", "oqpsk10500"]
    assert len(plans["oqpsk10500"]["ddc"]["offsets_hz"]) == 5 and len(plans["msk1200"]["ddc"]["offsets_hz"]) == 2
    problems = []
    for mode, plan in plans.items():
        dd, dm = plan["ddc"], plan["demod"]
        assert (dd["input_rate"], dd["interpolation"], dd["decimation"]) == (fs, 12, 625)
        got = _run_plan(iq, "cs16", dd, dm, stream, chunk)
        for ch, f in enumerate(dd["offsets_hz"]):
            i = int(np.argmin(np.abs(np.array(offs) - f)))          # which transmitted carrier this planned channel is
            k0, n, run = _decoded(sent[i], got[ch])
            dk0, dn, _ = direct[i]
            name = "%s channel %d at %.1f Hz (carrier at %.1f Hz)" % (mode, ch, f, offs[i])
            print("%s: %d of %d signal units CRC-valid from unit %d on; direct path %d from unit %d on" % (name, n, len(sent[i]), k0, dn, dk0))
            if k0 < 0 or not run:
                problems.append("%s: not a contiguous run of the transmitted units" % name)
            elif abs((k0 + n) - (dk0 + dn)) > frame[mode]:
                problems.append("%s: the run ends at unit %d, the direct path's at %d" % (name, k0 + n, dk0 + dn))
            elif k0 > max(slowest[mode], dk0) + frame[mode]:
                problems.append("%s: locks at unit %d, the direct path's slowest channel at %d" % (name, k0, max(slowest[mode], dk0)))
    assert not problems, problems
