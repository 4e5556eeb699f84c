"""GPU checks of the wideband IQ down-converter (jaero_b200.Ddc, include/jaero_b200.h jaero_ddc_*): every PCM sample against
the float64 reference (tests/ddc_reference.py), independence of how the stream is cut into writes, the retune rule, and a
known-answer run from one SDR stream through Ddc -> DemodBatch.write_device -> PChannelBatch on one CUDA stream."""
import numpy as np
import pytest

import ddc_reference as ref

pytestmark = pytest.mark.gpu

FS, D, B, DT = 2.4e6, 50, 12000.0, 4000.0


def _ddc(offsets, audio, gain, B=B, DT=DT):
    import jaero_b200
    return jaero_b200.Ddc(FS, D, offsets, audio, B, DT, gain=gain)


def _reference(x, offsets, audio, gain, T=None, S=None):
    import jaero_b200
    p = jaero_b200.ddc_plan(FS, D, B, DT)
    T = T if T is not None else [ref.tuning_word(o, FS) for o in offsets]
    S = S if S is not None else [ref.tuning_word(a, FS / D) for a in audio]
    return ref.ddc_reference(x, p["h1"], p["D1"], p["h2"], p["D2"], T, S, gain=gain)


def _assert_matches(got, val):
    """equal to the reference everywhere, except +-1 where the reference lies within 1e-6 LSB of a rounding boundary"""
    exp = np.clip(np.rint(val), -32768, 32767).astype(np.int64)
    diff = got.astype(np.int64) - exp
    near = np.abs(np.abs(val - np.floor(val)) - 0.5) < 1e-6
    assert not np.any((diff != 0) & ~(near & (np.abs(diff) <= 1))), np.argwhere((diff != 0) & ~near)[:10]
    n_near = int(np.count_nonzero(diff))
    print("samples within 1e-6 LSB of a rounding boundary that differ by one: %d of %d" % (n_near, diff.size))
    assert n_near < 1e-5 * diff.size


def _random_iq(fmt, n, seed):
    rng = np.random.default_rng(seed)
    if fmt == "cu8":
        return rng.integers(0, 256, size=2 * n, dtype=np.uint8)
    return rng.integers(-32768, 32768, size=2 * n, dtype=np.int16)


def _channels(C, seed):
    rng = np.random.default_rng(seed)
    edge = FS / 2 - B / 2
    off = rng.uniform(-edge, edge, size=C)
    if C > 1:
        off[0], off[1] = -edge, edge                             # both ends of the tunable range
    aud = rng.uniform(B / 2 + 1.0, FS / D / 2 - B / 2 - 1.0, size=C)
    return off, aud


@pytest.mark.parametrize("fmt", ["cu8", "cs16"])
@pytest.mark.parametrize("C,gain", [(1, 1.0), (33, 1.0), (300, 1.0), (33, 300.0)])
def test_ddc_equals_reference(fmt, C, gain):
    n = 150_001
    iq = _random_iq(fmt, n, seed=C + (7 if fmt == "cu8" else 0))
    off, aud = _channels(C, seed=C)
    d = _ddc(off, aud, gain)
    d.write(iq[:2 * 70_000], fmt)
    a = d.read_pcm()
    d.write(iq[2 * 70_000:], fmt)
    got = np.concatenate([a, d.read_pcm()], axis=1)
    inputs, clipped = d.stats()
    d.close()
    _, val, clip_ref, _ = _reference(ref.iq_to_complex(iq, fmt), off, aud, gain)
    assert inputs == n and got.shape == (C, (n - 1) // D + 1)
    _assert_matches(got, val)
    np.testing.assert_array_equal(clipped, clip_ref)
    if gain > 1:
        assert clip_ref.min() > 0                                # the high-gain case does clip, on every channel


def test_ddc_output_does_not_depend_on_how_the_stream_is_cut():
    import torch
    fmt, n = "cs16", 240_007
    iq = _random_iq(fmt, n, seed=3)
    off, aud = _channels(40, seed=4)
    d = _ddc(off, aud, 4.0)
    d.write(iq, fmt)
    whole = d.read_pcm()
    d.close()
    rng = np.random.default_rng(11)
    pieces = [1, D - 1, 7, 101, 997, 50_000, 2, 3, D, D + 1, 65_537]
    cuts = []
    while sum(cuts) < n:
        cuts.append(min(int(pieces[len(cuts) % len(pieces)] if len(cuts) < len(pieces) else rng.choice(pieces)), n - sum(cuts)))
    dev = torch.from_numpy(iq).cuda()
    torch.cuda.synchronize()
    for path in ("host", "device"):
        d = _ddc(off, aud, 4.0)
        parts, a = [], 0
        for c in cuts:
            if path == "host":
                d.write(iq[2 * a:2 * (a + c)], fmt)
            else:
                d.write_device(dev.data_ptr() + 4 * a, c, fmt)
            parts.append(d.read_pcm())
            a += c
        d.close()
        got = np.concatenate(parts, axis=1)
        assert got.shape == whole.shape
        assert np.array_equal(got, whole), path


def test_ddc_retune_follows_the_rule():
    """set_offset between writes applies to stage-1 samples whose input j*D1 arrives later; set_audio_freq to outputs whose
    input m*D arrives later"""
    fmt = "cu8"
    iq = _random_iq(fmt, 200_000, seed=21)
    off, aud = _channels(9, seed=22)
    d = _ddc(off, aud, 8.0)
    a, b = 60_013, 130_000
    d.write(iq[:2 * a], fmt); p0 = d.read_pcm()
    off2 = off.copy(); off2[3] = 123_456.78; off2[5] = -1_000_000.0
    d.set_offset(off2[3], channel=3); d.set_offset(off2[5], channel=5)
    d.write(iq[2 * a:2 * b], fmt); p1 = d.read_pcm()
    aud2 = np.full(9, 17_000.0)
    d.set_audio_freq(17_000.0)
    off3 = np.full(9, -250_000.0)
    d.set_offset(-250_000.0)
    d.write(iq[2 * b:], fmt); p2 = d.read_pcm()
    d.close()
    tw = lambda o: [ref.tuning_word(f, FS) for f in o]
    sw = lambda o: [ref.tuning_word(f, FS / D) for f in o]
    _, val, _, _ = _reference(ref.iq_to_complex(iq, fmt), None, None, 8.0, T=[(0, tw(off)), (a, tw(off2)), (b, tw(off3))],
                              S=[(0, sw(aud)), (b, sw(aud2))])
    _assert_matches(np.concatenate([p0, p1, p2], axis=1), val)


def _decoded(sent, got_list):
    """-> (index in `sent` of the first CRC-valid SU, number of CRC-valid SUs, whether they are a contiguous run of `sent`)"""
    got = [bytes(x) for b, ok in got_list for x in b[ok.astype(bool)]]
    if not got or got[0] not in sent:
        return -1, len(got), False
    k0 = sent.index(got[0])
    return k0, len(got), got == sent[k0:k0 + len(got)]


def _run_direct(pcm, kind, fb, audio, lockingbw):
    """the same demodulator and frame layer fed 48 kHz PCM straight from the generator (no DDC), written in the same 4800-sample
    pieces: the lock and the end-of-stream latency the DDC path is compared with"""
    import jaero_b200
    n_ch = pcm.shape[0]
    b = jaero_b200.DemodBatch(kind, n_ch, fb=fb, freq_center=audio, lockingbw=lockingbw)
    pc = jaero_b200.PChannelBatch(n_ch, fb)
    got = [[] for _ in range(n_ch)]
    for k, a in enumerate(range(0, pcm.shape[1], 4800)):
        b.write(pcm[:, a:a + 4800])
        pc.process_batch(b)
        if k % 10 == 9:
            for ch, r in enumerate(pc.read_sus()):
                got[ch].append((r[0], r[1]))
    for ch, r in enumerate(pc.read_sus()):
        got[ch].append((r[0], r[1]))
    b.close(); pc.close()
    return got


def _run_chain(iq, fmt, ddc_args, kind, fb, n_ch, audio, lockingbw, stream):
    """Ddc -> DemodBatch.write_device -> PChannelBatch.process_batch on one CUDA stream, no host copy of the PCM"""
    import torch
    import jaero_b200
    dev = torch.from_numpy(iq).cuda()
    torch.cuda.synchronize()
    d = jaero_b200.Ddc(FS, D, *ddc_args)
    b = jaero_b200.DemodBatch(kind, n_ch, fb=fb, freq_center=audio, lockingbw=lockingbw)
    pc = jaero_b200.PChannelBatch(n_ch, fb)
    d.set_stream(stream.cuda_stream); b.set_stream(stream.cuda_stream)
    bytes_per = 2 if fmt == "cu8" else 4
    n = iq.size // 2
    chunk = 240_000                                              # 0.1 s of IQ, 4800 PCM samples per channel
    got = [[] for _ in range(n_ch)]
    for k, a in enumerate(range(0, n, chunk)):
        c = min(chunk, n - a)
        d.write_device(dev.data_ptr() + bytes_per * a, c, fmt)
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


def test_sdr_stream_known_answer_through_ddc_demod_and_pchannel():
    """Every channel of the SDR stream decodes a contiguous run of the transmitted signal units, measured against the same
    demodulator and frame layer fed the same envelopes as 48 kHz PCM at the same Eb/N0 (the direct path):
    - the run ends where the direct path's run of that channel ends, within one frame. The last frames are still inside the
      demodulator, interleaver and decoder when the stream ends; the DDC adds no latency of its own;
    - it starts no later than one frame after the slowest lock the direct path shows among the channels of that mode. The
      demodulator locks at a frame boundary that depends on the noise realisation (on the direct path too, channels of the
      same Eb/N0 lock anywhere from the 2nd to the 5th 10.5 kbps frame), so a channel is compared with that spread, not with
      its own direct twin."""
    import torch
    from jaero_b200 import synth
    oq_off = [-700_123.0, -150_000.0, 260_500.0, 810_000.0]
    msk_off = [-420_000.0, 530_250.0]
    neighbour = oq_off[1] + B / 2 + DT + 5250.0 + 1000.0          # 10.5 kbps neighbour whose spectrum starts 1 kHz past B/2 + DT
    envs, sus, offs, ebn0, fbs = [], [], [], [], []
    for i, f in enumerate(oq_off):
        bits, s = synth.pchannel_bits(10500, 16, seed=300 + i, return_sus=True)
        envs.append(synth.oqpsk_envelope(bits, 10500.0)); sus.append(s); offs.append(f); ebn0.append(11.0); fbs.append(10500.0)
    for i, f in enumerate(msk_off):
        bits, s = synth.pchannel_bits(1200, 8, seed=400 + i, return_sus=True, loop=True, even_parity=True)
        envs.append(synth.msk_envelope(bits, 1200.0)); sus.append(s); offs.append(f); ebn0.append(12.0); fbs.append(1200.0)
    nb = synth.pchannel_bits(10500, 16, seed=999)
    envs.append(synth.oqpsk_envelope(nb, 10500.0)); offs.append(neighbour); ebn0.append(31.0); fbs.append(10500.0)   # 20 dB up
    sent = [[bytes(x) for x in s_.reshape(-1, 12)] for s_ in sus]
    direct = {}
    pcm = np.stack([synth.to_passband_int16(envs[i], 8000.0, ebn0_db=11.0, fb=10500.0, rng=np.random.default_rng(70 + i)) for i in range(4)])
    for ch, g in enumerate(_run_direct(pcm, "oqpsk", 10500, 8000.0, 10500)):
        direct[ch] = _decoded(sent[ch], g)
    pcm = np.stack([synth.to_passband_int16(envs[4 + i], 2000.0, ebn0_db=12.0, fb=1200.0, rng=np.random.default_rng(80 + i)) for i in range(2)])
    for ch, g in enumerate(_run_direct(pcm, "msk", 1200, 2000.0, 1800)):
        direct[4 + ch] = _decoded(sent[4 + ch], g)
    stream = torch.cuda.Stream()
    problems = []

    for i, (dk0, dn, drun) in direct.items():
        assert dk0 >= 0 and drun, "the direct path did not lock on channel %d" % i
    slowest = {"OQPSK": max(direct[i][0] for i in range(4)), "MSK": max(direct[i][0] for i in (4, 5))}

    def check(name, i, got_list, frame):
        k0, n, run = _decoded(sent[i], got_list)
        dk0, dn, _ = direct[i]
        mode = name.split()[1]
        print("%s: DDC path %d of %d signal units CRC-valid from unit %d on; direct 48 kHz path %d from unit %d on"
              % (name, n, len(sent[i]), k0, dn, dk0))
        if k0 < 0 or not run:
            problems.append("%s: not a contiguous run of the transmitted units" % name)
        elif abs((k0 + n) - (dk0 + dn)) > frame:
            problems.append("%s: the run ends at unit %d, the direct path's at %d" % (name, k0 + n, dk0 + dn))
        elif k0 > slowest[mode] + frame:
            problems.append("%s: locks at unit %d, the direct path's slowest %s channel at %d" % (name, k0, mode, slowest[mode]))

    for fmt in ("cs16", "cu8"):
        iq, lv = synth.wideband_iq(envs, offs, FS, ebn0, fmt=fmt, seed=5, fb=fbs, return_levels=True)
        g_oq = 0.2 * np.sqrt(2) / lv[0]
        oq_n = 4 if fmt == "cs16" else 1
        got = _run_chain(iq, fmt, (oq_off[:oq_n], 8000.0, B, DT, g_oq), "oqpsk", 10500, oq_n, 8000.0, 10500, stream)
        for ch in range(oq_n):
            check("%s OQPSK channel %d" % (fmt, ch), ch, got[ch], 26)
        if fmt == "cs16":
            g_msk = 0.2 * np.sqrt(2) / lv[4]
            got = _run_chain(iq, fmt, (msk_off, 2000.0, 3000.0, 1000.0, g_msk), "msk", 1200, 2, 2000.0, 1800, stream)
            for ch in range(2):
                check("%s MSK channel %d" % (fmt, ch), 4 + ch, got[ch], 6)
    assert not problems, problems


def test_single_stage_plan_equals_reference():
    """a small decimation plans one stage (D2 = 1, h2 = {1}, no stage-2 history); written in pieces"""
    import jaero_b200
    fs, dec = 96000.0, 2
    p = jaero_b200.ddc_plan(fs, dec, B, DT)
    assert p["D2"] == 1 and p["K2"] == 1 and list(p["h2"]) == [1.0]
    rng = np.random.default_rng(31)
    iq = _random_iq("cs16", 20_011, seed=32)
    off = rng.uniform(-(fs / 2 - B / 2), fs / 2 - B / 2, size=33); off[0] = fs / 2 - B / 2
    aud = rng.uniform(B / 2 + 1.0, fs / dec / 2 - B / 2 - 1.0, size=33)
    d = jaero_b200.Ddc(fs, dec, off, aud, B, DT, gain=16.0)
    parts, a = [], 0
    for c in (1, 2, 3, 997, 5000, 14_008):
        d.write(iq[2 * a:2 * (a + c)], "cs16"); parts.append(d.read_pcm()); a += c
    _, clipped = d.stats()
    d.close()
    T = [ref.tuning_word(o, fs) for o in off]
    S = [ref.tuning_word(x, fs / dec) for x in aud]
    _, val, clip_ref, _ = ref.ddc_reference(ref.iq_to_complex(iq, "cs16"), p["h1"], p["D1"], p["h2"], p["D2"], T, S, gain=16.0)
    _assert_matches(np.concatenate(parts, axis=1), val)
    np.testing.assert_array_equal(clipped, clip_ref)


def test_retune_rejections_leave_the_ddc_unchanged():
    import jaero_b200
    off, aud = _channels(5, seed=41)
    iq = _random_iq("cu8", 30_000, seed=42)
    d = _ddc(off, aud, 8.0)
    d.write(iq[:20_000], "cu8")
    for bad in (FS / 2 - B / 2 + 1.0, -FS / 2, float("nan")):
        with pytest.raises(jaero_b200.JaeroError, match="offset"):
            d.set_offset(bad, channel=2)
    for bad in (B / 2, FS / D / 2 - B / 2, -8000.0):
        with pytest.raises(jaero_b200.JaeroError, match="audio passband"):
            d.set_audio_freq(bad)
    with pytest.raises(jaero_b200.JaeroError, match="bad argument"):
        d.set_offset(0.0, channel=5)
    with pytest.raises(ValueError):
        d.write(iq.astype(np.int16), "cu8")
    d.write(iq[20_000:], "cu8")
    got = d.read_pcm()
    d.close()
    _, val, _, _ = _reference(ref.iq_to_complex(iq, "cu8"), off, aud, 8.0)
    _assert_matches(got, val[:, val.shape[1] - got.shape[1]:])
