"""The mode identifier on the GPU: its squared-signal spectrum against the long-double reference at every size, its independence of
how the stream is cut and of the batch's other channels, the rates and carriers it finds on the recordings and on synthetic
signals, and probe_carriers -> channel_plan on a wideband SDR stream."""
import numpy as np
import pytest

import ident_reference as ref
from conftest import load_excerpt

pytestmark = pytest.mark.gpu

FB = dict(zip(ref.MODES, (600, 1200, 8400, 10500)))


def _pcm(C, n, Fs, seed):
    """C channels: a few tones below Fs/2 at random levels plus noise, some channels near full scale"""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    out = np.empty((C, n), dtype=np.int16)
    for c in range(C):
        x = rng.normal(0, 0.02 + 0.1 * rng.random(), n)
        for _ in range(3):
            x += rng.random() * 0.3 * np.cos(2 * np.pi * rng.uniform(100, Fs / 2 - 100) / Fs * t + rng.uniform(0, 6.3))
        out[c] = np.clip(np.round(x * 32767), -32768, 32767)
    return out


def _run(ident, pcm, cuts, device=False):
    """write pcm [C, n] through ident in pieces of the sizes `cuts`, from host or device memory"""
    import torch
    dev = torch.from_numpy(np.ascontiguousarray(pcm)).cuda() if device else None
    torch.cuda.synchronize()
    a = 0
    for m in cuts:
        if device:
            ident.write_device(dev.data_ptr() + 2 * a, m, pcm.shape[1])
        else:
            ident.write(pcm[:, a:a + m])
        a += m
    assert a == pcm.shape[1]
    out = ident.read()
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("Fs", [48000, 44100, 12000])
@pytest.mark.parametrize("nfft", [1024, 2048, 4096, 8192, 16384])
def test_spectrum_matches_reference(nfft, Fs):
    """33 channels ending part-way through a frame, within 1e-10 of each channel's largest bin"""
    import jaero_b200
    C, n = 33, 5 * nfft // 2 + nfft // 3
    pcm = _pcm(C, n, Fs, nfft + Fs)
    d = jaero_b200.Identifier(Fs, C, nfft)
    got, F = _run(d, pcm, [n // 3, n - n // 3])
    d.close()
    want, Fr = ref.spectrum(pcm, nfft)
    assert F == Fr == 4
    err = np.max(np.abs(got - want), axis=1) / np.max(want, axis=1)
    assert np.all(err < 1e-10), err.max()


@pytest.mark.parametrize("C,nfft", [(1, 16384), (1, 1024), (300, 16384), (300, 1024)])
def test_spectrum_matches_reference_channel_counts(C, nfft):
    import jaero_b200
    n = 3 * nfft + 5
    pcm = _pcm(C, n, 48000, C * nfft)
    d = jaero_b200.Identifier(48000, C, nfft)
    got, F = _run(d, pcm, [n])
    d.close()
    check = range(C) if C < 40 else np.random.default_rng(1).choice(C, 24, replace=False)
    want, _ = ref.spectrum(pcm[list(check)], nfft)
    err = np.max(np.abs(got[list(check)] - want), axis=1) / np.max(want, axis=1)
    assert F == 5 and np.all(err < 1e-10), err.max()


def test_output_does_not_depend_on_the_cuts():
    """bitwise: one write, random cuts with 1-sample and empty writes, host or device memory, and write -> reset -> write"""
    import jaero_b200
    nfft, C = 2048, 7
    n = 11 * nfft + 333
    pcm = _pcm(C, n, 48000, 3)
    d = jaero_b200.Identifier(48000, C, nfft)
    ref_sq, ref_F = _run(d, pcm, [n])
    rng = np.random.default_rng(4)
    for trial in range(4):
        cuts = []
        left = n
        while left:
            m = int(min(left, rng.choice([0, 1, 1, 7, 1023, 2048, 5000])))
            cuts.append(m); left -= m
        d.reset()
        sq, F = _run(d, pcm, cuts, device=bool(trial & 1))
        assert F == ref_F and np.array_equal(sq, ref_sq), trial
    d.reset()
    _run(d, _pcm(C, 3 * nfft, 48000, 9), [3 * nfft])
    d.reset()
    sq, F = _run(d, pcm, [n], device=True)
    assert F == ref_F and np.array_equal(sq, ref_sq)
    d.close()


def test_channels_are_independent():
    """each channel of a 300-channel batch, in permuted order, equals that channel run alone, bitwise"""
    import jaero_b200
    nfft, C = 1024, 300
    n = 6 * nfft + 100
    pcm = _pcm(C, n, 48000, 11)
    perm = np.random.default_rng(12).permutation(C)
    d = jaero_b200.Identifier(48000, C, nfft)
    batch, _ = _run(d, pcm[perm], [n // 2, n - n // 2])
    d.close()
    one = jaero_b200.Identifier(48000, 1, nfft)
    for k, c in enumerate(perm):
        one.reset()
        sq, _ = _run(one, pcm[c:c + 1], [n])
        assert np.array_equal(sq[0], batch[k]), c
    one.close()


def test_recordings_identify_their_rates():
    """the 48 kHz excerpts in one batch (each zero-padded to the longest: a channel's scale does not move its lines or scores'
    ratios), the 44.1 kHz one alone"""
    import jaero_b200
    names = [e for e in ref.EXCERPTS if e[1] == 48000]
    pcms = [load_excerpt(e[0]) for e in names]
    n = max(len(p) for p in pcms)
    batch = np.zeros((len(pcms), n), dtype=np.int16)
    for c, p in enumerate(pcms):
        batch[c, :len(p)] = p
    d = jaero_b200.Identifier(48000, len(pcms), 16384)
    sq, F = _run(d, batch, [4800] * (n // 4800) + [n % 4800])
    d.close()
    rows = list(zip(names, sq, [48000] * len(names)))
    for e in ref.EXCERPTS:
        if e[1] != 48000:
            d = jaero_b200.Identifier(e[1], 1, 16384)
            p = load_excerpt(e[0])[None]
            s, _ = _run(d, p, [p.shape[1]], device=True)
            d.close()
            rows.append((e, s[0], e[1]))
    problems = []
    for (name, fs, fb, carriers), row, _ in rows:
        r = jaero_b200.identify(row, fs, F)
        print(name, r["mode"], "%.2f Hz" % r["carrier_hz"], "%.1f dB margin" % r["margin_db"])
        if r["mode"] != ref.MODES[ref.FBS.index(float(fb))] or min(abs(r["carrier_hz"] - c) for c in carriers) > 2.0:
            problems.append((name, r))
    assert not problems, problems


def _synth(mode, fc, seed, seconds=4.0, ebn0=4.0):
    from jaero_b200 import synth
    fb = FB[mode]
    n = int(seconds * 48000)
    rng = np.random.default_rng(seed)
    nb = int(np.ceil(seconds * fb)) + 8
    nb += (-nb) % 56                                                   # a whole number of samples at every rate
    bits = rng.integers(0, 2, nb)
    if mode.startswith("oqpsk"):
        env = synth.oqpsk_envelope(bits, float(fb))
    else:
        if (bits ^ (np.arange(nb) & 1) ^ 1).sum() & 1:                 # the MSK pre-coder wants even parity
            bits[-1] ^= 1
        env = synth.msk_envelope(bits, float(fb))
    return synth.to_passband_int16(env[:n], fc, ebn0_db=ebn0, fb=float(fb), rng=rng)


def test_synthetic_signals_at_4_db():
    """every mode at Eb/N0 4 dB and a random carrier, 4 s: the right mode and the carrier within 0.5 Hz; 64 channels of noise
    only: unknown everywhere"""
    import jaero_b200
    rng = np.random.default_rng(21)
    cases = []
    for mode in ref.MODES:
        for k in range(3):
            lo, hi = (1500.0, 4000.0) if mode.startswith("msk") else (6000.0, 12000.0)
            cases.append((mode, float(rng.uniform(lo, hi)), 500 + len(cases)))
    pcm = np.stack([_synth(m, fc, s) for m, fc, s in cases])
    d = jaero_b200.Identifier(48000, len(cases), 16384)
    sq, F = _run(d, pcm, [4800] * 40, device=True)
    d.close()
    problems = []
    for (mode, fc, _), row in zip(cases, sq):
        r = jaero_b200.identify(row, 48000, F)
        print(mode, "%.2f" % fc, r["mode"], "%+.3f Hz" % (r["carrier_hz"] - fc), "%.1f dB" % r["score_db"][mode])
        if r["mode"] != mode or abs(r["carrier_hz"] - fc) > 0.5:
            problems.append((mode, fc, r))
    noise = np.clip(np.round(rng.normal(0, 0.2 * 32767, size=(64, 192000))), -32768, 32767).astype(np.int16)
    d = jaero_b200.Identifier(48000, 64, 16384)
    sq, F = _run(d, noise, [4800] * 40)
    d.close()
    top = 0.0
    for row in sq:
        r = jaero_b200.identify(row, 48000, F)
        top = max(top, max(r["score_db"].values()))
        if r["mode"] != "unknown":
            problems.append(("noise", r))
    print("noise: largest score %.2f dB" % top)
    assert not problems, problems


def test_probe_carriers_then_channel_plan_decodes_the_sdr_stream():
    """The seven-carrier stream of test_scan_driven_sdr_stream_through_ddc_demod_and_pchannel. The scanner's carriers are given
    mode "unknown" and centres up to 150 Hz off; probe_carriers must recover every mode and centre within 1 Hz, and channel_plan
    on its output must decode every carrier under that test's criteria, all on one CUDA stream."""
    import torch
    import jaero_b200
    from jaero_b200 import synth
    from test_gpu_ddc import _decoded, _run_direct, _run_chain, FS as DDC_FS, D, B, DT
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
    truth_mode = ["oqpsk10500"] * 4 + ["msk1200"] * 2 + ["oqpsk10500"]
    oq_idx, msk_idx = [0, 1, 2, 3, 6], [4, 5]
    direct = {}
    pcm = np.stack([synth.to_passband_int16(envs[i], 8000.0, ebn0_db=ebn0[i], fb=10500.0, rng=np.random.default_rng(70 + i)) for i in oq_idx])
    for ch, g in enumerate(_run_direct(pcm, "oqpsk", 10500, 8000.0, 10500)):
        direct[oq_idx[ch]] = _decoded(sent[oq_idx[ch]], g)
    pcm = np.stack([synth.to_passband_int16(envs[i], 2000.0, ebn0_db=12.0, fb=1200.0, rng=np.random.default_rng(80 + i)) for i in msk_idx])
    for ch, g in enumerate(_run_direct(pcm, "msk", 1200, 2000.0, 1800)):
        direct[msk_idx[ch]] = _decoded(sent[msk_idx[ch]], g)
    slowest = {"oqpsk10500": max(direct[i][0] for i in oq_idx[:4]), "msk1200": max(direct[i][0] for i in msk_idx)}
    frame = {"oqpsk10500": 26, "msk1200": 6}

    iq = synth.wideband_iq(envs, offs, DDC_FS, ebn0, fmt="cs16", seed=5, fb=fbs)
    stream = torch.cuda.Stream()
    dev = torch.from_numpy(iq).cuda()
    torch.cuda.synchronize()
    sc = jaero_b200.Scanner(DDC_FS, 1 << 16, 1 << 15)
    sc.set_stream(stream.cuda_stream)
    for a in range(0, iq.size // 2, 240_000):
        sc.write_device(dev.data_ptr() + 4 * a, min(240_000, iq.size // 2 - a), "cs16")
    mean, _, _ = sc.read()
    sc.close()
    found = jaero_b200.find_carriers(mean, DDC_FS)
    assert len(found) == 7
    rng = np.random.default_rng(33)
    blind = [dict(c, mode="unknown", center_hz=c["center_hz"] + float(rng.uniform(-150, 150))) for c in found]
    probed = jaero_b200.probe_carriers(blind, DDC_FS, (dev.data_ptr(), iq.size // 2), "cs16", decimation=D, seconds=4.0,
                                       stream=stream.cuda_stream)
    torch.cuda.synchronize()
    del dev
    problems = []
    for c in probed:
        i = int(np.argmin(np.abs(np.array(offs) - c["center_hz"])))
        print("carrier at %.1f Hz: %s, %.2f Hz off, fb %.2f, %.1f dB" % (offs[i], c["mode"], c["center_hz"] - offs[i], c["fb_hz"], c["ident_score_db"]))
        if c["mode"] != truth_mode[i] or abs(c["center_hz"] - offs[i]) > 1.0:
            problems.append(c)
    assert not problems, problems
    plans, unplanned = jaero_b200.channel_plan(probed, DDC_FS, D)
    assert not unplanned, unplanned
    assert sorted(plans) == ["msk1200", "oqpsk10500"]
    for mode, plan in plans.items():
        dd, dm = plan["ddc"], plan["demod"]
        got = _run_chain(iq, "cs16", (dd["offsets_hz"], dd["audio_hz"], dd["bandwidth"], dd["transition"], dd["gain"]),
                         dm["kind"], dm["fb"], dm["n_channels"], dm["freq_center"], dm["lockingbw"], stream)
        for ch, f in enumerate(dd["offsets_hz"]):
            i = int(np.argmin(np.abs(np.array(offs) - f)))
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
