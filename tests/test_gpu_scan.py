"""GPU checks of the wideband carrier scanner (jaero_b200.Scanner, include/jaero_b200.h jaero_scan_*): mean and max-hold spectra
against the float64 reference (tests/scan_reference.py) at every size, independence of how the stream is cut into writes, a
known-answer spectrum of five carriers, a burst seen through max-hold, and a run in which the scanner alone plans the
down-converter and the demodulators of an SDR stream."""
import numpy as np
import pytest

import scan_reference as ref

pytestmark = pytest.mark.gpu

FS = 2.4e6


def _random_iq(fmt, n, seed):
    rng = np.random.default_rng(seed)
    if fmt == "cu8":
        return rng.integers(0, 256, size=2 * n, dtype=np.uint8)
    return rng.integers(-32768, 32768, size=2 * n, dtype=np.int16)


def _scan_host(iq, fmt, nfft, hop, cuts=None):
    import jaero_b200
    s = jaero_b200.Scanner(FS, nfft, hop)
    n = iq.size // 2
    a = 0
    for c in (cuts or [n]):
        s.write(iq[2 * a:2 * (a + c)], fmt)
        a += c
    out = s.read()
    s.close()
    return out


CASES = [(1 << p, h) for p in range(10, 17) for h in ("777", "q", "h", "n")]


@pytest.mark.parametrize("nfft,hop_kind", CASES)
def test_scan_equals_reference(nfft, hop_kind):
    hop = {"777": 777, "q": nfft // 4, "h": nfft // 2, "n": nfft}[hop_kind]
    for k, fmt in enumerate(("cu8", "cs16")):
        n = 2 * nfft + 5 * hop + 123 + 17 * k                          # ends part-way through a frame
        iq = _random_iq(fmt, n, seed=nfft + hop + k)
        mean, mx, F = _scan_host(iq, fmt, nfft, hop, cuts=[n // 3, n - n // 3])
        rm, rx, rF = ref.scan(ref.iq_to_complex(iq, fmt), nfft, hop)
        assert F == rF and F >= 3
        assert np.max(np.abs(mean - rm)) <= 1e-10 * np.max(rm), (fmt, np.max(np.abs(mean - rm)) / np.max(rm))
        assert np.max(np.abs(mx - rx)) <= 1e-10 * np.max(rx), fmt


def test_scan_hop_one_equals_reference():
    nfft, n = 1024, 3000
    iq = _random_iq("cs16", n, seed=5)
    mean, mx, F = _scan_host(iq, "cs16", nfft, 1, cuts=[100, 1500, 1400])
    rm, rx, rF = ref.scan(ref.iq_to_complex(iq, "cs16"), nfft, 1)
    assert F == rF == n - nfft + 1
    assert np.max(np.abs(mean - rm)) <= 1e-10 * np.max(rm)
    assert np.max(np.abs(mx - rx)) <= 1e-10 * np.max(rx)


def test_scan_does_not_depend_on_how_the_stream_is_cut():
    import torch
    import jaero_b200
    nfft, hop, fmt, n = 4096, 777, "cs16", 200_003
    iq = _random_iq(fmt, n, seed=3)
    whole = _scan_host(iq, fmt, nfft, hop)
    rng = np.random.default_rng(11)
    cuts = []
    while sum(cuts) < n:
        cuts.append(int(min(rng.choice([1, 2, 776, 777, 778, 4095, 4096, 4097, 9000, 30001]), n - sum(cuts))))
    host = _scan_host(iq, fmt, nfft, hop, cuts)
    dev = torch.from_numpy(iq).cuda()
    torch.cuda.synchronize()
    s = jaero_b200.Scanner(FS, nfft, hop)
    a = 0
    for c in cuts:
        s.write_device(dev.data_ptr() + 4 * a, c, fmt)
        a += c
    device = s.read()
    # reset restarts the count and the origin: the same stream after other samples gives the same result
    s.reset()
    assert s.read()[2] == 0
    s.write(_random_iq(fmt, 5000, seed=4)[:2 * 4999], fmt)
    s.reset()
    s.write(iq, fmt)
    after_reset = s.read()
    launches = s.launches
    s.close()
    for name, got in (("host", host), ("device", device), ("reset", after_reset)):
        assert got[2] == whole[2], name
        assert got[0].tobytes() == whole[0].tobytes() and got[1].tobytes() == whole[1].tobytes(), name
    assert launches > 0


def _known_answer_stream(fmt, seed=5):
    """2.4 MS/s, 4 s: 10.5 kbps OQPSK (11 dB) and its 20 dB stronger 10.5 kbps neighbour, 8400 bps OQPSK (alpha 0.6, 11 dB),
    1200 and 600 bps MSK (12 dB)"""
    from jaero_b200 import synth
    rng = np.random.default_rng(seed)
    envs, offs, ebn0, fbs, modes = [], [], [], [], []
    def add(env, f, e, fb, mode):
        envs.append(env); offs.append(f); ebn0.append(e); fbs.append(fb); modes.append(mode)
    add(synth.oqpsk_envelope(synth.pchannel_bits(10500, 8, seed=1), 10500.0), -600_000.0, 11.0, 10500.0, "oqpsk10500")
    add(synth.oqpsk_envelope(synth.pchannel_bits(10500, 8, seed=2), 10500.0), -600_000.0 + 16_250.0, 31.0, 10500.0, "oqpsk10500")
    add(synth.oqpsk_envelope(rng.integers(0, 2, size=4 * 8400).astype(np.uint8), 8400.0, alpha=0.6), -210_000.0, 11.0, 8400.0, "oqpsk8400")
    add(synth.msk_envelope(synth.pchannel_bits(1200, 4, seed=3, loop=True, even_parity=True), 1200.0), 250_300.0, 12.0, 1200.0, "msk1200")
    add(synth.msk_envelope(synth.pchannel_bits(600, 2, seed=4, loop=True, even_parity=True), 600.0), 705_000.0, 12.0, 600.0, "msk600")
    iq, lv = synth.wideband_iq(envs, offs, FS, ebn0, fmt=fmt, seed=seed, fb=fbs, return_levels=True)
    return iq, np.array(offs), lv, modes


@pytest.mark.parametrize("fmt", ["cs16", "cu8"])
def test_scan_known_answer(fmt):
    import jaero_b200
    iq, offs, lv, modes = _known_answer_stream(fmt)
    nfft, hop = 1 << 16, 1 << 15
    s = jaero_b200.Scanner(FS, nfft, hop)
    for a in range(0, iq.size, 2 * 240_000):
        s.write(iq[a:a + 2 * 240_000], fmt)
    mean, _, F = s.read()
    s.close()
    assert F == (iq.size // 2 - nfft) // hop + 1
    found = jaero_b200.find_carriers(mean, FS)
    bin_hz = FS / nfft
    for c in found:
        print("%10.1f Hz  width %7.1f Hz  %-10s  power %.3e  snr %5.1f dB  flags %d" % (c["center_hz"], c["width_hz"], c["mode"], c["power"], c["snr_db"], c["flags"]))
    assert len(found) == len(offs)
    order = np.argsort(offs)
    for c, k in zip(found, order):
        assert abs(c["center_hz"] - offs[k]) <= bin_hz, (c["center_hz"], offs[k])
        assert c["mode"] == modes[k], (c["center_hz"], c["width_hz"], c["mode"], modes[k])
        assert abs(10 * np.log10(c["power"] / lv[k] ** 2)) <= 1.0, (c["center_hz"], c["power"], lv[k] ** 2)
        assert c["flags"] == 0


def test_scan_burst_visible_in_max_hold():
    """a 1200 bps MSK carrier on for one 0.2 s burst of a 4 s stream (20 dB Eb/N0 during the burst) shows in max-hold"""
    import jaero_b200
    from jaero_b200 import synth
    env = synth.msk_envelope(synth.pchannel_bits(1200, 4, seed=6, loop=True, even_parity=True), 1200.0)
    gate = np.zeros(len(env)); gate[int(1.5 * 48000):int(1.7 * 48000)] = 1.0
    off = 333_333.0
    iq = synth.wideband_iq([env * gate], [off], FS, 20.0 + 10 * np.log10(0.2 / 4.0), fmt="cs16", seed=7, fb=1200.0)
    nfft = 1 << 16
    s = jaero_b200.Scanner(FS, nfft, nfft // 4)
    s.write(iq, "cs16")
    mean, mx, _ = s.read()
    s.close()
    found = jaero_b200.find_carriers(mx, FS)
    for c in found:
        print("max-hold: %10.1f Hz  width %7.1f Hz  snr %5.1f dB" % (c["center_hz"], c["width_hz"], c["snr_db"]))
    assert any(abs(c["center_hz"] - off) <= FS / nfft for c in found)


def test_scan_driven_sdr_stream_through_ddc_demod_and_pchannel():
    """The signal set of test_gpu_ddc's end-to-end run, but nothing from the generator reaches the receiver: the offsets, modes and
    gains come from Scanner -> find_carriers -> channel_plan. Every planned P-channel carrier (the 20 dB stronger neighbour too)
    decodes a contiguous run of its transmitted signal units, judged as that test judges it against the same demodulator fed the
    same envelope as 48 kHz PCM. The scanner, the down-converters, the batches and the frame layers share one CUDA stream."""
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
    oq_idx, msk_idx = [0, 1, 2, 3, 6], [4, 5]
    # the direct 48 kHz path: the lock and end-of-stream latency each channel is judged against
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
    del dev
    plans, unplanned = jaero_b200.channel_plan(jaero_b200.find_carriers(mean, DDC_FS), DDC_FS, D)
    assert not unplanned, unplanned
    assert sorted(plans) == ["msk1200", "oqpsk10500"]
    assert len(plans["oqpsk10500"]["ddc"]["offsets_hz"]) == 5 and len(plans["msk1200"]["ddc"]["offsets_hz"]) == 2
    problems = []
    for mode, plan in plans.items():
        dd, dm = plan["ddc"], plan["demod"]
        assert dd["input_rate"] == DDC_FS and dd["decimation"] == D
        got = _run_chain(iq, "cs16", (dd["offsets_hz"], dd["audio_hz"], dd["bandwidth"], dd["transition"], dd["gain"]),
                         dm["kind"], dm["fb"], dm["n_channels"], dm["freq_center"], dm["lockingbw"], stream)
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
