"""Receiver end to end on the GPU: a wideband SDR stream carrying synthetic P-channel carriers at 600, 1200 and 10 500 bps with
known ACARS messages and the committed 8400 bps recording, decoded by one Receiver; compared with the known messages, with the
recording decoded directly at 48 kHz, and with the same stages wired by hand."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import reasm_synth
from conftest import ROOT, load_excerpt

pytestmark = pytest.mark.gpu

SECONDS = 12.0
EBN0_DB = 10.0
ACQUIRE = 4.0
# (fb, offset Hz, lead-in frames of fill, frames of messages, tail frames of fill); every carrier is 12 s of frames. The lead-in
# covers the demodulator's lock (on this stream the 10.5 kbps carriers decode from about 3 s on), the tail the frame layer's
# delay line at the end of the stream. The 1200 bps carrier's first messages are sent inside the acquisition window, so they
# are decoded only if the receiver replays it.
P_CARRIERS = [(600, -610_000.0, 2, 2, 2), (1200, -230_000.0, 3, 7, 2), (10500, 310_000.0, 8, 13, 3), (10500, 720_000.0, 8, 13, 3)]
C_OFFSET = -900_000.0                  # where the 8400 bps recording's 8 kHz audio lands
BURST_OFFSET = 950_000.0
MODE = {600: "msk600", 1200: "msk1200", 10500: "oqpsk10500"}


def _sus_per_frame(fb):
    from jaero_b200 import synth
    fp = synth.frame_params(fb)
    return fp["blocks"] * 64 * fp["cols"] // 2 // 96


def _carrier(i, fb, lead, body, tail):
    """one P-channel carrier's envelope and its messages [(aesid, reg, label, text)]: messages fill `body` frames after `lead`
    frames of fill"""
    from jaero_b200 import synth
    k = _sus_per_frame(fb)
    rng = np.random.default_rng(1000 + i)
    sus, msgs = [], []
    while True:
        aes = 0x100000 * (i + 1) + len(msgs)
        reg = "N%d%02dQ" % (i, len(msgs))
        label = "".join("HQ15AB_"[x] for x in rng.integers(0, 7, 2))
        text = "C%d M%d %s" % (i, len(msgs), "".join("ABCDEFGHIJ"[x] for x in rng.integers(0, 10, int(rng.integers(2, 16)))))
        s = reasm_synth.isu_to_sus(aes, 0x90, len(msgs) & 15, 3, reasm_synth.acars_userdata(reg, label, ord("A") + len(msgs), text))
        if len(sus) + len(s) > body * k:
            break
        sus += s
        msgs.append((aes, reg, label, text))
    units = [synth.FILL_SU] * (lead * k) + sus
    units += [synth.FILL_SU] * ((lead + body + tail) * k - len(units))
    msk = fb != 10500
    bits = synth.pchannel_bits_from_sus(fb, units, loop=msk, even_parity=msk)
    env = synth.msk_envelope(bits, fb) if msk else synth.oqpsk_envelope(bits, fb)
    assert len(env) == int(SECONDS * 48000)
    return env, msgs


def _analytic(pcm, lo, hi, shift):
    """a real 48 kHz recording as a complex envelope: its band [lo, hi] Hz only, moved down by `shift` Hz"""
    x = np.asarray(pcm, dtype=np.float64)
    X = np.fft.fft(x)
    f = np.fft.fftfreq(len(x), 1.0 / 48000.0)
    X[(f < lo) | (f > hi)] = 0.0
    a = np.fft.ifft(2.0 * X)
    return a * np.exp(-2j * np.pi * shift * np.arange(len(x)) / 48000.0)


def _stream(fs, fmt, burst=False):
    from jaero_b200 import synth
    envs, offs, ebn0, fbs, msgs = [], [], [], [], []
    for i, (fb, off, lead, body, tail) in enumerate(P_CARRIERS):
        e, m = _carrier(i, fb, lead, body, tail)
        envs.append(e); offs.append(off); ebn0.append(EBN0_DB); fbs.append(float(fb)); msgs.append(m)
    envs.append(_analytic(load_excerpt("oqpsk_8400"), 300.0, 13000.0, 8000.0)); offs.append(C_OFFSET); ebn0.append(20.0); fbs.append(8400.0)
    if burst:
        envs.append(_analytic(load_excerpt("burst_msk_1200_a"), 300.0, 3500.0, 2000.0)); offs.append(BURST_OFFSET)
        ebn0.append(20.0); fbs.append(1200.0)
    iq = synth.wideband_iq(envs, offs, fs, ebn0, fmt=fmt, seed=77, fb=fbs)
    return iq, msgs


def _run(iq, fs, fmt, block=0.1, pieces=(1.7, 0.23, 3.1), emit_sus=True):
    """the whole stream through one Receiver, written from the host in pieces of the given lengths (seconds, cycled), then
    flushed -> (events, carriers, unplanned, stats)"""
    import jaero_b200
    n = iq.size // 2
    ev = []
    with jaero_b200.Receiver(fs, fmt, acquire_seconds=ACQUIRE, block_seconds=block, emit_sus=emit_sus) as rx:
        a, k = 0, 0
        while a < n:
            m = min(n - a, int(pieces[k % len(pieces)] * fs)); k += 1
            ev += rx.write(iq[2 * a:2 * (a + m)])
            a += m
        ev += rx.flush()
        return ev, rx.carriers(), rx.unplanned(), rx.stats()


def _acars(ev):
    return sorted((e["carrier"], e["aesid"], e["reg"].decode("latin-1").strip("."), e["label"].decode("latin-1"),
                   e["text"].decode("latin-1")) for e in ev if e["kind"] == "acars" and e["record_kind"] == 0)


_DIRECT = {}


def _direct_cchannel_sus(freq_center, as_placed=False):
    """the CRC-valid C-channel signal units (a Counter) that the demodulator and frame layer decode from the recording at 48 kHz
    with the demodulator centred at freq_center and channel_plan's other 8400 bps settings, in 0.1 s writes. As in the band,
    noise follows the recording up to SECONDS, so the frames still inside the decoder when the recording ends come out.
    as_placed: the recording as the band carries it (only its 300 Hz - 13 kHz band), back at 48 kHz real PCM."""
    from collections import Counter
    import jaero_b200
    key = (round(float(freq_center), 3), as_placed)
    if key not in _DIRECT:
        s = jaero_b200.CHANNEL_SETTINGS["oqpsk8400"]
        rec = load_excerpt("oqpsk_8400")
        if as_placed:
            a = _analytic(rec, 300.0, 13000.0, 0.0)
            rec = np.clip(np.round(a.real), -32768, 32767).astype(np.int16)
        tail = np.random.default_rng(3).normal(0.0, 0.1 * rec.std(), int(SECONDS * 48000) - len(rec))
        pcm = np.concatenate([rec, np.round(tail).astype(np.int16)])[None, :]
        b = jaero_b200.DemodBatch("oqpsk", 1, fb=8400, freq_center=key[0], lockingbw=s["lockingbw"])
        cc = jaero_b200.CChannelBatch(1)
        got = Counter()
        for k, a in enumerate(range(0, pcm.shape[1], 4800)):
            b.write(pcm[:, a:a + 4800]); cc.process_batch(b)
            if (k + 1) % 10 == 0:
                cc.tick(b)
            su, ok, _, _ = cc.read_frames()[0]
            got.update(x.tobytes() for f in range(len(ok)) for x, o in zip(su[f], ok[f]) if o)
        b.close(); cc.close()
        _DIRECT[key] = got
    return _DIRECT[key]


def _check_known_answer(ev, carriers, msgs, tag):
    planned_p = sorted((c["mode"], c["center_hz"]) for c in carriers if c["mode"] != "oqpsk8400")
    want_p = sorted((MODE[fb], off) for fb, off, *_ in P_CARRIERS)
    assert [m for m, _ in planned_p] == [m for m, _ in want_p], (tag, planned_p)
    assert all(abs(f - g) < 5.0 for (_, f), (_, g) in zip(planned_p, want_p)), (tag, planned_p)
    c8400 = [c["index"] for c in carriers if c["mode"] == "oqpsk8400"]
    assert c8400 and all(abs(carriers[i]["center_hz"] - C_OFFSET) < 8000.0 for i in c8400), (tag, carriers)
    # ACARS: exactly the sent messages, each on its own carrier
    idx = {}
    for c in carriers:
        if c["mode"] != "oqpsk8400":
            idx[c["index"]] = int(np.argmin([abs(c["center_hz"] - off) for _, off, *_ in P_CARRIERS]))
    got = _acars(ev)
    assert all(g[0] in idx for g in got), (tag, "a message from a carrier that sent none", got)
    want = sorted((ci, aes, reg, label, text) for ci, i in idx.items() for aes, reg, label, text in msgs[i])
    missing = sorted(set(want) - set(got)); extra = sorted(set(got) - set(want))
    print("%s: %d ACARS messages of %d sent; missing %s; extra %s" % (tag, len(got), len(want), missing, extra))
    assert got == want, (tag, missing, extra)
    frame_s = {600: 2.0, 1200: 1.0, 10500: 0.5}
    assert any(lead * frame_s[fb] < ACQUIRE and msgs[i] for i, (fb, _, lead, _, _) in enumerate(P_CARRIERS))
    # C-channel: the receiver reports at least 90 % of the CRC-valid units (counted with repeats) that the recording gives when
    # decoded directly at 48 kHz, as committed or as placed in the band, with the demodulator centred as channel_plan centres
    # it (8 kHz) or on the carrier the receiver identified (where its down-converter puts it). A unit no direct decode gives
    # must sit in a frame whose other CRC-valid units one does give: a frame the direct decodes also frame, not a false sync.
    # (On this band the receiver locks one frame earlier than every direct decode; that frame carries one such unit.)
    from collections import Counter
    rx_c = Counter(s for e in ev if e["kind"] == "cframe" for s, o in zip(e["sus"], e["crc_ok"]) if o)
    direct = Counter()
    for fc in [8000.0] + [8000.0 + (carriers[i]["center_hz"] - C_OFFSET) for i in c8400]:
        for placed in (False, True):
            direct = direct | _direct_cchannel_sus(fc, placed)
    frac = sum((rx_c & direct).values()) / max(1, sum(direct.values()))
    only_rx = [e for e in ev if e["kind"] == "cframe" and any(o and s not in direct for s, o in zip(e["sus"], e["crc_ok"]))]
    print("%s: C-channel %d CRC-valid units (%d distinct), directly %d (%d distinct), %.1f %% of those reported; %d frame(s) "
          "with units no direct decode gives" % (tag, sum(rx_c.values()), len(rx_c), sum(direct.values()), len(direct), 100 * frac,
                                                 len(only_rx)))
    assert direct, tag
    for e in only_rx:
        assert any(o and s in direct for s, o in zip(e["sus"], e["crc_ok"])), (tag, e["frame"], e["sus"], e["crc_ok"])
    assert frac >= 0.9, (tag, frac)


@pytest.fixture(scope="module")
def cs16_stream():
    return _stream(2.4e6, "cs16")


@pytest.fixture(scope="module")
def cs16_run(cs16_stream):
    iq, _ = cs16_stream
    return _run(iq, 2.4e6, "cs16")


def test_known_answer_all_four_continuous_modes(cs16_stream, cs16_run):
    _, msgs = cs16_stream
    ev, carriers, unplanned, st = cs16_run
    print("carriers:", [(c["mode"], round(c["center_hz"], 1), round(c["snr_db"], 1)) for c in carriers])
    print("unplanned:", [(c["mode"], round(c["center_hz"], 1), c["reason"]) for c in unplanned])
    print("stats:", st)
    _check_known_answer(ev, carriers, msgs, "2.4 MS/s cs16")
    assert st["blocks"] == 120 and abs(st["seconds"] - SECONDS) < 1e-9
    # the P-channel carriers' channels do not clip; the 8400 bps recording's channel may (channel_plan sets its gain from the
    # scanner's power of the recording's two overlapping carriers), and the C-channel check above holds with it
    assert all(c["ddc_clipped"] == 0 for c in st["carriers"] if c["mode"] != "oqpsk8400")
    su = [e for e in ev if e["kind"] == "su"]
    assert su and all(len(e["su"]) == 12 for e in su)


def test_same_as_the_stages_wired_by_hand(cs16_stream, cs16_run):
    """The plan and every decoded unit equal what the existing stages give when wired by hand: scanner, find_carriers,
    probe_carriers and channel_plan on the first ACQUIRE seconds, then per mode a Ddc, DemodBatch and frame layer fed the same
    0.1 s blocks from the start of the stream, ticked once per second of signal."""
    import torch
    import jaero_b200
    iq, _ = cs16_stream
    ev, carriers, _, st = cs16_run
    fs, fmt, block = 2.4e6, "cs16", 240_000
    L, M = jaero_b200.rate_ratio(fs)
    stream = torch.cuda.Stream()
    dev = torch.from_numpy(iq).cuda()
    torch.cuda.synchronize()
    n, acq = iq.size // 2, int(ACQUIRE * fs)
    sc = jaero_b200.Scanner(fs, 1 << 16)
    sc.set_stream(stream.cuda_stream)
    for a in range(0, acq, block):
        sc.write_device(dev.data_ptr() + 4 * a, min(block, acq - a), fmt)
    mean, _, _ = sc.read()
    sc.close()
    probed = jaero_b200.probe_carriers(jaero_b200.find_carriers(mean, fs), fs, (dev.data_ptr(), acq), fmt, interpolation=L,
                                       decimation=M, stream=stream.cuda_stream)
    plans, _ = jaero_b200.channel_plan(probed, fs, M, L)
    groups, order = [], sorted(plans, key=lambda m: plans[m]["carriers"][0]["center_hz"])
    for mode in order:
        p = plans[mode]
        d, b = jaero_b200.Ddc(**p["ddc"]), jaero_b200.DemodBatch(**p["demod"])
        d.set_stream(stream.cuda_stream); b.set_stream(stream.cuda_stream)
        layer = jaero_b200.CChannelBatch(b.n) if mode == "oqpsk8400" else jaero_b200.PChannelBatch(b.n, p["demod"]["fb"])
        groups.append((mode, d, b, layer))
    mine = [(m, c["center_hz"]) for m in order for c in plans[m]["carriers"]]
    assert mine == [(c["mode"], c["center_hz"]) for c in carriers]
    sus = [[] for _ in carriers]
    frames = [[] for _ in carriers]
    ticks = 0
    for a in range(0, n, block):
        m = min(block, n - a)
        for mode, d, b, layer in groups:
            d.write_device(dev.data_ptr() + 4 * a, m, fmt)
            b.write_device(*d.output())
            layer.process_batch(b)
        while (a + m) // int(fs) > ticks:
            for _, _, b, layer in groups:
                layer.tick(b)
            ticks += 1
        first = 0
        for mode, d, b, layer in groups:
            if mode == "oqpsk8400":
                for ch, (su, ok, voice, fr) in enumerate(layer.read_frames()):
                    frames[first + ch] += [([x.tobytes() for x in su[k]], [bool(o) for o in ok[k]], voice[k].tobytes(), int(fr[k]))
                                           for k in range(len(fr))]
            else:
                for ch, (su, ok, idx, fr) in enumerate(layer.read_sus()):
                    sus[first + ch] += [(su[k].tobytes(), int(ok[k]), int(idx[k]), int(fr[k])) for k in range(len(ok))]
            first += b.n
    for _, d, b, layer in groups:
        d.close(); b.close(); layer.close()
    del dev
    rx_sus = [[] for _ in carriers]
    rx_frames = [[] for _ in carriers]
    for e in ev:
        if e["kind"] == "su":
            rx_sus[e["carrier"]].append((e["su"], 1, e["index"], e["frame"]))
        elif e["kind"] == "cframe":
            rx_frames[e["carrier"]].append((e["sus"], e["crc_ok"], e["voice"], e["frame"]))
    for c in range(len(carriers)):
        assert rx_sus[c] == [s for s in sus[c] if s[1]], c
        assert st["carriers"][c]["sus"] == len(sus[c]) + 3 * len(frames[c])
        assert st["carriers"][c]["crc_failures"] == sum(1 for s in sus[c] if not s[1]) + sum(3 - sum(f[1]) for f in frames[c])
        assert rx_frames[c] == frames[c], c
    assert sum(len(s) for s in sus) > 0 and sum(len(f) for f in frames) > 0


def test_rational_rate_known_answer():
    iq, msgs = _stream(2.5e6, "cu8")
    ev, carriers, unplanned, st = _run(iq, 2.5e6, "cu8", emit_sus=False)
    print("carriers:", [(c["mode"], round(c["center_hz"], 1)) for c in carriers], "unplanned:", len(unplanned))
    _check_known_answer(ev, carriers, msgs, "2.5 MS/s cu8")
    assert not [e for e in ev if e["kind"] == "su"]


def test_block_sizes_give_the_same_messages(cs16_stream, cs16_run):
    """0.05, 0.1 and 0.37 s blocks decode the same ACARS messages. The signal units themselves may differ: the P-channel layer
    applies DCD per call (DESIGN.md section 8), so a different call pattern can change soft bits near a DCD change."""
    iq, _ = cs16_stream
    ref = _acars(cs16_run[0])
    assert ref
    for block in (0.05, 0.37):
        ev, _, _, st = _run(iq, 2.4e6, "cs16", block=block, pieces=(0.9, 2.05), emit_sus=False)
        assert _acars(ev) == ref, block
        assert abs(st["seconds"] - SECONDS) < 1e-9


def test_nothing_to_decode():
    import jaero_b200
    rng = np.random.default_rng(5)
    fs = 2.4e6
    iq = np.clip(np.round(rng.standard_normal(2 * int(5 * fs)) * 0.25 * 32768 / np.sqrt(2)), -32768, 32767).astype(np.int16)
    with jaero_b200.Receiver(fs, "cs16", acquire_seconds=ACQUIRE) as rx:
        ev = []
        for a in range(0, iq.size, 2 * 300_000):
            ev += rx.write(iq[a:a + 2 * 300_000])
        ev += rx.flush()
        assert ev == []
        assert rx.acquired
        assert all(c["mode"] == "unknown" for c in rx.carriers())
        assert all(c["reason"] == "unknown mode" for c in rx.unplanned())
        assert rx.stats()["seconds"] == pytest.approx(5.0)


def test_a_burst_carrier_does_no_harm(cs16_run):
    iq, _ = _stream(2.4e6, "cs16", burst=True)
    ev, carriers, unplanned, _ = _run(iq, 2.4e6, "cs16", emit_sus=False)
    near = [(c["mode"], round(c["center_hz"], 1)) for c in carriers if abs(c["center_hz"] - BURST_OFFSET) < 10e3]
    left = [(c["mode"], round(c["center_hz"], 1), c["reason"]) for c in unplanned if abs(c["center_hz"] - BURST_OFFSET) < 10e3]
    print("burst carrier: planned as %s, unplanned as %s" % (near, left))
    ref_carriers = cs16_run[1]
    key = lambda c: (c["mode"], round(c["center_hz"]))
    ref = {key(c): c["index"] for c in ref_carriers}
    got = {key(c): c["index"] for c in carriers}
    mapped = sorted((ref[key(carriers[e[0]])],) + e[1:] for e in _acars(ev) if key(carriers[e[0]]) in ref)
    assert set(ref) <= set(got)
    assert mapped == _acars(cs16_run[0])


def test_cli_prints_the_objects_events(tmp_path, cs16_stream, cs16_run):
    """tools/receive.py on the stream written as a raw cs16 file prints the receiver's events (signal units not asked for) as
    JSON lines, exits 0 and reports the same plan"""
    import jaero_b200.receiver as rcv
    iq, _ = cs16_stream
    ev, carriers, _, _ = cs16_run
    path = tmp_path / "band.cs16"
    iq.astype("<i2").tofile(path)
    want = [json.loads(json.dumps(rcv.jsonable(e))) for e in ev if e["kind"] != "su"]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "receive.py"), "--rate", "2400000", "--format", "cs16",
                        str(path)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    got = [json.loads(line) for line in r.stdout.splitlines()]
    assert got == want
    report = json.loads(r.stderr[r.stderr.index("{"):])
    assert [(c["mode"], c["center_hz"]) for c in report["carriers"]] == [(c["mode"], c["center_hz"]) for c in carriers]
    assert report["stats"]["blocks"] == 120
