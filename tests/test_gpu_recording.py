"""RecordingDecoder end to end on the GPU: a 48 s band at 1.2 MS/s with P-channel carriers at 600, 1200 and 10 500 bps whose
known ACARS messages run across every segment boundary, and the 8400 bps recording placed across a boundary on a carrier of
random 8400 bps bits; decoded as parallel segments and compared with the known messages and with one Receiver."""
import json
import os
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest

import reasm_synth
from conftest import ROOT, load_excerpt
from test_gpu_receiver import _acars, _analytic

pytestmark = pytest.mark.gpu

FS, FMT = 1.2e6, "cs16"
SECONDS = 48.0
EBN0_DB = 10.0
BLOCK = 0.1
# (fb, offset Hz, lead-in frames of fill, tail frames of fill): messages fill every frame between, so they run across every
# segment boundary of both segment lengths below
P_CARRIERS = [(600, -420_000.0, 2, 2), (1200, -170_000.0, 3, 2), (10500, 160_000.0, 8, 3)]
C_OFFSET = 410_000.0
MODE = {600: "msk600", 1200: "msk1200", 10500: "oqpsk10500"}
SEGMENTS = (7, 10)             # neither divides the other


def _c_start():
    """where the 8400 bps recording starts: its 8 s hold the first boundary of 10 s segments (10 + lead) and, being longer than
    7 s, a boundary of 7 s segments"""
    from jaero_b200.recording import DEFAULT_LEAD_SECONDS
    return 6 + DEFAULT_LEAD_SECONDS["oqpsk8400"]


def _carrier(i, fb, lead, tail):
    from jaero_b200 import synth
    fp = synth.frame_params(fb)
    k = fp["blocks"] * 64 * fp["cols"] // 2 // 96
    frames = int(SECONDS * fb) // fp["frame_bits"]
    rng = np.random.default_rng(2000 + i)
    sus, msgs = [], []
    while True:
        aes = 0x200000 * (i + 1) + len(msgs)
        reg = "R%d%03dQ" % (i, len(msgs))
        label = "".join("HQ15AB_"[x] for x in rng.integers(0, 7, 2))
        text = "S%d M%d %s" % (i, len(msgs), "".join("ABCDEFGHIJ"[x] for x in rng.integers(0, 10, int(rng.integers(2, 30)))))
        s = reasm_synth.isu_to_sus(aes, 0x90, len(msgs) & 15, 3, reasm_synth.acars_userdata(reg, label, ord("A") + len(msgs) % 26,
                                                                                             text))
        if len(sus) + len(s) > (frames - lead - tail) * k:
            break
        sus += s
        msgs.append((aes, reg, label, text))
    units = [synth.FILL_SU] * (lead * k) + sus
    units += [synth.FILL_SU] * (frames * k - len(units))
    msk = fb != 10500
    bits = synth.pchannel_bits_from_sus(fb, units, loop=msk, even_parity=msk)
    env = synth.msk_envelope(bits, fb) if msk else synth.oqpsk_envelope(bits, fb)
    assert len(env) == int(SECONDS * 48000)
    return env, msgs


def _unit(x):
    return x / np.sqrt(np.mean(np.abs(x) ** 2))


@pytest.fixture(scope="module")
def band():
    from jaero_b200 import synth
    envs, offs, fbs, msgs = [], [], [], []
    for i, (fb, off, lead, tail) in enumerate(P_CARRIERS):
        e, m = _carrier(i, fb, lead, tail)
        envs.append(e); offs.append(off); fbs.append(float(fb)); msgs.append(m)
    rec = _unit(_analytic(load_excerpt("oqpsk_8400"), 300.0, 13000.0, 8000.0))
    a = int(_c_start() * 48000)
    rnd = lambda n, seed: _unit(synth.oqpsk_envelope(np.random.default_rng(seed).integers(0, 2, (n * 8400 // 48000 // 14 + 2) * 14)
                                                     .astype(np.uint8), 8400))[:n]
    tail = int(SECONDS * 48000) - a - len(rec)
    envs.append(np.concatenate([rnd(a, 5), rec, rnd(tail, 6)])); offs.append(C_OFFSET); fbs.append(8400.0)
    iq = synth.wideband_iq(envs, offs, FS, [EBN0_DB] * 3 + [20.0], fmt=FMT, seed=91, fb=fbs)
    return iq, msgs


def _write_all(rx, iq, pieces=(1.7, 0.23, 3.1)):
    n, ev, a, k = iq.size // 2, [], 0, 0
    while a < n:
        m = min(n - a, int(pieces[k % len(pieces)] * FS)); k += 1
        ev += rx.write(iq[2 * a:2 * (a + m)])
        a += m
    return ev + rx.flush()


def _decode(iq, **kw):
    import jaero_b200
    with jaero_b200.RecordingDecoder(FS, FMT, emit_sus=True, **kw) as rx:
        ev = _write_all(rx, iq)
        return ev, rx.carriers(), rx.stats()


@pytest.fixture(scope="module")
def receiver_run(band):
    import jaero_b200
    iq, _ = band
    with jaero_b200.Receiver(FS, FMT, emit_sus=True) as rx:
        ev = _write_all(rx, iq)
        return ev, rx.carriers(), rx.stats()


def _sent(carriers, msgs):
    idx = {c["index"]: int(np.argmin([abs(c["center_hz"] - off) for _, off, _, _ in P_CARRIERS]))
           for c in carriers if c["mode"] != "oqpsk8400"}
    return sorted((ci, aes, reg, label, text) for ci, i in idx.items() for aes, reg, label, text in msgs[i])


def _no_late_locks(st):
    """every P-channel segment locks before its stretch begins. The 8400 bps recording starts inside one segment's stretch,
    after random bits that carry no frame, so that one segment's first CRC-valid frame comes after its stretch began, and the
    segments over the random bits alone give no CRC-valid frame; no other may"""
    for c in st["carriers"]:
        assert c["late_locks"] <= (c["mode"] == "oqpsk8400"), c
        assert c["unlocked_segments"] == 0 or c["mode"] == "oqpsk8400", c


def _by_carrier(ev, kind):
    out = {}
    for e in ev:
        if e["kind"] == kind:
            out.setdefault(e["carrier"], []).append(e)
    return out


def test_the_band_plans_every_carrier(receiver_run):
    _, carriers, _ = receiver_run
    assert sorted(c["mode"] for c in carriers) == sorted([MODE[fb] for fb, *_ in P_CARRIERS] + ["oqpsk8400"])


def test_one_segment_is_the_receiver(band, receiver_run):
    """segments longer than the recording: one per carrier, each run from the start like Receiver's channel -> the same events,
    carriers and counts"""
    iq, _ = band
    ev, carriers, st = _decode(iq, segment_seconds=60)
    rev, rcarriers, rst = receiver_run
    assert carriers == rcarriers
    assert len(ev) == len(rev)
    assert ev == rev
    keys = ("carrier", "mode", "center_hz", "sus", "crc_failures", "messages", "cframes", "ddc_clipped")
    assert [{k: c[k] for k in keys} for c in st["carriers"]] == [{k: c[k] for k in keys} for c in rst["carriers"]]
    assert st["blocks"] == rst["blocks"] and st["seconds"] == rst["seconds"]
    assert all(g["segments_per_chunk"] == 4096 and g["chunks"] == 1 and g["batch_width"] == g["carriers"] for g in st["groups"])
    print("time to the first CRC-valid frame from a cold start:",
          {c["mode"]: c["lock_seconds"] for c in st["carriers"]})


@pytest.fixture(scope="module", params=SEGMENTS)
def segmented(request, band):
    iq, _ = band
    return request.param, _decode(iq, segment_seconds=request.param)


def test_segments_decode_what_the_receiver_decodes(band, receiver_run, segmented):
    seg, (ev, carriers, st) = segmented
    _, msgs = band
    rev, rcarriers, rst = receiver_run
    print("segments of %d s:" % seg, json.dumps(st["groups"]))
    print("per carrier:", [(c["mode"], c["boundary_matches"], c["unmatched"], c["late_locks"], c["lock_seconds"])
                           for c in st["carriers"]])
    assert [(c["mode"], c["center_hz"]) for c in carriers] == [(c["mode"], c["center_hz"]) for c in rcarriers]
    assert all(g["segments_per_chunk"] > 1 for g in st["groups"])
    # ACARS: the sent messages, and the receiver's
    assert _acars(ev) == _sent(carriers, msgs) == _acars(rev)
    # P-channel: per carrier the same CRC-valid units in the same order, each decoded within one block of the receiver
    got, want = _by_carrier(ev, "su"), _by_carrier(rev, "su")
    assert sorted(got) == sorted(want)
    for c in want:
        assert [e["su"] for e in got[c]] == [e["su"] for e in want[c]], c
        assert max(abs(a["input_seconds"] - b["input_seconds"]) for a, b in zip(got[c], want[c])) <= BLOCK + 1e-9, c
    for c in set(_by_carrier(rev, "acars")):
        a, b = _by_carrier(ev, "acars")[c], _by_carrier(rev, "acars")[c]
        assert [x["text"] for x in a] == [x["text"] for x in b]
        assert max(abs(x["input_seconds"] - y["input_seconds"]) for x, y in zip(a, b)) <= BLOCK + 1e-9, c
    _no_late_locks(st)
    assert sum(c["boundary_matches"] for c in st["carriers"]) > 0
    # C-channel: at least 90 % of the receiver's CRC-valid units, and no frame twice (frames are 0.49 s apart)
    cf, rcf = _by_carrier(ev, "cframe"), _by_carrier(rev, "cframe")
    units = Counter(s for c in cf for e in cf[c] for s, o in zip(e["sus"], e["crc_ok"]) if o)
    runits = Counter(s for c in rcf for e in rcf[c] for s, o in zip(e["sus"], e["crc_ok"]) if o)
    print("C-channel: %d CRC-valid units, the receiver %d" % (sum(units.values()), sum(runits.values())))
    assert runits and sum((units & runits).values()) >= 0.9 * sum(runits.values())
    for c in cf:
        t = np.array([e["input_seconds"] for e in cf[c]])
        assert np.all(np.diff(t) > 2 * BLOCK + 1e-9), c
    # every event's time is on the block grid and the list is ordered by time, then carrier
    assert ev == sorted(ev, key=lambda e: (e["input_seconds"], e["carrier"]))


def test_the_8400_recording_straddles_a_boundary():
    from jaero_b200.recording import layout
    a = _c_start()
    for seg in SEGMENTS:
        g = layout(FS, BLOCK, seg)["oqpsk8400"]
        assert any(a + 1 <= g.start(k) / g.per <= a + 7 for k in range(1, 10)), seg


def test_chunks_give_the_same_messages(band):
    """two channels per batch: two segments per chunk, so the recording takes several chunks per group"""
    iq, msgs = band
    ev, carriers, st = _decode(iq, segment_seconds=7, max_channels=2)
    assert all(g["chunks"] >= 3 and g["batch_width"] == 2 for g in st["groups"]), st["groups"]
    assert _acars(ev) == _sent(carriers, msgs)
    _no_late_locks(st)


def test_a_short_lead_is_reported_as_late_locks(band):
    """a 1 s lead, shorter than every P-channel mode's time to its first CRC-valid frame (2.6 s or more on this band): each
    P-channel carrier reports late locks (the default leads report none, above)"""
    iq, _ = band
    _, _, st = _decode(iq, segment_seconds=7, lead_seconds=1)
    late = {c["mode"]: c["late_locks"] for c in st["carriers"]}
    print("late locks with a 1 s lead:", late)
    assert all(v > 0 for m, v in late.items() if m != "oqpsk8400"), late


def test_a_recording_that_ends_inside_a_block(band):
    """0.04 s short of whole blocks: the last block is written in two parts where a segment's PCM ends in it, so the last
    segment ends where the recording ends. The signal units and messages are the receiver's on the same IQ"""
    import jaero_b200
    iq, msgs = band
    iq = iq[:iq.size - 2 * int(0.04 * FS)]
    with jaero_b200.Receiver(FS, FMT, emit_sus=True) as rx:
        rev = _write_all(rx, iq)
    ev, carriers, st = _decode(iq, segment_seconds=7)
    assert all(g["segments_per_chunk"] > 1 and g["pcm_bytes"] == 0 and g["pcm_bytes_peak"] > 0 for g in st["groups"])
    assert _acars(ev) == _acars(rev) and _acars(ev)
    got, want = _by_carrier(ev, "su"), _by_carrier(rev, "su")
    assert sorted(got) == sorted(want)
    for c in want:
        assert [e["su"] for e in got[c]] == [e["su"] for e in want[c]], c
    assert max(e["input_seconds"] for e in ev) <= st["seconds"] + 1e-9
    _no_late_locks(st)


def test_nothing_to_decode():
    import jaero_b200
    rng = np.random.default_rng(5)
    iq = np.clip(np.round(rng.standard_normal(2 * int(6 * FS)) * 0.25 * 32768 / np.sqrt(2)), -32768, 32767).astype(np.int16)
    with jaero_b200.RecordingDecoder(FS, FMT, segment_seconds=7) as rx:
        assert _write_all(rx, iq) == []
        assert rx.acquired and all(c["mode"] == "unknown" for c in rx.carriers())
        assert rx.stats()["seconds"] == pytest.approx(6.0)


def test_writes_after_flush_are_refused(band):
    import jaero_b200
    iq, _ = band
    with jaero_b200.RecordingDecoder(FS, FMT, segment_seconds=7) as rx:
        rx.write(iq[:2 * int(5 * FS)])
        rx.flush()
        assert rx.flush() == []
        with pytest.raises(ValueError, match="flushed"):
            rx.write(iq[:1000])


def test_cli_prints_the_objects_events(tmp_path, band):
    import jaero_b200
    import jaero_b200.receiver as rcv
    iq, _ = band
    with jaero_b200.RecordingDecoder(FS, FMT, segment_seconds=10) as rx:
        ev = _write_all(rx, iq)
        carriers = rx.carriers()
    path = tmp_path / "band.cs16"
    iq.astype("<i2").tofile(path)
    want = [json.loads(json.dumps(rcv.jsonable(e))) for e in ev]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "receive.py"), "--rate", "1200000", "--format", "cs16",
                        "--segment", "10", str(path)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    got = [json.loads(line) for line in r.stdout.splitlines()]
    assert got == want and any(e["kind"] == "acars" for e in got)
    report = json.loads(r.stderr[r.stderr.index("{"):])
    assert [(c["mode"], c["center_hz"]) for c in report["carriers"]] == [(c["mode"], c["center_hz"]) for c in carriers]
    assert report["stats"]["groups"] and report["stats"]["blocks"] == int(SECONDS / BLOCK)
