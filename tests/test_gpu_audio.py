"""AudioDecoder end to end on the GPU: the reference's 44.1 kHz recording against the oracle's signal units, the 48 kHz
excerpts against the same stages wired by hand, identification of every continuous excerpt, synthetic recordings of known
ACARS messages cut into segments at 48 and 44.1 kHz, recordings decoded together against each alone, and the CLI."""
import hashlib
import json
import os
import subprocess
import sys
import wave
from collections import Counter

import numpy as np
import pytest

import ident_reference as iref
import reasm_synth
from conftest import ROOT, load_excerpt

pytestmark = pytest.mark.gpu

GOLD = os.path.join(ROOT, "tests", "golden")
# the continuous 48 kHz excerpts: (fixture, mode, the freq_center their fixtures are decoded with)
EXCERPTS = [("oqpsk_10500", "oqpsk10500", 5760.0), ("oqpsk_8400", "oqpsk8400", 8000.0), ("msk_600", "msk600", 1000.0),
            ("msk_1200", "msk1200", 2000.0)]
MODE = {600: "msk600", 1200: "msk1200", 10500: "oqpsk10500"}
CENTER = {600: 1500.0, 1200: 2400.0, 10500: 7000.0}
# synthetic recordings: (bit rate, seconds, seed); none is a whole number of 10 s segments
SYNTH = [(600, 37, 0), (1200, 61, 1), (10500, 23, 2)]


def _decode(recs, rate=48000, **kw):
    import jaero_b200
    with jaero_b200.AudioDecoder(rate, emit_sus=True, **kw) as dec:
        ev = dec.decode(recs)
        return ev, dec.carriers(), dec.unplanned(), dec.stats()


def _chain(pcm, mode, center):
    """one DemodBatch channel (CHANNEL_SETTINGS, AFC on) and its frame layer, fed the recording zero-padded to whole 0.1 s
    blocks, ticked every whole second, read every block -> the events AudioDecoder forms, carrier 0"""
    import jaero_b200
    s = jaero_b200.CHANNEL_SETTINGS[mode]
    m = 4800
    x = np.zeros(-(-len(pcm) // m) * m, dtype=np.int16)
    x[:len(pcm)] = pcm
    b = jaero_b200.DemodBatch(s["kind"], 1, fb=s["fb"], freq_center=center, lockingbw=s["lockingbw"], afc=True)
    p = mode != "oqpsk8400"
    layer = jaero_b200.PChannelBatch(1, s["fb"]) if p else jaero_b200.CChannelBatch(1)
    rs = jaero_b200.Reassembler() if p else None
    ev = []
    base = dict(carrier=0, center_hz=float(center), mode=mode)
    for j in range(len(x) // m):
        b.write(x[None, j * m:(j + 1) * m])
        layer.process_batch(b)
        if (j + 1) % 10 == 0:
            layer.tick(b)
        t = min((j + 1) * m, len(pcm)) / 48000
        if p:
            su, ok, idx, frame = layer.read_sus()[0]
            for k in np.flatnonzero(ok):
                ev.append(dict(kind="su", input_seconds=t, su=su[k].tobytes(), index=int(idx[k]), frame=int(frame[k]), **base))
                rs.push_su(su[k].tobytes())
            for rec in rs.pop_all():
                rec["record_kind"], rec["acars_mode"] = rec.pop("kind"), rec.pop("mode")
                ev.append(dict(kind="acars", input_seconds=t, **base, **rec))
        else:
            for su, ok, voice, frame in zip(*layer.read_frames()[0]):
                ev.append(dict(kind="cframe", input_seconds=t, sus=[u.tobytes() for u in su], crc_ok=[bool(o) for o in ok],
                               voice=voice.tobytes(), frame=int(frame), **base))
    for o in (b, layer, rs):
        if o is not None:
            o.close()
    return [{k: e[k] for k in sorted(e)} for e in ev]


def _of(ev, c, drop_carrier=True):
    return [{k: v for k, v in sorted(e.items()) if not (drop_carrier and k == "carrier")} for e in ev if e["carrier"] == c]


def _acars(ev, c):
    return [(e["aesid"], e["reg"].decode("latin-1").strip("."), e["label"].decode("latin-1"), e["text"].decode("latin-1"))
            for e in ev if e["kind"] == "acars" and e["record_kind"] == 0 and e["carrier"] == c]


def _units(ev, c):
    return [e["su"] for e in ev if e["kind"] == "su" and e["carrier"] == c]


def _synth(fb, seconds, seed, rate=48000):
    """a recording of known ACARS messages: P-channel frames of fill around messages that fill every frame between -> (PCM
    at rate, messages)"""
    from jaero_b200 import synth
    fp = synth.frame_params(fb)
    k = fp["blocks"] * 64 * fp["cols"] // 2 // 96
    frames = -(-int(seconds * fb) // fp["frame_bits"]) + 1
    rng = np.random.default_rng(3000 + seed)
    lead = -(-8 * fb // fp["frame_bits"])                           # 8 s of fill first: the first segment starts cold
    tail = max(2, -(-2 * fb // fp["frame_bits"]))
    sus, msgs = [], []
    while True:
        aes = 0x300000 * (seed + 1) + len(msgs)
        reg = "A%d%03dZ" % (seed, len(msgs))
        label = "".join("HQ15AB_"[x] for x in rng.integers(0, 7, 2))
        text = "R%d M%d %s" % (seed, len(msgs), "".join("ABCDEFGHIJ"[x] for x in rng.integers(0, 10, int(rng.integers(2, 30)))))
        s = reasm_synth.isu_to_sus(aes, 0x90, len(msgs) & 15, 3,
                                   reasm_synth.acars_userdata(reg, label, ord("A") + len(msgs) % 26, text))
        if len(sus) + len(s) > (frames - lead - tail - 2) * k:
            break
        sus += s
        msgs.append((aes, reg, label, text))
    units = [synth.FILL_SU] * (lead * k) + sus
    units += [synth.FILL_SU] * (frames * k - len(units))
    msk = fb != 10500
    bits = synth.pchannel_bits_from_sus(fb, units, loop=msk, even_parity=msk)
    env = synth.msk_envelope(bits, fb) if msk else synth.oqpsk_envelope(bits, fb)
    env = env[:seconds * 48000]
    pcm = synth.to_passband_int16(env, CENTER[fb], ebn0_db=10.0, fb=float(fb), rng=np.random.default_rng(77 + seed))
    return _at(pcm, rate), msgs


def _at(pcm, rate):
    if rate == 48000:
        return pcm
    from fractions import Fraction
    from scipy.signal import resample_poly
    q = Fraction(rate, 48000)
    y = resample_poly(pcm.astype(np.float64), q.numerator, q.denominator)
    return np.clip(np.round(y), -32768, 32767).astype(np.int16)


@pytest.fixture(scope="module")
def synthetic():
    return [_synth(fb, sec, seed) for fb, sec, seed in SYNTH]


# ------------------------------------------------------------------------------------------------------ 1. oracle anchor
def test_44k1_recording_gives_the_oracles_signal_units():
    want = json.load(open(os.path.join(GOLD, "native_rate_outputs.json")))["oqpsk_10500_44k1"]
    ev, carriers, unplanned, st = _decode([load_excerpt("oqpsk_10500_44k1")], 44100, modes="oqpsk10500", centers_hz=5760,
                                          segment_seconds=60)
    got = [e["su"].hex() for e in ev if e["kind"] == "su"]
    assert len(got) == want["n_su_crc_ok"]
    assert hashlib.sha256(json.dumps(got).encode()).hexdigest() == want["su_crc_ok_sha256"]
    assert not unplanned and carriers[0]["mode_given"] and carriers[0]["center_given"] and carriers[0]["ident_score_db"] is None
    assert st["recordings"] == [dict(index=0, seconds=12.0, resample_clipped=want["resampled_clipped"])]
    assert st["groups"][0]["chunks"] == 1 and st["groups"][0]["batch_width"] == 1


# ------------------------------------------------------------------------------------------------------ 2. hand-wired chain
def test_excerpts_give_the_hand_wired_chains_events():
    pcms = [load_excerpt(name) for name, _, _ in EXCERPTS]
    ev, carriers, _, st = _decode(pcms, modes=[m for _, m, _ in EXCERPTS], centers_hz=[c for _, _, c in EXCERPTS],
                                  segment_seconds=60)
    assert [(c["index"], c["mode"], c["center_hz"]) for c in carriers] == [(i, m, c) for i, (_, m, c) in enumerate(EXCERPTS)]
    for i, (name, mode, center) in enumerate(EXCERPTS):
        want = [dict(e) for e in _chain(pcms[i], mode, center)]
        got = _of(ev, i, drop_carrier=False)
        for e in want:
            e["carrier"] = i
        print(name, len(got), "events", {k: sum(e["kind"] == k for e in got) for k in ("su", "acars", "cframe")})
        assert got == [{k: e[k] for k in sorted(e)} for e in want], name
        assert got, name
    assert ev == sorted(ev, key=lambda e: (e["input_seconds"], e["carrier"]))
    assert [r["seconds"] for r in st["recordings"]] == [len(p) / 48000 for p in pcms]


def test_decode_runs_once():
    import jaero_b200
    with jaero_b200.AudioDecoder(48000, modes="msk1200", centers_hz=2000) as dec:
        dec.decode([load_excerpt("msk_1200")])
        with pytest.raises(ValueError, match="already called"):
            dec.decode([load_excerpt("msk_1200")])


# ------------------------------------------------------------------------------------------------------ 3. identification
def test_identification_of_every_continuous_excerpt_and_of_noise():
    """the excerpts together, each identified from all of it (identify_seconds covers the longest, as the identifier's own test
    averages them), and 6 s of noise"""
    rng = np.random.default_rng(11)
    noise = np.clip(np.round(rng.standard_normal(6 * 48000) * 3000), -32768, 32767).astype(np.int16)
    pcms = [load_excerpt(name) for name, _, _ in EXCERPTS] + [noise]
    ev, carriers, unplanned, _ = _decode(pcms, identify_seconds=20, segment_seconds=60)
    ref = {e[0]: e[3] for e in iref.EXCERPTS}
    got = {c["index"]: c for c in carriers}
    for i, (name, mode, _) in enumerate(EXCERPTS):
        c = got[i]
        print(name, c["mode"], "%.2f Hz" % c["center_hz"], "%.1f dB margin" % c["ident_margin_db"])
        assert c["mode"] == mode and not c["mode_given"] and not c["center_given"], c
        assert min(abs(c["center_hz"] - f) for f in ref[name]) <= 2.0, c
    assert [(u["index"], u["reason"]) for u in unplanned] == [(len(EXCERPTS), "unknown mode")]
    assert not [e for e in ev if e["carrier"] == len(EXCERPTS)]
    assert any(e["kind"] == "su" for e in ev)


# ------------------------------------------------------------------------------------------------------ 4. segments
@pytest.mark.parametrize("rate", [48000, 44100])
def test_segments_give_every_message_once(synthetic, rate):
    recs = [_at(pcm, rate) for pcm, _ in synthetic]
    kw = dict(modes=[MODE[fb] for fb, _, _ in SYNTH], centers_hz=[CENTER[fb] for fb, _, _ in SYNTH])
    ev, _, _, st = _decode(recs, rate, segment_seconds=10, **kw)
    one, _, _, _ = _decode(recs, rate, segment_seconds=100, **kw)
    print("segments at %d Hz:" % rate, json.dumps(st["groups"]))
    print("per recording:", [(c["mode"], c["boundary_matches"], c["unmatched"], c["late_locks"], c["lock_seconds"])
                             for c in st["carriers"]])
    for i, (_, msgs) in enumerate(synthetic):
        assert _acars(ev, i) == msgs, i
        assert _units(ev, i) == _units(one, i) and _units(ev, i), i
    assert all(g["segments_per_chunk"] > 1 and g["chunks"] == 1 for g in st["groups"])
    assert all(c["late_locks"] == 0 and c["unlocked_segments"] == 0 for c in st["carriers"]), st["carriers"]
    assert sum(c["boundary_matches"] for c in st["carriers"]) > 0


def test_22050_recordings_give_every_message_once(synthetic):
    """22050 Hz, an ordinary WAV rate whose ratio to 48 kHz (320/147) only the rate converter allows: the 600 and 1200 bps
    recordings (10.5 kbps does not fit below its 11 025 Hz Nyquist frequency)"""
    recs = [_at(pcm, 22050) for pcm, _ in synthetic[:2]]
    kw = dict(modes=[MODE[fb] for fb, _, _ in SYNTH[:2]], centers_hz=[CENTER[fb] for fb, _, _ in SYNTH[:2]])
    ev, _, _, st = _decode(recs, 22050, segment_seconds=10, **kw)
    one, _, _, _ = _decode(recs, 22050, segment_seconds=100, **kw)
    for i, (_, msgs) in enumerate(synthetic[:2]):
        assert _acars(ev, i) == msgs, i
        assert _units(ev, i) == _units(one, i) and _units(ev, i), i
    assert [r["seconds"] for r in st["recordings"]] == [37.0, 61.0]
    assert all(c["late_locks"] == 0 and c["unlocked_segments"] == 0 for c in st["carriers"]), st["carriers"]


def test_reading_stops_at_the_last_decoded_recording(synthetic):
    """a long recording of noise next to a short decodable one: the noise is left undecoded, and the rate converter is fed
    only the identification window and up to the short recording's end, not to the noise's end"""
    rng = np.random.default_rng(12)
    noise = np.clip(np.round(rng.standard_normal(300 * 44100) * 3000), -32768, 32767).astype(np.int16)
    short = _at(synthetic[2][0], 44100)
    ev, carriers, unplanned, st = _decode([noise, short], 44100, segment_seconds=10)
    assert [c["index"] for c in carriers] == [1] and [(u["index"], u["reason"]) for u in unplanned] == [(0, "unknown mode")]
    assert _acars(ev, 1) == synthetic[2][1] and not _of(ev, 0)
    assert st["recordings"][0]["seconds"] == 300.0 and st["read_seconds"] == 23


@pytest.mark.parametrize("rate", [48000, 44100])
def test_8400_recording_in_short_segments_reports_only_frames_of_its_one_segment_run(rate):
    pcm = _at(load_excerpt("oqpsk_8400"), rate)
    kw = dict(modes="oqpsk8400", centers_hz=8000.0)
    ev, _, _, st = _decode([pcm], rate, segment_seconds=5, lead_seconds=2, **kw)
    one, _, _, _ = _decode([pcm], rate, segment_seconds=60, **kw)
    frames = lambda e: [(tuple(x["sus"]), tuple(x["crc_ok"])) for x in e if x["kind"] == "cframe" and any(x["crc_ok"])]
    got, want = frames(ev), frames(one)
    print("8400 bps at %d Hz: %d frames with a CRC-valid unit, one segment %d" % (rate, len(got), len(want)), st["carriers"])
    assert st["groups"][0]["segments_per_chunk"] > 1
    assert got and not Counter(got) - Counter(want)             # no frame more often than the one-segment run has it


# ------------------------------------------------------------------------------------------------------ 5. independence
@pytest.mark.parametrize("max_channels", [4096, 8])
def test_recordings_together_give_what_each_gives_alone(synthetic, max_channels):
    """three 10.5 kbps and three 600 bps recordings of different lengths, with one 1200 and one 8400 bps excerpt. With 8
    channels a batch holds two segments of each of the three recordings of a group, so the 10.5 kbps and 600 bps groups take
    several chunks"""
    longer = np.concatenate([synthetic[2][0], synthetic[2][0]])[:37 * 48000 + 1234]    # not a whole block
    recs = [synthetic[2][0], load_excerpt("msk_1200"), synthetic[0][0], longer, load_excerpt("oqpsk_8400"),
            load_excerpt("oqpsk_10500"), load_excerpt("msk_600"), synthetic[0][0][:29 * 48000 + 77]]
    modes = ["oqpsk10500", "msk1200", "msk600", "oqpsk10500", "oqpsk8400", "oqpsk10500", "msk600", "msk600"]
    centers = [CENTER[10500], 2000.0, CENTER[600], CENTER[10500], 8000.0, 5760.0, 1000.0, CENTER[600]]
    ev, _, _, st = _decode(recs, segment_seconds=10, modes=modes, centers_hz=centers, max_channels=max_channels)
    print("groups with max_channels=%d:" % max_channels, json.dumps(st["groups"]))
    if max_channels == 8:
        assert all(g["chunks"] > 1 for g in st["groups"] if g["carriers"] == 3), st["groups"]
    for i in range(len(recs)):
        alone, _, _, _ = _decode([recs[i]], segment_seconds=10, modes=modes[i], centers_hz=centers[i])
        assert _of(ev, i) == _of(alone, 0), i
        assert _of(ev, i), i


# ------------------------------------------------------------------------------------------------------ 6. CLI
def test_cli_prints_the_objects_events(tmp_path, synthetic):
    import jaero_b200.receiver as rcv
    pcm = synthetic[1][0][:30 * 48000]
    path = tmp_path / "rec.wav"
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1); w.setsampwidth(2); w.setframerate(48000)
        w.writeframes(pcm.astype("<i2").tobytes())
    ev, _, _, _ = _decode([pcm], modes="msk1200", centers_hz=CENTER[1200])
    want = [json.loads(json.dumps(dict(rcv.jsonable(e), file=str(path)))) for e in ev]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "decode_audio.py"), "--mode", "msk1200", "--center",
                        str(CENTER[1200]), "--sus", str(path)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    got = [json.loads(line) for line in r.stdout.splitlines()]
    assert got == want and any(e["kind"] == "acars" for e in got)
    report = json.loads(r.stderr[r.stderr.index("{"):])
    assert report["sample_rate"] == 48000 and report["carriers"][0]["file"] == str(path) and report["stats"]["groups"]
