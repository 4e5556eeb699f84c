"""BurstAudioDecoder end to end on the GPU: the committed burst excerpts against the oracle's R/T packets, tiled recordings cut
into short segments against the straight one-channel chain, recordings of every burst mode decoded together against each
alone, identification of the burst rate, a 22 050 Hz recording through the rate converter, and the CLI."""
import hashlib
import json
import os
import subprocess
import sys
import wave

import numpy as np
import pytest

from conftest import ROOT, load_excerpt

pytestmark = pytest.mark.gpu

GOLD = os.path.join(ROOT, "tests", "golden")
# the committed burst excerpts: (fixture, mode, rate, golden file)
EXCERPTS = [("burst_msk_1200_a", "burst_msk1200", 48000, "expected_outputs.json"),
            ("burst_msk_1200_b", "burst_msk1200", 48000, "expected_outputs.json"),
            ("burst_oqpsk_10500", "burst_oqpsk10500", 48000, "expected_outputs.json"),
            ("burst_oqpsk_10500_44k1", "burst_oqpsk10500", 44100, "native_rate_outputs.json")]
FB = {"burst_msk600": 600, "burst_msk1200": 1200, "burst_oqpsk10500": 10500}


def _decode(recs, rate=48000, **kw):
    import jaero_b200
    with jaero_b200.BurstAudioDecoder(rate, emit_packets=True, **kw) as dec:
        ev = dec.decode(recs)
        return ev, dec.carriers(), dec.unplanned(), dec.stats()


def _chain(pcm, mode, rate=48000):
    """the straight chain: a Resampler at other rates than 48 kHz, one burst demodulator channel with the batch's defaults and
    its R/T layer, fed the recording zero-padded to whole 0.1 s blocks from device memory, ticked every whole second, read
    every block, packets to a Reassembler -> the events BurstAudioDecoder forms, carrier 0"""
    import torch
    import jaero_b200
    n = rate // 10
    x = np.zeros(-(-len(pcm) // n) * n, dtype=np.int16)
    x[:len(pcm)] = pcm
    dev = torch.from_numpy(x).cuda()
    torch.cuda.synchronize()
    rs = jaero_b200.Resampler(rate, 1) if rate != 48000 else None
    cls = jaero_b200.BurstOqpskBatch if mode == "burst_oqpsk10500" else jaero_b200.BurstMskBatch
    b = cls(1, fb=float(FB[mode]))
    rt = jaero_b200.RTChannelBatch(1, FB[mode])
    ra = jaero_b200.Reassembler()
    ev = []
    for j in range(len(x) // n):
        if rs is None:
            ptr, m = dev.data_ptr() + 2 * j * n, n
        else:
            rs.write_device(dev.data_ptr() + 2 * j * n, n, len(x))
            ptr, m, _ = rs.output()
            rs.read_pcm()                                        # the burst batch runs on its own stream
        b.write_device(ptr, m, m)
        rt.process_burst(b)
        if (j + 1) % 10 == 0:
            rt.tick()
        t = min((j + 1) * n, len(pcm)) / rate
        for q in rt.read_packets()[0]:
            info = q["bytes"].tobytes()
            ev.append(dict(kind="rtpacket", input_seconds=t, type="R" if q["type"] == 1 else "T", nsus=q["nsus"], bytes=info))
            if q["type"] == 1:
                ra.push_r(info, downlink=True)
            else:
                ra.push_t_packet(info, q["nsus"])
            for rec in ra.pop_all():
                rec["record_kind"], rec["acars_mode"] = rec.pop("kind"), rec.pop("mode")
                ev.append(dict(kind="acars", input_seconds=t, **rec))
    for o in (rs, b, rt, ra):
        if o is not None:
            o.close()
    return ev


def _of(ev, c):
    """recording c's events without the fields the chain does not form"""
    return [{k: v for k, v in e.items() if k not in ("carrier", "center_hz", "mode")} for e in ev if e["carrier"] == c]


def _packets(ev, c=None):
    return [(e["type"], e["nsus"], e["bytes"]) for e in ev if e["kind"] == "rtpacket" and (c is None or e["carrier"] == c)]


def _acars(ev, c=None):
    return [{k: v for k, v in e.items() if k not in ("carrier", "center_hz", "mode", "input_seconds")}
            for e in ev if e["kind"] == "acars" and (c is None or e["carrier"] == c)]


def _golden(name, fname):
    g = json.load(open(os.path.join(GOLD, fname)))[name]
    return g["rt_packets"]


def _summary(packets):
    return [dict(type={"R": 1, "T": 2}[k], nsus=n, n_bytes=len(b), sha256=hashlib.sha256(b).hexdigest()) for k, n, b in packets]


# ------------------------------------------------------------------------------------------------------ excerpts
@pytest.mark.parametrize("name, mode, rate, fname", EXCERPTS)
def test_each_excerpt_in_one_segment_gives_the_oracle_packets(name, mode, rate, fname):
    pcm = load_excerpt(name)
    ev, car, _, st = _decode([pcm], rate, modes=mode, segment_seconds=20)
    assert st["groups"][0]["segments"] == 1 and car[0]["mode"] == mode and car[0]["mode_given"]
    assert _summary(_packets(ev)) == _golden(name, fname)
    assert _of(ev, 0) == _chain(pcm, mode, rate)


# ------------------------------------------------------------------------------------------------------ segments
SEG = 5


def _tiled(name, mode, seconds=120, seed=0):
    """the excerpt repeated to about `seconds`, between gaps of noise at the excerpt's quietest level: every other copy placed so
    that its first packet is emitted within two blocks of a segment boundary, the others after a random gap"""
    import jaero_b200
    x = load_excerpt(name)
    geo = jaero_b200.BurstAudioDecoder(48000, segment_seconds=SEG).geometry[mode]
    first = _chain(x, mode)[0]["input_seconds"]                # end of the block that emits the excerpt's first packet
    rng = np.random.default_rng(100 + seed)
    sigma = min(np.std(x[a:a + 4800].astype(np.float64)) for a in range(0, len(x) - 4800, 4800))
    noise = lambda k: np.clip(np.round(rng.normal(0, sigma, k)), -32768, 32767).astype(np.int16)
    out, pos, k = [noise(48000)], 48000, 0
    while pos < seconds * 48000:
        if k % 2 == 0:
            g = 1
            while geo.start(g) * 4800 <= pos + first * 48000 + 48000:
                g += 1
            gap = int(geo.start(g) * 4800 - first * 48000 + 4800 - pos + rng.integers(-9600, 9600))
        else:
            gap = int(rng.integers(12000, 150000))
        out += [noise(gap), x]
        pos += gap + len(x)
        k += 1
    return np.concatenate(out)


@pytest.mark.parametrize("name, mode", [(n, m) for n, m, r, _ in EXCERPTS if r == 48000])
def test_a_tiled_recording_in_short_segments_equals_the_straight_chain(name, mode):
    pcm = _tiled(name, mode)
    want = _chain(pcm, mode)
    assert len(_packets(want)) >= 15
    ev, _, _, st = _decode([pcm], modes=mode, segment_seconds=SEG)
    assert _packets(ev) == _packets(want)
    assert _acars(ev) == _acars(want)
    assert [e["input_seconds"] for e in ev] == [e["input_seconds"] for e in want]
    c = st["carriers"][0]
    assert c["boundary_matches"] > 0 and c["packets"] == len(_packets(want)), st
    assert st["groups"][0]["chunks"] == 1 and st["groups"][0]["segments"] > 20
    # a few segments per chunk: several chunks, the same stream
    ev2, _, _, st2 = _decode([pcm], modes=mode, segment_seconds=SEG, max_channels=5)
    assert st2["groups"][0]["chunks"] > 3 and st2["groups"][0]["batch_width"] == 5
    assert _of(ev2, 0) == _of(ev, 0)
    assert st2["carriers"][0]["boundary_matches"] == c["boundary_matches"]


def test_bursts_within_the_carrier_detect_hold_across_boundaries_equal_the_straight_chain():
    """the excerpt tiled with gaps of 0.25 to 3 s, so a copy's first burst often comes within the R/T layer's 4 s carrier-detect
    hold of the previous copy's last sync, where the chain does not search for its unique word: the segments, which start a
    lead that covers that hold early, decide each such burst as the chain does, including the ones just after a boundary"""
    x = load_excerpt("burst_oqpsk_10500")
    rng = np.random.default_rng(21)
    sigma = min(np.std(x[a:a + 4800].astype(np.float64)) for a in range(0, len(x) - 4800, 4800))
    out = []
    while sum(len(o) for o in out) < 150 * 48000:
        out += [np.clip(np.round(rng.normal(0, sigma, int(rng.integers(12000, 144000)))), -32768, 32767).astype(np.int16), x]
    pcm = np.concatenate(out)
    want = _chain(pcm, "burst_oqpsk10500")
    ev, _, _, st = _decode([pcm], modes="burst_oqpsk10500", segment_seconds=SEG)
    assert _packets(ev) == _packets(want) and len(_packets(want)) >= 30
    assert _acars(ev) == _acars(want)
    assert [e["input_seconds"] for e in ev] == [e["input_seconds"] for e in want]


def _stretched_600(name):
    """a 1200 bps burst recording time-stretched 2x: the same bursts at 600 bps"""
    from scipy.signal import resample_poly
    y = resample_poly(load_excerpt(name).astype(np.float64), 2, 1)
    return np.clip(np.round(y), -32768, 32767).astype(np.int16)


def test_recordings_of_every_mode_together_give_what_each_gives_alone():
    recs = [(_tiled("burst_msk_1200_a", "burst_msk1200", 40, 1), "burst_msk1200"),
            (load_excerpt("burst_oqpsk_10500"), "burst_oqpsk10500"),
            (np.concatenate([_stretched_600("burst_msk_1200_a")] * 3), "burst_msk600"),
            (_tiled("burst_oqpsk_10500", "burst_oqpsk10500", 30, 2), "burst_oqpsk10500"),
            (_tiled("burst_msk_1200_b", "burst_msk1200", 25, 3), "burst_msk1200")]
    ev, car, _, st = _decode([r for r, _ in recs], modes=[m for _, m in recs], segment_seconds=SEG)
    assert [c["mode"] for c in car] == [m for _, m in recs]
    assert len(st["groups"]) == 3
    for c, (r, m) in enumerate(recs):
        alone, _, _, _ = _decode([r], modes=m, segment_seconds=SEG)
        assert _of(ev, c) == _of(alone, 0), c
        # the 2x-stretched 1200 bps excerpt gives no packets at 600 bps: its row checks only that the group runs alongside
        assert m == "burst_msk600" or len(_packets(alone)) > 0, c


# ------------------------------------------------------------------------------------------------------ identification
def test_each_excerpt_is_identified_at_its_burst_rate_and_noise_is_unplanned():
    names = [(n, m) for n, m, r, _ in EXCERPTS if r == 48000]
    noise = np.random.default_rng(5).normal(0, 300, 10 * 48000).astype(np.int16)
    ev, car, unplanned, st = _decode([load_excerpt(n) for n, _ in names] + [noise])
    assert [(c["index"], c["mode"], c["mode_given"]) for c in car] == [(i, m, False) for i, (_, m) in enumerate(names)]
    assert [(u["index"], u["reason"]) for u in unplanned] == [(len(names), "unknown mode")]
    for i, (n, _) in enumerate(names):
        assert _summary(_packets(ev, i)) == _golden(n, "expected_outputs.json")


# ------------------------------------------------------------------------------------------------------ other rates
def test_a_22050_hz_recording_equals_the_chain_with_a_rate_converter():
    from scipy.signal import resample_poly
    # the 1200 bps excerpt: its carrier (1831 Hz) lies well below 11 025 Hz, the 10.5 kbps one (11 173 Hz) does not
    x = resample_poly(load_excerpt("burst_msk_1200_a").astype(np.float64), 147, 320)
    pcm = np.clip(np.round(x), -32768, 32767).astype(np.int16)
    want = _chain(pcm, "burst_msk1200", 22050)
    assert len(_packets(want)) >= 1
    ev, _, _, st = _decode([pcm], 22050, modes="burst_msk1200", segment_seconds=20)
    assert _of(ev, 0) == want
    assert st["recordings"][0]["resample_clipped"] == 0


# ------------------------------------------------------------------------------------------------------ CLI
def test_the_cli_prints_the_object_s_events(tmp_path):
    from jaero_b200.receiver import jsonable
    a = load_excerpt("burst_msk_1200_a")
    b = load_excerpt("burst_oqpsk_10500_44k1")
    with wave.open(str(tmp_path / "a.wav"), "wb") as w:
        w.setnchannels(1); w.setsampwidth(2); w.setframerate(48000); w.writeframes(a.astype("<i2").tobytes())
    b.astype("<i2").tofile(tmp_path / "b.s16")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "decode_bursts.py"), "--packets", "--rate", "44100",
                        "--mode", "burst_oqpsk10500", str(tmp_path / "b.s16")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    ev, _, _, _ = _decode([b], 44100, modes="burst_oqpsk10500")
    assert [json.loads(x) for x in r.stdout.splitlines()] == [json.loads(json.dumps(dict(jsonable(e), file=str(tmp_path / "b.s16"))))
                                                              for e in ev]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "decode_bursts.py"), "--packets", str(tmp_path / "a.wav")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    ev, _, _, _ = _decode([a], 48000)
    assert [json.loads(x) for x in r.stdout.splitlines()] == [json.loads(json.dumps(dict(jsonable(e), file=str(tmp_path / "a.wav"))))
                                                              for e in ev]
    assert len(ev) > 0 and json.loads(r.stderr)["carriers"][0]["mode"] == "burst_msk1200"
