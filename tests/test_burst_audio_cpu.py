"""BurstAudioDecoder and tools/decode_bursts.py without a device: the setting and recording checks with their texts, the burst
segment geometry and its lead derivation from the library's constants, the packet stitch rule on constructed packet tables and
the CLI's argument errors."""
import os
import re
import subprocess
import sys
import wave

import numpy as np
import pytest

from jaero_b200.bursts import (AGC_SECONDS, BURST_CHUNK, BURST_MODES, DCD_HOLD_SECONDS, DEFAULT_BURST_LEAD_SECONDS,
                               IDENT_THRESHOLD_DB, TIMEOUT_SECONDS, TRI_SAMPLES, burst_layout, stitch_packets)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOL = os.path.join(ROOT, "tools", "decode_bursts.py")
CSRC = os.path.join(ROOT, "jaero_b200", "csrc")


# ------------------------------------------------------------------------------------------------------ settings
@pytest.mark.parametrize("kw, text", [
    (dict(sample_rate=44100.5), "sample_rate must be a positive whole number of hertz, got 44100.5"),
    (dict(sample_rate=0), "sample_rate must be a positive whole number of hertz"),
    (dict(sample_rate=True), "sample_rate must be a positive whole number of hertz"),
    (dict(sample_rate=48001), "sample_rate 48001 Hz cannot be converted to 48 kHz"),
    (dict(modes="msk1200"), "modes: 'msk1200' is a continuous mode; continuous recordings are decoded by AudioDecoder"),
    (dict(modes=["burst_msk600", "oqpsk8400"]), "modes: 'oqpsk8400' is a continuous mode"),
    (dict(modes="burst_msk2400"), "modes: 'burst_msk2400' is not one of the burst modes burst_msk600, burst_msk1200, "
                                  "burst_oqpsk10500"),
    (dict(segment_seconds=7.5), "segment_seconds must be a whole number of seconds, got 7.5"),
    (dict(segment_seconds=0), "segment_seconds must be at least 1, got 0"),
    (dict(segment_seconds=1), "segment_seconds 1 is too short: a segment must be longer than two guards of 0.50 s"),
    (dict(lead_seconds=-1), "lead_seconds must be a whole number of seconds, got -1"),
    (dict(lead_seconds=1.5), "lead_seconds must be a whole number of seconds, got 1.5"),
    (dict(lead_seconds={"msk600": 3}), "lead_seconds for unknown mode(s) msk600"),
    (dict(max_channels=0), "max_channels must be a positive whole number, got 0"),
    (dict(max_channels=2.0), "max_channels must be a positive whole number, got 2.0"),
    (dict(block_seconds=0), "block_seconds must be in (0, 1]"),
    (dict(block_seconds="x"), "block_seconds must be in (0, 1]"),
    (dict(block_seconds=0.3), "block_seconds: a second of input (44100 samples) is not a whole number of 0.3 s blocks"),
    (dict(block_seconds=100 / 44100), "block_seconds: a 0.0022675736961451248 s block (100 samples) does not give a whole"),
    (dict(block_seconds=0.5), "block_seconds 0.5 gives 24000 samples at 48 kHz, more than one burst demodulator chunk (16384)"),
    (dict(identify_seconds=0), "identify_seconds must be a positive number of seconds, got 0"),
    (dict(identify_seconds=float("inf")), "identify_seconds must be a positive number of seconds"),
])
def test_decoder_refuses_bad_settings_before_the_device(kw, text):
    import jaero_b200
    args = dict(sample_rate=44100)
    args.update(kw)
    with pytest.raises(ValueError) as e:
        jaero_b200.BurstAudioDecoder(**args)
    assert text in str(e.value) and str(e.value).startswith("BurstAudioDecoder: "), str(e.value)


def _pcm(n, seed=0):
    return np.random.default_rng(seed).integers(-1000, 1000, n).astype(np.int16)


@pytest.mark.parametrize("kw, recs, text", [
    (dict(), [_pcm(100).reshape(10, 10)], "recording 0 must be 1-D int16 PCM, got int16 of shape (10, 10)"),
    (dict(), [_pcm(100), _pcm(100).astype(np.int32)], "recording 1 must be 1-D int16 PCM, got int32"),
    (dict(), [_pcm(100), np.zeros(0, dtype=np.int16)], "recording 1 is empty"),
    (dict(), [], "recordings is empty"),
    (dict(), _pcm(100), "recordings must be a list of 1-D int16 arrays, got ndarray"),
    (dict(modes=["burst_msk600", "burst_msk1200", None]), [_pcm(100), _pcm(100)], "modes has 3 entries for 2 recordings"),
    (dict(modes=["burst_msk600"]), [_pcm(100), _pcm(100)], "modes has 1 entries for 2 recordings"),
])
def test_decode_refuses_bad_recordings_before_the_device(kw, recs, text):
    import jaero_b200
    dec = jaero_b200.BurstAudioDecoder(48000, **kw)
    with pytest.raises(ValueError) as e:
        dec.decode(recs)
    assert text in str(e.value) and str(e.value).startswith("BurstAudioDecoder: "), str(e.value)
    assert dec.stats()["carriers"] == [] and dec.carriers() == [] and dec.unplanned() == []


@pytest.mark.parametrize("fs, block, m", [(11025, 0.04, 1920), (22050, 0.1, 4800), (44100, 0.1, 4800), (48000, 0.1, 4800),
                                           (48000, 0.25, 12000), (96000, 0.05, 2400)])
def test_a_whole_hertz_rate_the_converter_takes_is_accepted(fs, block, m):
    import jaero_b200
    dec = jaero_b200.BurstAudioDecoder(fs, block_seconds=block)
    assert dec.sample_rate == fs and all(g.m == m for g in dec.geometry.values())
    assert set(dec.geometry) == set(BURST_MODES)


# ------------------------------------------------------------------------------------------------------ geometry
def _constant(path, pattern):
    with open(os.path.join(CSRC, path)) as fh:
        src = fh.read()
    return re.search(pattern, src)


def test_the_lead_constants_are_the_library_s():
    """BURST_CHUNK from burst.cuh; the R/T time-out (fb x 3 bits at 600 and 1200 bps, fb bits at 10 500) from capi.cu; the
    trident fill, restated from capi.cu's symbol counts with its rounding"""
    assert int(_constant("burst.cuh", r"BURST_CHUNK = (\d+);").group(1)) == BURST_CHUNK
    assert _constant("capi.cu", r"rp\.total_number_of_bits = rp\.oqpsk \? ifb : ifb \* 3;")
    for mode, fb in (("burst_msk600", 600), ("burst_msk1200", 1200), ("burst_oqpsk10500", 10500)):
        bits = fb if fb == 10500 else fb * 3
        assert TIMEOUT_SECONDS[mode] == bits / fb
    assert _constant("capi.cu", r"p\.tri_sz = qround\(\(256\.0 \+ 16\.0 \+ 16\.0\) \* SPS\)")
    assert _constant("capi.cu", r"p\.tri_sz = qround\(200\.0 \* SPS\)")
    assert _constant("capi.cu", r"p\.tri_sz = qround\(224 \* SPS\)")
    assert TRI_SAMPLES == {"burst_msk600": int(224 * 48000 / 600 + 0.5), "burst_msk1200": int(200 * 48000 / 1200 + 0.5),
                           "burst_oqpsk10500": int(288 * 2 * 48000 / 10500 + 0.5)}
    # the burst front's AGC window: agc_len = 1 s of samples
    assert _constant("capi.cu", r"p\.agc_len = \(int\)round\(1 \* p\.Fs\);") and AGC_SECONDS == 1
    # carrier detect: 12 on a sync, 3 off per 1 s tick, down when it reaches 0
    assert int(_constant("rtchannel.cu", r"s\.datacd = 1; s\.datacdcountdown = (\d+);").group(1)) == 12
    assert int(_constant("frame_stages.cuh", r"s\.datacdcountdown -= (\d+);").group(1)) == 3
    assert DCD_HOLD_SECONDS == 12 // 3


def test_the_identification_threshold_is_identify_s():
    import inspect
    from jaero_b200 import identify
    assert IDENT_THRESHOLD_DB == inspect.signature(identify).parameters["threshold_db"].default


@pytest.mark.parametrize("mode", BURST_MODES)
def test_the_default_leads_cover_the_time_out_fill_chunk_agc_and_carrier_detect_hold(mode):
    need = TIMEOUT_SECONDS[mode] + (TRI_SAMPLES[mode] + BURST_CHUNK) / 48000 + AGC_SECONDS + DCD_HOLD_SECONDS
    lead = DEFAULT_BURST_LEAD_SECONDS[mode]
    assert lead == int(lead) and need <= lead < need + 1
    assert DEFAULT_BURST_LEAD_SECONDS == {"burst_msk600": 9, "burst_msk1200": 9, "burst_oqpsk10500": 7}


@pytest.mark.parametrize("rate, block", [(48000, 0.1), (44100, 0.1), (48000, 0.25), (48000, 0.02)])
def test_the_guard_covers_one_chunk_and_one_block(rate, block):
    import jaero_b200
    geo = jaero_b200.BurstAudioDecoder(rate, block_seconds=block).geometry
    for mode, g in geo.items():
        assert g.guard * g.m >= BURST_CHUNK + g.m and (g.guard - 1) * g.m < BURST_CHUNK + g.m
        assert g.lead == DEFAULT_BURST_LEAD_SECONDS[mode] * g.per and g.seg == 10 * g.per
        assert g.window == g.lead + g.seg + g.guard


def test_lead_seconds_as_a_number_or_by_mode():
    geo = burst_layout(48000, 0.1, 10, lead_seconds=3)
    assert {m: g.lead for m, g in geo.items()} == {m: 30 for m in BURST_MODES}
    geo = burst_layout(48000, 0.1, 10, lead_seconds={"burst_oqpsk10500": 5})
    assert {m: g.lead for m, g in geo.items()} == {"burst_msk600": 90, "burst_msk1200": 90, "burst_oqpsk10500": 50}


# ------------------------------------------------------------------------------------------------------ stitching
GEO = burst_layout(48000, 0.1, 10)["burst_oqpsk10500"]        # lead 70, seg 100, guard 5 blocks: boundaries at 170, 270, ...
STARTS = [GEO.start(s) for s in range(4)]


def _pk(kind, nsus, tag):
    return (kind, nsus, bytes([tag]) * (6 + 12 * nsus))


def _stitch(table, ends=None):
    """table: [(row, segment, block, packet)] -> (kept (row, block, packet) list, matched, unmatched)"""
    rows = np.array([p[0] for p in table], dtype=np.int64)
    seg = np.array([p[1] for p in table], dtype=np.int64)
    t = np.array([p[2] for p in table], dtype=np.int64)
    recs = [p[3] for p in table]
    keep, matched, unmatched = stitch_packets(rows, recs, seg, t, STARTS, GEO.guard, None if ends is None else
                                              np.asarray(ends)[rows])
    return [(table[i][0], table[i][1], table[i][2]) for i in np.flatnonzero(keep)], matched, unmatched


def test_a_copy_in_each_neighbour_gives_the_owner_s_copy():
    b = STARTS[1]
    a = _pk(2, 10, 1)
    # the same packet emitted by both at b (owned by 1), and another at b - 1 by 0 and b by 1 (both in their own stretch: 0's)
    kept, matched, _ = _stitch([(0, 0, b, a), (0, 1, b, a)])
    assert kept == [(0, 1, b)] and matched.all()
    c = _pk(1, 0, 2)
    kept, matched, _ = _stitch([(0, 0, b - 1, c), (0, 1, b, c)])
    assert kept == [(0, 0, b - 1)] and matched.all()
    kept, _, _ = _stitch([(0, 0, b - 3, c), (0, 1, b - 3, c)])   # both before b: the owner is 0
    assert kept == [(0, 0, b - 3)]


def test_two_different_packets_one_block_apart_are_both_kept():
    b = STARTS[2]
    p, q = _pk(2, 10, 3), _pk(2, 10, 4)
    r = _pk(2, 9, 3)                                          # p's first bytes with another SU count
    table = [(0, 1, b - 1, p), (0, 2, b - 1, p), (0, 1, b, q), (0, 2, b, q), (0, 2, b + 1, r), (0, 1, b + 1, r)]
    kept, matched, unmatched = _stitch(table)
    assert sorted(kept) == [(0, 1, b - 1), (0, 2, b), (0, 2, b + 1)]
    assert matched.all() and not unmatched.any()
    # one copy each, one block apart: neither is the other's partner
    kept, matched, unmatched = _stitch([(0, 1, b - 1, p), (0, 2, b, q)])
    assert sorted(kept) == [(0, 1, b - 1), (0, 2, b)] and not matched.any() and unmatched.all()


def test_identical_packets_far_apart_are_both_kept():
    b = STARTS[1]
    p = _pk(2, 8, 5)
    table = [(0, 0, b - 4, p), (0, 1, b + 4, p), (0, 1, b + 40, p), (0, 0, 30, p)]
    kept, matched, _ = _stitch(table)
    assert sorted(kept) == [(0, 0, 30), (0, 0, b - 4), (0, 1, b + 4), (0, 1, b + 40)] and not matched.any()


def test_a_partnerless_packet_in_the_window_is_kept():
    b = STARTS[1]
    p = _pk(1, 0, 6)
    for seg, t in ((0, b + 2), (1, b - 2), (0, b - GEO.guard), (1, b + GEO.guard)):
        kept, matched, unmatched = _stitch([(0, seg, t, p)])
        assert kept == [(0, seg, t)] and unmatched.all() and not matched.any()
    # outside the window and outside its own stretch: another segment's, dropped
    kept, _, _ = _stitch([(0, 0, b + GEO.guard + 1, p), (0, 1, b - GEO.guard - 1, p)])
    assert kept == []


def test_rows_are_stitched_apart():
    b = STARTS[1]
    p = _pk(2, 10, 7)
    kept, matched, _ = _stitch([(0, 0, b, p), (1, 1, b, p)])
    assert sorted(kept) == [(0, 0, b), (1, 1, b)] and not matched.any()


def test_a_boundary_past_a_recording_s_end_is_ignored():
    """row 1 ends at block b - 2, before the boundary b: its segment 0 is its last, so its packets near b are its own and are
    neither matched nor unmatched; row 0 runs past b and keeps its boundary rule"""
    b = STARTS[1]
    p, q = _pk(2, 10, 8), _pk(1, 0, 9)
    table = [(1, 0, b - 3, p), (1, 0, b + 1, q), (0, 0, b, p), (0, 1, b, p)]
    kept, matched, unmatched = _stitch(table, ends=[400, b - 2])
    assert sorted(kept) == [(0, 1, b), (1, 0, b - 3), (1, 0, b + 1)]
    assert matched.tolist() == [False, False, True, True] and not unmatched[:2].any()


# ------------------------------------------------------------------------------------------------------ CLI
def _wav(path, data, rate=44100, width=2, channels=1):
    with wave.open(str(path), "wb") as w:
        w.setnchannels(channels); w.setsampwidth(width); w.setframerate(rate)
        w.writeframes(np.ascontiguousarray(data).tobytes())


def _cli(args):
    return subprocess.run([sys.executable, TOOL] + args, capture_output=True, text=True, stdin=subprocess.DEVNULL, timeout=120)


@pytest.fixture
def files(tmp_path):
    _wav(tmp_path / "mono.wav", _pcm(4410).astype("<i2"))
    _wav(tmp_path / "byte.wav", np.zeros(500, dtype=np.uint8), width=1)
    _pcm(4800).tofile(tmp_path / "raw.s16")
    return tmp_path


@pytest.mark.parametrize("args, text", [
    (["raw.s16"], "raw.s16 is not a WAV file: raw 16-bit PCM needs --rate"),
    (["byte.wav"], "the WAV has 8-bit samples"),
    (["--rate", "44100.5", "raw.s16"], "--rate must be a positive whole number of hertz"),
    (["--rate", "fast", "raw.s16"], "--rate must be a number of hertz"),
    (["--rate", "48001", "raw.s16"], "--rate: sample_rate 48001 Hz cannot be converted"),
    (["--segment", "7.5", "mono.wav"], "--segment: segment_seconds must be a whole number of seconds"),
    (["--segment", "1", "mono.wav"], "--segment: segment_seconds 1.0 is too short"),
    (["--block", "0.3", "mono.wav"], "--block: block_seconds: a second of input (44100 samples) is not a whole number"),
    (["--identify", "0", "mono.wav"], "--identify: identify_seconds must be a positive number"),
    (["--mode", "oqpsk10500", "mono.wav"], "--mode: modes: 'oqpsk10500' is a continuous mode"),
    (["--mode", "burst", "mono.wav"], "--mode: modes: 'burst' is not one of the burst modes"),
    (["--channel", "1", "mono.wav"], "the WAV has 1 channel(s); --channel 1 does not exist"),
    (["--channel", "-1", "mono.wav"], "--channel must be 0 or more"),
    (["missing.wav"], "missing.wav: "),
    ([], "the following arguments are required: FILE"),
])
def test_cli_argument_errors(files, args, text):
    r = _cli([str(files / a) if a.endswith((".wav", ".s16")) else a for a in args])
    assert r.returncode == 2, r.stderr
    assert text in r.stderr and "Traceback" not in r.stderr, r.stderr
    assert r.stdout == ""
