"""AudioDecoder and tools/decode_audio.py without a device: the setting and recording checks with their texts, the segment grid
of recordings of different lengths (dead and live segments, lock counts, stitching), the WAV and raw readers and the CLI's
argument errors."""
import os
import subprocess
import sys
import wave

import numpy as np
import pytest

from jaero_b200.recording import _SegmentEngine, _Segments, layout, stitch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOL = os.path.join(ROOT, "tools", "decode_audio.py")
sys.path.insert(0, os.path.join(ROOT, "tools"))


# ------------------------------------------------------------------------------------------------------ settings
@pytest.mark.parametrize("kw, text", [
    (dict(sample_rate=44100.5), "sample_rate must be a positive whole number of hertz, got 44100.5"),
    (dict(sample_rate=0), "sample_rate must be a positive whole number of hertz"),
    (dict(sample_rate="x"), "sample_rate must be a positive whole number of hertz"),
    (dict(sample_rate=48001), "sample_rate 48001 Hz cannot be converted to 48 kHz"),
    (dict(segment_seconds=7.5), "segment_seconds must be a whole number of seconds, got 7.5"),
    (dict(segment_seconds=4), "segment_seconds 4 is too short for msk600"),
    (dict(lead_seconds=-1), "lead_seconds must be a whole number of seconds, got -1"),
    (dict(max_channels=0), "max_channels must be a positive whole number, got 0"),
    (dict(block_seconds=0.3), "block_seconds: a second of input (44100 samples) is not a whole number of 0.3 s blocks"),
    (dict(block_seconds=0.125, sample_rate=48000), "block_seconds 0.125 is longer than a quarter of the shortest frame"),
    (dict(block_seconds=0), "block_seconds must be in (0, 1]"),
    (dict(sample_rate=44101), "sample_rate 44101 Hz cannot be converted to 48 kHz: jaero_b200 error -1: jaero_resample_plan: "
                              "output_rate/input_rate reduces to 48000/44101; L and M must not exceed 1024"),
    (dict(sample_rate=11025), "block_seconds: a second of input (11025 samples) is not a whole number of 0.1 s blocks"),
    (dict(block_seconds=100 / 44100), "block_seconds: a 0.0022675736961451248 s block (100 samples) does not give a whole number"),
    (dict(identify_seconds=0), "identify_seconds must be a positive number of seconds, got 0"),
    (dict(identify_seconds="soon"), "identify_seconds must be a positive number of seconds"),
    (dict(modes="msk2400"), "modes: 'msk2400' is not one of the continuous modes"),
    (dict(modes=["msk600", "burst_msk1200"]), "modes: 'burst_msk1200' is a burst (R/T) mode; burst recordings are not supported"),
    (dict(centers_hz=0), "centers_hz must be audio frequencies in (0, 24000) Hz or None, got 0"),
    (dict(centers_hz=[1000.0, 30000.0]), "centers_hz must be audio frequencies in (0, 24000) Hz or None, got 30000.0"),
    (dict(centers_hz="mid"), "centers_hz must be audio frequencies"),
])
def test_decoder_refuses_bad_settings_before_the_device(kw, text):
    import jaero_b200
    args = dict(sample_rate=44100)
    args.update(kw)
    with pytest.raises(ValueError) as e:
        jaero_b200.AudioDecoder(**args)
    assert text in str(e.value) and str(e.value).startswith("AudioDecoder: "), str(e.value)


def _pcm(n, seed=0):
    return np.random.default_rng(seed).integers(-1000, 1000, n).astype(np.int16)


@pytest.mark.parametrize("kw, recs, text", [
    (dict(), [_pcm(100).reshape(10, 10)], "recording 0 must be 1-D int16 PCM, got int16 of shape (10, 10)"),
    (dict(), [_pcm(100), _pcm(100).astype(np.int32)], "recording 1 must be 1-D int16 PCM, got int32"),
    (dict(), [_pcm(100).astype(np.float32)], "recording 0 must be 1-D int16 PCM, got float32"),
    (dict(), [_pcm(100), np.zeros(0, dtype=np.int16)], "recording 1 is empty"),
    (dict(), [], "recordings is empty"),
    (dict(), _pcm(100), "recordings must be a list of 1-D int16 arrays, got ndarray"),
    (dict(modes=["msk600", "msk1200", None]), [_pcm(100), _pcm(100)], "modes has 3 entries for 2 recordings"),
    (dict(centers_hz=[1000.0]), [_pcm(100), _pcm(100)], "centers_hz has 1 entries for 2 recordings"),
])
def test_decode_refuses_bad_recordings_before_the_device(kw, recs, text):
    import jaero_b200
    dec = jaero_b200.AudioDecoder(48000, **kw)
    with pytest.raises(ValueError) as e:
        dec.decode(recs)
    assert text in str(e.value) and str(e.value).startswith("AudioDecoder: "), str(e.value)
    assert dec.stats()["carriers"] == [] and dec.carriers() == [] and dec.unplanned() == []


@pytest.mark.parametrize("fs, block, m", [(8000, 0.1, 4800), (11025, 0.04, 1920), (16000, 0.1, 4800), (22050, 0.1, 4800),
                                           (32000, 0.1, 4800), (44100, 0.1, 4800), (48000, 0.1, 4800), (96000, 0.1, 4800)])
def test_a_whole_hertz_rate_the_converter_takes_is_accepted(fs, block, m):
    """the block grid is checked against the rate converter's ratio, not the down-converter's: 22050 Hz is 320/147 and
    11025 Hz 640/147, beyond the down-converter's interpolation of 256"""
    import jaero_b200
    dec = jaero_b200.AudioDecoder(fs, block_seconds=block)
    assert dec.sample_rate == fs and all(g.m == m for g in dec.geometry.values())


def test_a_library_that_is_not_built_is_not_reported_as_a_bad_rate(monkeypatch, tmp_path):
    import jaero_b200
    monkeypatch.setattr(jaero_b200, "_lib", None)
    monkeypatch.setattr(jaero_b200, "LIB_PATH", str(tmp_path / "libjaero_b200.so"))
    with pytest.raises(jaero_b200.JaeroError, match="is not built"):
        jaero_b200.AudioDecoder(44100)


# ------------------------------------------------------------------------------------------------------ the segment grid
def test_rows_of_different_lengths_have_dead_and_live_segments():
    """recordings of 37, 61 and 23 s at 10 s segments, 6 s lead, 0.1 s blocks: segment g owns from 10 g + 6 s (g >= 1). A
    segment is live when its stretch starts before its recording's end: 4, 6 and 2 segments; the last chunk holds 6"""
    geo = layout(48000, 0.1, 10, lead_seconds=6)["oqpsk10500"]
    ends = np.array([370, 610, 230])
    S = geo.final_segments(int(ends.max()))
    assert S == 6
    end, alive = geo.rows(0, S, int(ends.max()), ends)
    assert alive.sum(axis=1).tolist() == [4, 6, 2]
    for c, e in enumerate(ends):
        for s in range(S):
            assert alive[c, s] == (geo.start(s) < e)
            assert end[c, s] == e - s * geo.seg                  # a segment holds PCM up to its recording's end
    # a later chunk of two segments from segment 3: only the longest recording's are both live
    end, alive = geo.rows(3, 2, 610 - 300, ends)
    assert alive.tolist() == [[True, False], [True, True], [False, False]]
    assert end[:, 0].tolist() == [70, 310, -70]
    # one row without ends: every segment runs to the end of the PCM
    end, alive = geo.rows(0, 3, 250)
    assert alive.all() and end.tolist() == [[250, 150, 50]]


def _records(frames):
    """[(row, segment, block, crc_ok)] -> a P-channel table as _chunk builds it (one record per frame, frame number = block)"""
    rec = np.zeros((len(frames), 16), dtype=np.uint8)
    for i, (_, _, t, ok) in enumerate(frames):
        rec[i, 12], rec[i, 14], rec[i, 15] = ok, t & 255, t >> 8
    col = lambda k: np.array([f[k] for f in frames], dtype=np.int64)
    return dict(rec=rec, car=col(0), gs=col(1), t=col(2))


def test_dead_segments_count_as_neither_late_nor_unlocked():
    geo = layout(48000, 0.1, 10, lead_seconds=6)["oqpsk10500"]
    ends = np.array([370, 610, 230])
    g = _Segments("oqpsk10500", [0, 1, 2], {}, geo, ends=ends)
    S = geo.final_segments(610)
    _, alive = geo.rows(0, S, 610, ends)
    frames = []
    for c, e in enumerate(ends):
        for s in range(S):
            if alive[c, s] and not (c == 1 and s == 4):           # recording 1's fifth segment never locks
                t0 = s * geo.seg + (30 if not (c == 0 and s == 2) else 80)    # recording 0's third segment locks late
                frames.append((c, s, t0, 1))
    _SegmentEngine._locks(_SegmentEngine(), g, _records(frames), S, alive)
    assert g.late.tolist() == [1, 0, 0]
    assert g.unlocked.tolist() == [0, 1, 0]
    assert g.lock_blocks.tolist() == [81, 31, 31]


def test_stitch_keeps_one_copy_per_boundary_frame_for_rows_with_different_segment_counts():
    """three rows, frames every 5 blocks, each frame emitted by every live segment running then; the rows end at blocks 370,
    610 and 258, so they have 4, 6 and 2 segments, and the last one ends 2 blocks before the boundary at 260 it never reaches.
    Every row's stream has each of its frames once, and only boundaries inside a row are matched: no frame near a boundary
    the row never reaches is reported as unmatched"""
    geo = layout(48000, 0.1, 10, lead_seconds=6)["oqpsk10500"]
    ends = np.array([370, 610, 258])
    S = geo.final_segments(610)
    starts = [geo.start(s) for s in range(S)]
    end, alive = geo.rows(0, S, 610, ends)
    car, seg, t = [], [], []
    for c in range(3):
        for s in range(S):
            if not alive[c, s]:
                continue
            a, z = s * geo.seg, s * geo.seg + min(end[c, s], geo.window)
            for tk in range(0, 700, 5):
                if a + 3 <= tk < z:
                    car.append(c); seg.append(s); t.append(tk + c)
    car, seg, t = np.array(car), np.array(seg), np.array(t)
    keep, matched, unmatched = stitch(car, seg, t, starts, geo.guard, ends[car])
    for c in range(3):
        got = sorted(t[keep & (car == c)].tolist())
        assert got == sorted(set(t[car == c].tolist())), c
    assert not unmatched.any()
    # boundaries matched per row: one frame pair per boundary the row reaches
    for c in range(3):
        inner = [b for b in starts[1:] if b < ends[c]]
        assert len(inner) == alive[c].sum() - 1
        want = len({x for x in t[car == c].tolist() if any(abs(x - b) <= geo.guard for b in inner)})
        assert int((matched & keep & (car == c)).sum()) == want > 0, c
    # without ends, the short rows' frames near the boundaries they never reach come back as unmatched
    _, _, unmatched = stitch(car, seg, t, starts, geo.guard)
    assert unmatched.any()


# ------------------------------------------------------------------------------------------------------ readers
def _wav(path, data, rate=44100, width=2, channels=1):
    with wave.open(str(path), "wb") as w:
        w.setnchannels(channels); w.setsampwidth(width); w.setframerate(rate)
        w.writeframes(np.ascontiguousarray(data).tobytes())


def test_mono_wav_round_trip(tmp_path):
    from decode_audio import read_audio
    x = _pcm(12345, 1)
    _wav(tmp_path / "a.wav", x.astype("<i2"), rate=44100)
    pcm, fs = read_audio(str(tmp_path / "a.wav"))
    assert fs == 44100 and pcm.dtype == np.int16 and pcm.ndim == 1 and np.array_equal(pcm, x)


@pytest.mark.parametrize("channel", [0, 1])
def test_stereo_wav_gives_the_chosen_channel(tmp_path, channel):
    from decode_audio import read_audio
    x = np.stack([_pcm(5000, 2), _pcm(5000, 3)], axis=1)           # frames of (left, right)
    _wav(tmp_path / "s.wav", x.astype("<i2"), rate=48000, channels=2)
    pcm, fs = read_audio(str(tmp_path / "s.wav"), channel=channel)
    assert fs == 48000 and pcm.flags.c_contiguous and np.array_equal(pcm, x[:, channel])


def test_raw_round_trip(tmp_path):
    from decode_audio import read_audio
    x = _pcm(7777, 4)
    x.astype("<i2").tofile(tmp_path / "r.s16")
    pcm, fs = read_audio(str(tmp_path / "r.s16"), rate=22050)
    assert fs == 22050 and pcm.dtype == np.int16 and np.array_equal(pcm, x)


@pytest.mark.parametrize("width", [1, 3])
def test_other_sample_widths_are_refused(tmp_path, width):
    from decode_audio import AudioFileError, read_audio
    _wav(tmp_path / "w.wav", np.zeros(300 * width, dtype=np.uint8), width=width)
    with pytest.raises(AudioFileError) as e:
        read_audio(str(tmp_path / "w.wav"))
    assert "the WAV has %d-bit samples; only 16-bit PCM WAV is read" % (8 * width) in str(e.value)


def test_a_float_wav_is_refused(tmp_path):
    """WAVE_FORMAT_IEEE_FLOAT (3), 32-bit mono"""
    from decode_audio import AudioFileError, read_audio
    data = np.zeros(100, dtype="<f4").tobytes()
    fmt = (3).to_bytes(2, "little") + (1).to_bytes(2, "little") + (48000).to_bytes(4, "little") + (192000).to_bytes(4, "little") \
        + (4).to_bytes(2, "little") + (32).to_bytes(2, "little")
    body = b"WAVE" + b"fmt " + len(fmt).to_bytes(4, "little") + fmt + b"data" + len(data).to_bytes(4, "little") + data
    (tmp_path / "f.wav").write_bytes(b"RIFF" + len(body).to_bytes(4, "little") + body)
    with pytest.raises(AudioFileError, match="encoding is not PCM"):
        read_audio(str(tmp_path / "f.wav"))


def test_raw_input_needs_a_rate(tmp_path):
    from decode_audio import AudioFileError, read_audio
    _pcm(100).tofile(tmp_path / "r.s16")
    with pytest.raises(AudioFileError, match="is not a WAV file: raw 16-bit PCM needs --rate"):
        read_audio(str(tmp_path / "r.s16"))


# ------------------------------------------------------------------------------------------------------ CLI
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
    (["--segment", "3", "mono.wav"], "--segment: segment_seconds 3.0 is too short for msk600"),
    (["--block", "0.3", "mono.wav"], "--block: block_seconds: a second of input (44100 samples) is not a whole number"),
    (["--identify", "0", "mono.wav"], "--identify: identify_seconds must be a positive number"),
    (["--mode", "burst_oqpsk10500", "mono.wav"], "--mode: modes: 'burst_oqpsk10500' is a burst (R/T) mode"),
    (["--center", "-5", "mono.wav"], "--center: centers_hz must be audio frequencies"),
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
