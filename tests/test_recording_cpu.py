"""RecordingDecoder without a device: stitching of constructed frame lists, the segment and chunk arithmetic at 2.4 and
2.5 MS/s, and the argument checks with their texts."""
import os
import subprocess
import sys

import numpy as np
import pytest

from jaero_b200 import recording
from jaero_b200.recording import layout, stitch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = 6                     # guard, blocks


def _run(frames, starts, guard=G):
    """frames: [(segment, block, name)] of one carrier -> the kept names in stream order, and the matched / unmatched names"""
    seg = [f[0] for f in frames]
    t = [f[1] for f in frames]
    keep, matched, unmatched = stitch(np.zeros(len(frames)), seg, t, starts, guard)
    kept = sorted((t[i], seg[i], frames[i][2]) for i in np.flatnonzero(keep))
    return ([k[2] for k in kept], {frames[i][2] for i in np.flatnonzero(matched)},
            {frames[i][2] for i in np.flatnonzero(unmatched)})


def _two(b, s0, s1, period=5):
    """frames of segment 0 at s0 (blocks) and of segment 1 at s1, named by the frame they are (a frame every `period`
    blocks from block 0, emitted one block late in a copy when its block is given as (block, +1))"""
    out = []
    for seg, ts in ((0, s0), (1, s1)):
        for t in ts:
            d = 0
            if isinstance(t, tuple):
                t, d = t
            out.append((seg, t + d, "f%d" % (t // period)))
    return out


@pytest.mark.parametrize("d0, d1", [(0, 0), (-1, 0), (0, 1), (1, 0), (0, -1)])
def test_a_frame_both_segments_emit_near_the_boundary_is_kept_once(d0, d1):
    """segment 0 runs to b + guard, segment 1 starts well before b - guard; a frame every 5 blocks. Around b the two copies
    of each frame are emitted up to one block apart either way; the stream has every frame once, in order"""
    b = 50
    s0 = [(t, d0 if abs(t - b) <= 1 else 0) for t in range(0, b + G, 5)]
    s1 = [(t, d1 if abs(t - b) <= 1 else 0) for t in range(30, 101, 5)]
    kept, matched, unmatched = _run(_two(b, s0, s1), [0, b])
    assert kept == ["f%d" % k for k in range(0, 21)]
    assert not unmatched
    assert {"f9", "f10", "f11"} <= matched


def test_crossed_copies_keep_the_earlier_segment():
    """the frame at the boundary: segment 0 emits it in the first block after b, segment 1 in the last block before b.
    Neither copy is inside its own stretch, so segment 0's is kept"""
    b = 50
    frames = [(0, t, "f%d" % (t // 5)) for t in range(0, 46, 5)] + [(0, 50, "f10"), (0, 55, "f11")]
    frames += [(1, 49, "f10")] + [(1, t, "f%d" % (t // 5)) for t in range(55, 101, 5)]
    keep, matched, unmatched = stitch(np.zeros(len(frames)), [f[0] for f in frames], [f[1] for f in frames], [0, b], G)
    kept = [(frames[i][0], frames[i][1]) for i in np.flatnonzero(keep)]
    assert (0, 50) in kept and (1, 49) not in kept
    assert (0, 55) not in kept and (1, 55) in kept       # inside segment 1's stretch: segment 1's copy
    names = sorted((frames[i][1], frames[i][2]) for i in np.flatnonzero(keep))
    assert [n for _, n in names] == ["f%d" % k for k in range(0, 21)]


def test_a_late_lock_keeps_the_earlier_segments_frames():
    """segment 1 locks only after b: its first frames are missing, segment 0's copies are kept (unmatched), nothing twice"""
    b = 50
    frames = _two(b, range(0, b + G, 5), range(60, 101, 5))
    kept, matched, unmatched = _run(frames, [0, b])
    assert kept == ["f%d" % k for k in range(0, 21)]
    assert unmatched == {"f9", "f10", "f11"}


def test_a_frame_only_the_earlier_segment_has_is_kept():
    b = 50
    frames = _two(b, range(0, b + G, 5), [t for t in range(30, 101, 5) if t != 50])
    kept, matched, unmatched = _run(frames, [0, b])
    assert kept == ["f%d" % k for k in range(0, 21)]
    assert unmatched == {"f10"}
    assert "f9" in matched and "f11" in matched


def test_frames_outside_the_windows_come_from_their_owner_only():
    """segment 1's lead (before b - guard) and segment 0's frames are dropped outside their stretches, whatever they hold"""
    b = 50
    frames = _two(b, range(0, b + G, 5), range(20, 101, 5))
    keep, _, _ = stitch(np.zeros(len(frames)), [f[0] for f in frames], [f[1] for f in frames], [0, b], G)
    for i, (s, t, _) in enumerate(frames):
        if abs(t - b) > G:
            assert keep[i] == ((s == 0) == (t < b)), (s, t)


def test_runs_of_identical_fill_frames_are_matched_by_time():
    """every frame carries the same fill units: matching is by emission time, so each is kept once"""
    b = 50
    frames = [(0, t, "fill") for t in range(0, b + G, 5)] + [(1, t, "fill") for t in range(30, 101, 5)]
    keep, matched, _ = stitch(np.zeros(len(frames)), [f[0] for f in frames], [f[1] for f in frames], [0, b], G)
    t = sorted(frames[i][1] for i in np.flatnonzero(keep))
    assert t == list(range(0, 101, 5))


def test_many_segments_and_carriers_at_once():
    """three carriers, five segments, each frame of a carrier emitted by every segment running then (the later segment's copy
    a block early or late at random near the boundaries): the stream of each carrier has every frame once and in order"""
    rng = np.random.default_rng(7)
    seg_b, lead, period = 40, 12, 5
    starts = [0] + [g * seg_b + lead for g in range(1, 5)]
    car, seg, t, name = [], [], [], []
    for c in range(3):
        off = c                                           # each carrier's frames on its own phase
        for g in range(5):
            a, z = g * seg_b, g * seg_b + lead + seg_b + G
            if g == 4:
                z = 5 * seg_b + lead
            for k in range(0, 400, 1):
                tk = k * period + off
                if a + 3 <= tk < z:
                    car.append(c); seg.append(g); name.append(k)
                    t.append(tk + int(rng.integers(-1, 2)) * (g > 0 and abs(tk - starts[g]) <= G))
    keep, _, _ = stitch(car, seg, t, starts, G)
    for c in range(3):
        got = sorted((t[i], name[i]) for i in np.flatnonzero(keep) if car[i] == c)
        names = [n for _, n in got]
        assert names == sorted(set(names)) and names == list(range(names[0], names[-1] + 1)), c


def test_nothing_to_stitch():
    keep, matched, unmatched = stitch([], [], [], [0, 10], G)
    assert len(keep) == len(matched) == len(unmatched) == 0


# ------------------------------------------------------------------------------------------------------ arithmetic
@pytest.mark.parametrize("rate, m", [(2.4e6, 4800), (2.5e6, 4800)])
def test_segment_grid_at_sdr_rates(rate, m):
    geo = layout(rate, 0.1, 10, lead_seconds=None, max_channels=4096)
    for mode, g in geo.items():
        assert g.per == 10 and g.m == m and g.seg == 100
        assert g.lead == 10 * recording.DEFAULT_LEAD_SECONDS[mode]
        assert g.guard == {"msk600": 21, "msk1200": 11, "oqpsk10500": 6, "oqpsk8400": 6}[mode]
        assert g.window == g.lead + g.seg + g.guard
        assert g.start(0) == 0 and g.start(3) == 300 + g.lead
        assert g.chunk_blocks(4) == 3 * 100 + g.window


@pytest.mark.parametrize("n, cap, S", [(1, 4096, 4096), (4, 4096, 1024), (5, 4096, 819), (64, 4096, 64), (4096, 4096, 1),
                                       (5000, 4096, 1), (3, 16, 5), (3, 2, 1)])
def test_segments_per_chunk_are_capped_by_max_channels(n, cap, S):
    g = layout(2.4e6, 0.1, 10, max_channels=cap)["oqpsk10500"]
    assert g.segments_per_chunk(n) == S
    assert n * S <= cap or S == 1


def test_the_last_chunk_has_every_segment_whose_stretch_starts_before_the_end():
    g = layout(2.5e6, 0.1, 7, lead_seconds=3)["msk1200"]          # seg 70, lead 30: segment s owns from 70 s + 30 (s >= 1)
    assert g.final_segments(1) == 1 and g.final_segments(100) == 1 and g.final_segments(101) == 2
    assert g.final_segments(170) == 2 and g.final_segments(171) == 3
    for blocks in range(1, 2000, 17):
        S = g.final_segments(blocks)
        assert S == 1 or g.start(S - 1) < blocks
        assert g.start(S) >= blocks
    # the 120 s recording at 10 s segments: 11 segments at every lead of 10 s or more below 20 s, 12 below 10 s
    for mode, geo in layout(2.4e6, 0.1, 10).items():
        assert geo.final_segments(1200) == (11 if geo.lead >= 100 else 12), mode


def test_leads_by_mode():
    geo = layout(2.4e6, 0.05, 10, lead_seconds={"msk600": 3})
    assert geo["msk600"].lead == 60 and geo["oqpsk8400"].lead == 20 * recording.DEFAULT_LEAD_SECONDS["oqpsk8400"]
    assert all(g.lead == 0 for g in layout(2.4e6, 0.1, 10, lead_seconds=0).values())


# ------------------------------------------------------------------------------------------------------ argument checks
@pytest.mark.parametrize("kw, text", [
    (dict(segment_seconds=7.5), "segment_seconds must be a whole number of seconds, got 7.5"),
    (dict(segment_seconds="x"), "segment_seconds must be a whole number of seconds"),
    (dict(segment_seconds=0), "segment_seconds must be at least 1"),
    (dict(segment_seconds=4), "segment_seconds 4 is too short for msk600"),
    (dict(lead_seconds=2.5), "lead_seconds must be a whole number of seconds, got 2.5"),
    (dict(lead_seconds=-1), "lead_seconds must be a whole number of seconds, got -1"),
    (dict(lead_seconds={"msk2400": 3}), "lead_seconds for unknown mode(s) msk2400"),
    (dict(max_channels=0), "max_channels must be a positive whole number, got 0"),
    (dict(max_channels=10.5), "max_channels must be a positive whole number"),
    (dict(block_seconds=0.3), "a second of input (2400000 samples) is not a whole number of 0.3 s blocks"),
    (dict(block_seconds=0.125), "block_seconds 0.125 is longer than a quarter of the shortest frame"),
    (dict(block_seconds=0), "block_seconds must be in (0, 1]"),
    (dict(input_rate=2.5e6, block_seconds=0.0016), "does not give a whole number of 48 kHz samples"),
])
def test_decoder_refuses_bad_settings_before_the_device(kw, text):
    import jaero_b200
    args = dict(input_rate=2.4e6, fmt="cu8", segment_seconds=10)
    args.update(kw)
    with pytest.raises(ValueError) as e:
        jaero_b200.RecordingDecoder(**args)
    assert text in str(e.value) and str(e.value).startswith("RecordingDecoder: ")


def test_receiver_checks_still_apply():
    import jaero_b200
    with pytest.raises(ValueError):
        jaero_b200.RecordingDecoder(2.4e6, "cs8")
    with pytest.raises(TypeError):
        jaero_b200.RecordingDecoder(2.4e6, "cu8", threshold=3.0)
    with pytest.raises(ValueError):
        jaero_b200.RecordingDecoder(2.4e6 + 0.5, "cu8")


@pytest.mark.parametrize("args, text", [
    (["--segment", "7.5"], "--segment"),
    (["--segment", "3"], "--segment"),
    (["--segment", "10", "--block", "0.3"], "--segment"),
])
def test_cli_refuses_bad_segment_settings(args, text):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "receive.py"), "--rate", "2400000", "--format", "cu8"]
                       + args + ["-"], capture_output=True, text=True, stdin=subprocess.DEVNULL, timeout=120)
    assert r.returncode != 0
    assert text in r.stderr and "Traceback" not in r.stderr, r.stderr
    assert r.stdout == ""
