"""CPU tests: the run-time controls of the continuous demodulators (CenterFreqChangedSlot, setAFC, setSQL, setCPUReduce) in
the restated oracle against the reference's own slots (oracle/_ref), on the committed recordings, with the schedules of
tests/control_schedules.py; and those schedules reach the branches they are there for."""
import hashlib
import multiprocessing as mp

import numpy as np
import pytest

import control_schedules as cs
from conftest import load_excerpt
from oracle import ref, restated

needs_ref = pytest.mark.skipif(not (ref.available() and hasattr(ref.lib(), "jref_set_center_freq")),
                               reason="oracle/_ref not built with the control entry points (needs /root/reference)")
NAMES = list(cs.RECORDINGS)
ALL = NAMES + list(cs.SYNTHETIC)


def _settings(name):
    return cs.RECORDINGS[name] if name in cs.RECORDINGS else cs.SYNTHETIC[name]


def _stream(name):
    return load_excerpt(name) if name in cs.RECORDINGS else cs.synthetic_stream(name)


def _run(name, stop_at_events=False):
    """restated run of one stream under its schedule; with stop_at_events also [(tag, calls, state before, state after)]
    of every event"""
    kind, kw, _ = _settings(name)
    pcm = _stream(name)
    ev = cs.recording_schedule(name, len(pcm))
    tags = {a: t for a, _, t in ev}
    d = restated.OracleDemod(kind, **kw)
    seen = []
    for a, n, calls in restated.write_plan(len(pcm), 4800, cs.events(ev)):
        if calls and stop_at_events:
            before = d.state()
            restated.apply_calls(d, calls)
            seen.append((tags[a], calls, before, d.state()))
        else:
            restated.apply_calls(d, calls)
        d.write(pcm[a:a + n])
    return d.take_soft(), d.state(), d.take_cfe_log(), seen


@pytest.mark.parametrize("name", ALL)
def test_schedule_reaches_every_branch(name):
    """Each tagged event finds the demodulator in the state it is there for, and the centre change takes the branch named
    (on the recordings and on the synthetic 8000 bps stream the GPU tests also run the schedule on)."""
    kind, kw, _ = _settings(name)
    thr, half, fb = kw["signalthreshold"], kw["lockingbw"] / 2.0, kw["fb"]
    lo = 0.5 * fb if kind == "oqpsk" else 0.75 * fb
    hi = 24000.0 - lo
    clamps = not (kind == "oqpsk" and fb == 8400)                 # 8400 bps skips the per-mode clamp (oqpskdemodulator.cpp:293)
    soft, _, _, seen = _run(name, stop_at_events=True)
    assert len(soft) > 1000
    hit = set()
    for tags, calls, b, s in seen:
        for tag in filter(None, tags.split(",")):
            hit.add(tag)
            req = [c[1] for c in calls if c[0] == "set_center_freq"]
            if tag == "inside":
                assert abs(b["mixer2_freq"] - s["center_freq"]) <= half and s["mixer2_freq"] == b["mixer2_freq"]
            elif tag == "below":
                assert b["mixer2_freq"] - s["center_freq"] < -half and s["mixer2_freq"] == s["center_freq"] - half
            elif tag == "above":
                assert b["mixer2_freq"] - s["center_freq"] > half and s["mixer2_freq"] == s["center_freq"] + half
            elif tag == "follow":
                assert s["mixer2_freq"] == s["center_freq"] == req[-1] and abs(b["mixer2_freq"] - req[-1]) > 0.001
            elif tag == "clamp_low":
                assert s["center_freq"] == (lo if clamps else req[-1])
            elif tag == "clamp_high":
                assert s["center_freq"] == (hi if clamps else req[-1])
            elif tag == "negative":
                assert s["center_freq"] == (lo if clamps else 0.0)
            elif tag in ("afc_off_locked", "sql_locked"):
                assert b["mse"] < thr and abs(b["mixer2_freq"] - b["center_freq"]) < 60.0, (tag, b)
            elif tag == "sql_unlocked":
                assert b["mse"] > thr, b
            elif tag in ("offset_locked", "afc_on_pulling", "afc_off_pulling"):
                # locked with mixer2 more than 3 Hz off mixer_center: the AFC counts down to a re-centre (demod_stages.cuh:202,216)
                assert s["mse"] < thr and abs(s["mixer2_freq"] - s["center_freq"]) > 3.0, (tag, s)
    assert hit >= {"inside", "below", "above", "follow", "clamp_low", "clamp_high", "negative", "afc_off_locked", "sql_locked",
                   "sql_unlocked", "offset_locked", "afc_on_pulling", "afc_off_pulling", "cpu_reduce_on", "cpu_reduce_off_in_run"}


def test_event_positions_sit_on_the_epoch_edges():
    """bef / aft / mid land one sample before a trigger sample, right after one and halfway between, and the CPU-reduce
    switch-off falls inside the ring run that follows coarseCounter reaching Fs."""
    for name in ALL:
        kind, kw, t_lock = _settings(name)
        T = cs.trigger_every(kw)
        ev = cs.recording_schedule(name, len(_stream(name)))
        offs = {a % T for a, _, _ in ev}
        assert {T - 2, 0, T // 2, T - 1} <= offs, (name, sorted(offs))
        on = [a for a, _, t in ev if t == "cpu_reduce_on"][0]
        off = [a for a, _, t in ev if t == "cpu_reduce_off_in_run"][0]
        assert on % T == 0 and cs.FS <= off - on < cs.FS + cs.trigger_every(kw, True)


def test_write_plan_cuts_at_events():
    plan = restated.write_plan(10000, 4800, [(4799, [("set_afc", 0)]), (1, [("set_sql", 1), ("set_dcd", 1)])])
    assert [(a, n) for a, n, _ in plan] == [(0, 1), (1, 4798), (4799, 1), (4800, 4800), (9600, 400)]
    assert plan[1][2] == [("set_sql", 1), ("set_dcd", 1)] and plan[2][2] == [("set_afc", 0)]
    assert [(a, n) for a, n, _ in restated.write_plan(7, [3, 1, 5])] == [(0, 3), (3, 1), (4, 3)]
    with pytest.raises(AssertionError):
        restated.write_plan(10, 4, [(3, [("bogus",)])])


@needs_ref
@pytest.mark.parametrize("name", ALL)
def test_restated_controls_match_reference(name):
    """The restated slots and flags equal the reference's own: SHA-identical soft bits, identical coarse-estimate logs and
    equal loop state after every schedule (one fresh process per reference run: the reference keeps function statics)."""
    kind, kw, _ = _settings(name)
    pcm = _stream(name)
    ev = cs.events(cs.recording_schedule(name, len(pcm)))
    with mp.get_context("spawn").Pool(1, maxtasksperchild=1) as pool:
        rs, rstate, rcfe = pool.apply(ref.run_demod_job, ((kind, kw, pcm, 4800, None, ev),))
    soft, state, cfe, _ = _run(name)
    assert len(soft) == len(rs) and hashlib.sha256(soft.tobytes()).hexdigest() == hashlib.sha256(rs.tobytes()).hexdigest()
    assert np.array_equal(cfe, rcfe)
    assert state == rstate
