"""The frame-layer stream builders (tests/frame_streams.py) checked on the restated oracle, CPU only: clean streams decode to
exactly what was planted, and every adversarial family reaches the edge it was built for."""
import numpy as np
import pytest

import frame_streams as fs
from oracle import restated


def run_p(fb, m):
    o = restated.OraclePChannel(fb)
    a = 0
    for k, n in enumerate(m["cuts"]):
        o.process(m["soft"][a:a + n]); a += n
        if k in m["lost"]:
            o.lost_signal()
    b, ok, fr = o.take_sus()
    o.close()
    return b, ok, fr


def run_c(m):
    o = restated.OracleCChannel()
    a = 0
    for k, n in enumerate(m["cuts"]):
        o.process(m["soft"][a:a + n]); a += n
        if k in m["lost"]:
            o.lost_signal()
    su, ok, voice = o.take_frames()
    o.close()
    return su, ok, voice


def run_rt(fb, m, vector_semantics=False):
    o = restated.OracleRTChannel(fb)
    a = 0
    for n in m["cuts"]:
        o.process(m["soft"][a:a + n], vector_semantics); a += n
    pk, tr = o.packets(), o.trials
    o.close()
    return pk, tr


def planted_run(b, ok, sus):
    """indices, among the planted signal units, of the CRC-valid units decoded (-1: not planted)"""
    return [next((k for k in range(len(sus)) if np.array_equal(sus[k], x)), -1) for x, o in zip(b, ok) if o]


def assert_decodes_planted(b, ok, sus, n_sus, tag=""):
    """the CRC-valid units are planted units, in order, with none skipped, and include all of the second frame (the first
    is cut short by the decoder's start-up; the delay line still holds the last units)"""
    run = planted_run(b, ok, sus)
    assert run and run == list(range(run[0], run[0] + len(run))) and run[0] <= n_sus and len(run) >= n_sus, (tag, run)


@pytest.mark.parametrize("fb", [10500, 1200, 600])
def test_p_offset_family_covers_every_offset_and_decodes_what_was_planted(fb):
    g = fs.p_geometry(fb)
    fam = fs.p_offset_family(fb)
    arms = 2 if g["oqpsk"] else 1
    assert sorted({(m["state"], m["arm"], m["offset"]) for m in fam}) == sorted(
        (s, a, o) for s in ("idle", "running") for a in range(arms) for o in range(32))
    for m in fam:
        uw_last = 80 + m["arm"] + g["uw_len"] - 1 + (g["frame"] if m["state"] == "running" else 0)
        assert uw_last - m["cuts"][0] == m["offset"]
        b, ok, fr = run_p(fb, m)
        assert_decodes_planted(b, ok, m["sus"], g["sus_per_frame"], m["tag"])


@pytest.mark.parametrize("fb", [10500, 1200, 600])
def test_p_mutation_family_reaches_its_edges(fb):
    g = fs.p_geometry(fb)
    fam = {m["tag"]: m for m in fs.p_mutation_family(fb)}
    n_sus = g["sus_per_frame"]
    clean = fam["p-clean"]
    b, ok, _ = run_p(fb, clean)
    assert_decodes_planted(b, ok, clean["sus"], n_sus)

    def same(t):
        bt, okt, _ = run_p(fb, fam[t])
        return len(bt) == len(b) and np.array_equal(bt, b) and np.array_equal(okt, ok)

    if g["oqpsk"]:
        # the phase-invariant detectors correct an inverted arm, one or both
        assert same("p-invert-both") and same("p-invert-arm0") and same("p-invert-arm1")
    else:
        assert len(run_p(fb, fam["p-invert-both"])[0]) == 0      # the MSK detector is exact: an inverted stream never syncs
    for k in (0, 13, 31):                                         # one UW bit wrong: frame 1 never syncs (its exact twin does)
        assert len(run_p(fb, fam["p-uw-wrong-%d" % k])[0]) < len(b)
    synced = [d for d in range(-72, -63) if not same("p-plant-%+d" % d)]
    # 10.5 kbps with DCD up: a copy framed from counter value number_of_bits - 67 on syncs, one from - 68 does not (its
    # interleaved bits are spread over the block, so the Viterbi decoder repairs the data it overwrote). MSK searches always.
    assert synced == (list(range(-67, -63)) if g["oqpsk"] else list(range(-72, -63))), synced
    for t in ("p-slip-insert", "p-slip-delete"):                  # a slip loses sync until the next UW
        assert run_p(fb, fam[t])[1].sum() < ok.sum(), t
    assert same("p-long-noise")
    assert len(run_p(fb, fam["p-lost-mid-frame"])[0]) < len(b)  # LostSignal in frame 2: that frame is lost


def run_p_deviation(st, lost_at=None):
    """the reference over p_dcd_deviation_stream's schedule; lost_at: a LostSignal just before that stream index"""
    o = restated.OraclePChannel(10500)
    a, dcd = 0, []
    for k, n in enumerate(st["cuts"]):
        seg = st["soft"][a:a + n]
        if lost_at is not None and a <= lost_at < a + n:
            o.process(seg[:lost_at - a]); o.lost_signal(); o.process(seg[lost_at - a:])
        else:
            o.process(seg)
        a += n
        if k in st["ticks"]:
            o.update_dcd()
        dcd.append(o.dcd)
    b, ok, fr = o.take_sus()
    o.close()
    return b, ok, fr, dcd


def test_p_dcd_deviation_stream_is_the_case_it_claims():
    st = fs.p_dcd_deviation_stream()
    b, ok, fr, dcd = run_p_deviation(st)
    b0, ok0, _, dcd0 = run_p_deviation(fs.p_dcd_deviation_stream(copy=False))
    assert dcd[0] is False and dcd[1] is False and dcd[2] is True   # down after the tick, raised again by frame 3's CRCs
    n = 26
    assert not ok[:3 * n - 1].any() and ok[3 * n - 1:4 * n - 1].all()   # frames 0..2 fail (25 + 26 + 26 units), 3 is good
    # the reference ignores the copy: everything is as without it
    assert np.array_equal(b, b0) and np.array_equal(ok, ok0) and dcd == dcd0
    # an AeroL made to search at the copy (LostSignal just before it) syncs on it, and decodes differently from there
    b1, ok1, _, _ = run_p_deviation(st, lost_at=st["copy_first"])
    assert np.array_equal(b1[:4 * n - 1], b[:4 * n - 1]) and not np.array_equal(b1, b)


@pytest.mark.parametrize("fb", [10500, 1200, 600])
def test_rt_family_decodes_what_was_planted_and_splits_at_its_gates(fb):
    oq = fb == 10500
    for m in fs.rt_family(fb):
        pk, tr = run_rt(fb, m)
        if "planted" in m:
            assert len(pk) == len(m["planted"]), m["tag"]
            for p, (typ, nsus, info) in zip(pk, m["planted"]):
                assert p["type"] == typ and p["nsus"] == nsus, m["tag"]
                if oq or typ == 1:
                    assert np.array_equal(p["bytes"][:len(info)], info), m["tag"]
        if "accepted" in m:
            assert len(pk) == sum(m["accepted"]), (m["tag"], m["fills"], len(pk))
        if m["tag"].startswith("rt-uw"):
            assert len(pk) == (2 if m["uw_errors"] == 4 else 0), m["tag"]
    fills = sorted({f for m in fs.rt_family(fb) if "fills" in m for f in m["fills"]})
    edge = (230 if oq else 250) - (64 if oq else 32)
    assert edge in fills and edge + 1 in fills and min(fills) == 0 and max(fills) == 400
    if oq:                                                        # the longest T packet fills the whole block
        assert any(m["tag"] == "rt-t-30-31" for m in fs.rt_family(fb))


def test_c_family_splits_at_the_detector_tolerance():
    fam = {m["tag"]: m for m in fs.c_family()}
    su0, ok0, v0 = run_c(fam["c-shift-0"])
    assert len(su0) >= 5 and ok0.sum() >= 10
    for t, m in fam.items():
        if t.startswith("c-shift-"):                              # filler in front (either arm first) changes nothing
            su, ok, v = run_c(m)
            assert np.array_equal(su, su0) and np.array_equal(ok, ok0) and np.array_equal(v, v0), t
    body = fam["c-pre-norm-6"]
    base = run_c(dict(body, soft=fs.c_source()[fs.c_sync_points(fs.c_source())[0] - 120:], cuts=[len(body["soft"])], lost=set()))
    for inv in ("norm", "inv"):
        n6 = len(run_c(fam["c-pre-%s-6" % inv])[0]); n7 = len(run_c(fam["c-pre-%s-7" % inv])[0])
        assert n6 == len(base[0]) and n7 == n6 - 1, (inv, n6, n7)
    assert len(run_c(fam["c-one-arm"])[0]) == len(base[0]) - 1
    mid = [m for t, m in fam.items() if t.startswith("c-word1-midshift-")]
    assert {(m["word1_hit"], m["word2_lost"]) for m in mid} == {(True, False), (True, True), (False, False)}
    for t, m in fam.items():
        if t.startswith("c-word1-midshift-"):
            assert len(run_c(m)[0]) == len(base[0]) - (1 if m["word2_lost"] else 0), t
    assert len(run_c(fam["c-lost-mid-frame"])[0]) == len(base[0]) - 2
