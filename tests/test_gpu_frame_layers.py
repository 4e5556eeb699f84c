"""The P-, C- and R/T-channel frame layers on the device against the restated oracle (one oracle object per channel) on the
constructed streams of tests/frame_streams.py, at 1, 33 and 300 channels: channel c carries family member c mod M with its
own cut sequence, so in one call channels complete different numbers of blocks, frames and packets. Every field both sides
expose is compared bit for bit after every read. Then the per-call limits: at capacity the output equals the oracle's, one
past it the next read reports the overflow, and the layer recovers on the read after."""
import ctypes

import numpy as np
import pytest

import frame_streams as fs
from conftest import has_cuda
from oracle import restated

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]
TICK = 4                     # a global AeroL::updateDCD after every TICK-th call
LOST_ALL = 5                 # P and C mutation runs: LostSignal on every channel at once after this call
E_OVERFLOW = -4


def _limits():
    """the per-call and per-read limits as the layers define them (jaero_b200/csrc/frame_layers.cuh)"""
    import os
    import re
    from conftest import ROOT
    with open(os.path.join(ROOT, "jaero_b200", "csrc", "frame_layers.cuh")) as fh:
        src = fh.read()
    return {k: int(re.search(r"static const int %s = (\d+);" % k, src).group(1)) for k in ("RT_SLOTS", "RT_OUT", "CC_QUEUE", "CC_OUT")}


LIMITS = _limits()


def _jb():
    import jaero_b200
    return jaero_b200


def _chunks(ms, pos, r):
    out = []
    for c, m in enumerate(ms):
        n = m["cuts"][r] if r < len(m["cuts"]) else 0
        out.append(m["soft"][pos[c]:pos[c] + n]); pos[c] += n
    return out


# ------------------------------------------------------------------------------------------------ P-channel
def device_dcd(calls):
    """The DCD the device reports after each call, from what the reference did in it: calls = [(syncs, crc_ok of the units
    completed in the call, in order, tick after it, LostSignal after it)]. The device applies the units' CRC-driven countdown
    updates (aerol.cpp:1601-1608) at the end of the call, after every UW sync of the call has set the countdown to 12
    (DESIGN.md section 8); the reference applies them at the frame's last bit. Ticks and LostSignals between calls are the
    reference's (AeroL::updateDCD, AeroL::LostSignal)."""
    cd, dcd, out = 0, 0, []
    for syncs, oks, tick, lost in calls:
        if syncs:
            cd, dcd = 12, 1
        for ok in oks:
            if ok:
                if cd < 12:
                    cd += 2
            elif cd > 0:
                cd -= 3
            if not dcd and cd > 2:
                dcd = 1
        if tick:
            if cd > 0:
                cd -= 3
            elif cd < 0:
                cd = 0
            if dcd and not cd:
                dcd = 0
        if lost:
            cd, dcd = 0, 0
        out.append(dcd)
    return np.array(out)


def oracle_p(fb, m, rounds, lost_all=None, lost_at=None, ticks=None):
    """the reference under the member's schedule (a tick after every TICK-th call, or after the calls in `ticks`); lost_at:
    a LostSignal just before that stream index as well"""
    o = restated.OraclePChannel(fb)
    a, dcd, calls, acc = 0, [], [], []
    for r in range(rounds):
        n = m["cuts"][r] if r < len(m["cuts"]) else 0
        seg = m["soft"][a:a + n]
        s0 = o.syncs
        if lost_at is not None and a <= lost_at < a + n:
            o.process(seg[:lost_at - a]); o.lost_signal(); o.process(seg[lost_at - a:])
        else:
            o.process(seg)
        a += n
        b, ok, fr = o.take_sus()
        acc.append((b, ok, fr))
        tick = (r in ticks) if ticks is not None else r % TICK == TICK - 1
        lost = r in m["lost"] or r == lost_all
        if tick:
            o.update_dcd()
        if lost:
            o.lost_signal()
        dcd.append(int(o.dcd))
        calls.append((o.syncs - s0, list(ok), tick, lost))
    o.close()
    b, ok, fr = (np.concatenate([x[i] for x in acc]) for i in range(3))
    idx = np.zeros(len(fr), dtype=np.int64)                      # index of each unit in its frame
    for k in range(1, len(fr)):
        idx[k] = idx[k - 1] + 1 if fr[k] == fr[k - 1] else 0
    return dict(b=b, ok=ok, fr=fr, idx=idx, dcd=np.array(dcd), device_dcd=device_dcd(calls))


def run_p(fb, fam, C, perm=None, lost_all=None):
    jb = _jb()
    M = len(fam)
    sel = [(perm[c] if perm is not None else c) % M for c in range(C)]
    ms = [fam[k] for k in sel]
    R = max(len(m["cuts"]) for m in ms)
    pc = jb.PChannelBatch(C, fb)
    pos = [0] * C
    got = [[] for _ in range(C)]
    dcd = []
    for r in range(R):
        pc.process_softbits(_chunks(ms, pos, r))
        if r % TICK == TICK - 1:
            pc.tick()
        for c, m in enumerate(ms):
            if r in m["lost"]:
                pc.lost_signal(channel=c)
        if r == lost_all:
            pc.lost_signal()
        dcd.append(pc.stats()[0].copy())
        if r % 3 == 2 or r == R - 1:
            for c, x in enumerate(pc.read_sus()):
                got[c].append(x)
    _, tot, okc = pc.stats()
    pc.close()
    return sel, R, got, np.array(dcd), tot, okc


@pytest.mark.parametrize("C", [1, 33, 300])
@pytest.mark.parametrize("fb,family", [(10500, "offset"), (1200, "offset"), (600, "offset"),
                                       (10500, "mutation"), (1200, "mutation"), (600, "mutation")])
def test_pchannel_matches_the_oracle(fb, family, C):
    fam = fs.p_offset_family(fb) if family == "offset" else fs.p_mutation_family(fb)
    lost_all = LOST_ALL if family == "mutation" else None
    sel, R, got, dcd, tot, okc = run_p(fb, fam, C, lost_all=lost_all)
    ref = {}
    n_diverged = 0
    for c, k in enumerate(sel):
        if k not in ref:
            ref[k] = oracle_p(fb, fam[k], R, lost_all=lost_all)
        o = ref[k]
        b = np.concatenate([g[0] for g in got[c]]); ok = np.concatenate([g[1] for g in got[c]])
        idx = np.concatenate([g[2] for g in got[c]]); fr = np.concatenate([g[3] for g in got[c]])
        tag = fam[k]["tag"]
        if not (len(b) == len(o["b"]) and np.array_equal(b, o["b"])) and "plant_first" in fam[k]:
            # A UW copy that the reference ignores because its DCD is up, while the device's is still down (its countdown
            # updates land later in the call, DESIGN.md section 8): the device syncs on it. It then decodes what the
            # reference decodes when it is made to search there, LostSignal just before the copy.
            assert fb == 10500 and fam[k]["plant_d"] <= -68, tag
            o = oracle_p(fb, fam[k], R, lost_all=lost_all, lost_at=fam[k]["plant_first"])
            n_diverged += 1
        assert np.array_equal(b, o["b"]) and np.array_equal(ok, o["ok"]), tag
        assert np.array_equal(idx, o["idx"]) and np.array_equal(fr, o["fr"] % 65536), tag     # frame number modulo 2^16
        assert tot[c] == len(o["ok"]) and okc[c] == o["ok"].sum(), tag
        # DCD after every call: the reference's wherever the countdown order does not matter, and exactly the documented
        # deviation where it does
        assert np.array_equal(dcd[:, c], o["device_dcd"]), tag


def _oracle_p_deviation(st, lost_at=None):
    """the reference over p_dcd_deviation_stream's schedule (one tick, after call 0); lost_at: a LostSignal just before that
    stream index, which makes it search where the device searches. -> (units, crc flags, frames, DCD, device DCD)"""
    o = oracle_p(10500, dict(st, lost=set()), len(st["cuts"]), lost_at=lost_at, ticks=st["ticks"])
    return o["b"], o["ok"], o["fr"] % 65536, list(o["dcd"]), list(o["device_dcd"])


def test_pchannel_dcd_deviation_is_only_the_predicted_one():
    """The known deviation (DESIGN.md section 8): DCD is down with the counter running, a frame's good CRCs raise it, and the
    next frame, in the same call, carries an exact UW copy in its data region. Up to that frame the device is the reference;
    the reference ignores the copy; the device syncs on it and from there decodes exactly what the reference decodes when it
    is made to search at the copy. Without the copy the device is the reference throughout."""
    jb = _jb()
    st, st0 = fs.p_dcd_deviation_stream(), fs.p_dcd_deviation_stream(copy=False)
    pc = jb.PChannelBatch(2, 10500)
    got = [[], []]
    dcd = []
    a = 0
    for k, n in enumerate(st["cuts"]):
        pc.process_softbits([st0["soft"][a:a + n], st["soft"][a:a + n]]); a += n
        if k in st["ticks"]:
            pc.tick()
        dcd.append(pc.stats()[0].copy())
        for c, x in enumerate(pc.read_sus()):
            got[c].append(x)
    pc.close()
    dcd = np.array(dcd)
    dev = [[np.concatenate([g[i] for g in got[c]]) for i in (0, 1, 3)] for c in range(2)]
    ref0, ref, emu = _oracle_p_deviation(st0), _oracle_p_deviation(st), _oracle_p_deviation(st, lost_at=st["copy_first"])
    n = 26
    assert ref[3] == [0, 0, 1, 1] and ref[1][3 * n - 1:4 * n - 1].all()           # DCD down, then raised by frame 3's CRCs
    for x, y in zip(ref[:3], ref0[:3]):                                          # the reference ignores the copy
        assert np.array_equal(x, y)
    for x, y in zip(dev[0], ref0[:3]):                                           # no copy: the device is the reference
        assert np.array_equal(x, y)
    assert list(dcd[:, 0]) == ref0[4]                                            # DCD: the documented countdown order
    for x, y in zip(dev[1], emu[:3]):                                            # copy: the device syncs on it
        assert np.array_equal(x, y)
    assert list(dcd[:, 1]) == emu[4]
    assert np.array_equal(dev[1][0][:4 * n - 1], ref[0][:4 * n - 1]) and not np.array_equal(dev[1][0], ref[0])


def test_pchannel_channel_order_does_not_matter():
    fam = fs.p_mutation_family(10500)
    C = 33
    _, _, got, _, _, _ = run_p(10500, fam, C)
    perm = np.random.default_rng(7).permutation(C)
    sel2, _, got2, _, _, _ = run_p(10500, fam, C, perm=perm)
    for c in range(C):
        a = [np.concatenate([g[i] for g in got[perm[c]]]) for i in range(4)]
        b = [np.concatenate([g[i] for g in got2[c]]) for i in range(4)]
        assert all(np.array_equal(x, y) for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------------ C-channel
def oracle_c(m, rounds, lost_all=None):
    o = restated.OracleCChannel()
    a, dcd = 0, []
    for r in range(rounds):
        n = m["cuts"][r] if r < len(m["cuts"]) else 0
        o.process(m["soft"][a:a + n]); a += n
        if r % TICK == TICK - 1:
            o.update_dcd()
        if r in m["lost"] or r == lost_all:
            o.lost_signal()
        dcd.append(int(o.dcd))
    su, ok, voice = o.take_frames()
    o.close()
    return su, ok, voice, np.array(dcd)


def run_c(fam, C, perm=None, lost_all=None):
    jb = _jb()
    sel = [(perm[c] if perm is not None else c) % len(fam) for c in range(C)]
    ms = [fam[k] for k in sel]
    R = max(len(m["cuts"]) for m in ms)
    cc = jb.CChannelBatch(C)
    pos = [0] * C
    got = [[] for _ in range(C)]
    dcd = []
    for r in range(R):
        cc.process(_chunks(ms, pos, r))
        if r % TICK == TICK - 1:
            cc.tick()
        for c, m in enumerate(ms):
            if r in m["lost"]:
                cc.lost_signal(channel=c)
        if r == lost_all:
            cc.lost_signal()
        dcd.append(cc.stats()[0].copy())
        for c, x in enumerate(cc.read_frames()):
            got[c].append(x)
    _, tot, okc = cc.stats()
    cc.close()
    out = [[np.concatenate([g[i] for g in got[c]]) for i in range(4)] for c in range(C)]
    return sel, R, out, np.array(dcd), tot, okc


@pytest.mark.parametrize("lost_all", [None, LOST_ALL])
@pytest.mark.parametrize("C", [1, 33, 300])
def test_cchannel_matches_the_oracle(C, lost_all):
    fam = fs.c_family()
    sel, R, out, dcd, tot, okc = run_c(fam, C, lost_all=lost_all)
    ref = {}
    for c, k in enumerate(sel):
        if k not in ref:
            ref[k] = oracle_c(fam[k], R, lost_all)
        su, ok, voice, odcd = ref[k]
        tag = fam[k]["tag"]
        gsu, gok, gv, gfr = out[c]
        assert gsu.shape == su.shape and np.array_equal(gsu, su) and np.array_equal(gok, ok) and np.array_equal(gv, voice), tag
        assert np.array_equal(gfr, np.arange(len(su))), tag
        assert np.array_equal(dcd[:, c], odcd), tag
        assert tot[c] == ok.size and okc[c] == ok.sum(), tag


def test_cchannel_channel_order_does_not_matter():
    fam = fs.c_family()
    C = 33
    _, _, out, _, _, _ = run_c(fam, C)
    perm = np.random.default_rng(8).permutation(C)
    _, _, out2, _, _, _ = run_c(fam, C, perm=perm)
    for c in range(C):
        assert all(np.array_equal(x, y) for x, y in zip(out[perm[c]], out2[c]))


# ------------------------------------------------------------------------------------------------ R/T
def oracle_rt(fb, m, vector):
    o = restated.OracleRTChannel(fb)
    a, tr = 0, []
    for n in m["cuts"]:
        o.process(m["soft"][a:a + n], vector); a += n
        tr.append(o.trials)
    pk = o.packets()
    o.close()
    return pk, tr


def run_rt(fb, fam, C, vector, perm=None):
    jb = _jb()
    sel = [(perm[c] if perm is not None else c) % len(fam) for c in range(C)]
    ms = [fam[k] for k in sel]
    R = max(len(m["cuts"]) for m in ms)
    rt = jb.RTChannelBatch(C, fb)
    rt.set_vector_mode(vector)
    pos = [0] * C
    got = [[] for _ in range(C)]
    trials = []
    for r in range(R):
        rt.process(_chunks(ms, pos, r))
        for c, pk in enumerate(rt.read_packets()):
            got[c] += pk
        trials.append(rt.stats()[0].copy())
    rt.close()
    return sel, got, np.array(trials)


@pytest.mark.parametrize("vector", [False, True])
@pytest.mark.parametrize("C", [1, 33, 300])
@pytest.mark.parametrize("fb", [10500, 1200, 600])
def test_rt_matches_the_oracle(fb, C, vector):
    fam = fs.rt_family(fb)
    sel, got, trials = run_rt(fb, fam, C, vector)
    ref = {}
    for c, k in enumerate(sel):
        if k not in ref:
            ref[k] = oracle_rt(fb, fam[k], vector)
        pk, tr = ref[k]
        m = fam[k]
        assert len(got[c]) == len(pk), m["tag"]
        for g, p in zip(got[c], pk):
            assert g["type"] == p["type"] and g["nsus"] == p["nsus"] and np.array_equal(g["bytes"], p["bytes"]), m["tag"]
            # The two sides stamp a packet differently. Both count the soft values the layer took (start-of-burst markers
            # included, values dropped in vector mode excluded). The device gives the count up to and including the first value
            # of the packet's block; the oracle the count up to the value that completed the trial which decoded it. That trial
            # took 16 (n + 1) values for a packet of n bytes (R: 19 of 20 decoded bytes kept; T: the last byte chopped).
            assert p["bit_index"] == g["start_bit"] + 16 * (len(p["bytes"]) + 1) - 1, m["tag"]
        assert np.array_equal(trials[:len(m["cuts"]), c], tr), m["tag"]


@pytest.mark.parametrize("fb", [10500, 1200])
def test_rt_channel_order_does_not_matter(fb):
    fam = fs.rt_family(fb)
    C = 33
    _, got, tr = run_rt(fb, fam, C, False)
    perm = np.random.default_rng(9).permutation(C)
    _, got2, tr2 = run_rt(fb, fam, C, False, perm=perm)
    for c in range(C):
        assert len(got[perm[c]]) == len(got2[c]) and np.array_equal(tr[:, perm[c]], tr2[:, c])
        for g, h in zip(got[perm[c]], got2[c]):
            assert g["type"] == h["type"] and g["nsus"] == h["nsus"] and g["start_bit"] == h["start_bit"]
            assert np.array_equal(g["bytes"], h["bytes"])


# ------------------------------------------------------------------------------------------------ limits and recovery
def _read_rt_raw(rt, cap=None):
    """the C ABI read, which hands over what it holds even when it reports an overflow -> (rc, per channel [(start, bytes)])"""
    jb = _jb()
    cap = cap or LIMITS["RT_OUT"]
    out = np.zeros((rt.n, cap, rt.RECORD), dtype=np.uint8)
    counts = np.zeros(rt.n, dtype=np.int32)
    rc = jb.lib().jaero_rt_read_packets(rt.h, out.ctypes.data_as(ctypes.c_void_p), cap, counts.ctypes.data_as(ctypes.c_void_p))
    recs = []
    for c in range(rt.n):
        r = []
        for k in range(counts[c]):
            h = out[c, k, :16].view(np.int32)
            r.append((int(h[3]), out[c, k, 16:16 + int(h[2])].tobytes()))
        recs.append(r)
    return rc, recs


def _read_cc_raw(cc, cap=None):
    jb = _jb()
    cap = cap or LIMITS["CC_OUT"]
    out = np.zeros((cc.n, cap, cc.RECORD), dtype=np.uint8)
    counts = np.zeros(cc.n, dtype=np.int32)
    rc = jb.lib().jaero_cchannel_read_frames(cc.h, out.ctypes.data_as(ctypes.c_void_p), cap, counts.ctypes.data_as(ctypes.c_void_p))
    return rc, [out[c, :counts[c]] for c in range(cc.n)]


def test_rt_slot_limit_which_packet_is_lost_and_recovery():
    """A call can open as many new packets as there are slots less the one carried in (the packet being filled when the call
    starts; a fresh layer carries its initial block). That many UWs in one call decode as the oracle decodes them; with one
    more, the packet being filled when the extra UW arrives is lost and the read reports it; the read after that succeeds
    and the packets that follow are the oracle's. Each packet starts at the value after its UW's last bit."""
    jb = _jb()
    fb, C = 1200, 33
    n_new = LIMITS["RT_SLOTS"] - 1
    soft, payloads, uw_last = fs.rt_many_packets(fb, n_new + 3)
    bounds = list(np.nonzero(soft == -1)[0]) + [len(soft)]      # burst k = soft[bounds[k]:bounds[k + 1]]
    o = restated.OracleRTChannel(fb); o.process(soft); ref = [p["bytes"].tobytes() for p in o.packets()]; o.close()
    assert [r[:17] for r in ref] == [p[:17].tobytes() for p in payloads]
    start = [u + 2 for u in uw_last]                             # values counted from 1: the one after the UW
    # capacity
    rt = jb.RTChannelBatch(C, fb)
    rt.process([soft[:bounds[n_new]]] * C)
    rc, recs = _read_rt_raw(rt)
    assert rc == 0 and all(r == [(start[k], ref[k]) for k in range(n_new)] for r in recs)
    rt.close()
    # one past: packet n_new - 1 is the one lost
    rt = jb.RTChannelBatch(C, fb)
    rt.process([soft[:bounds[n_new + 1]]] * C)
    rc, recs = _read_rt_raw(rt)
    assert rc == E_OVERFLOW
    kept = [k for k in range(n_new + 1) if k != n_new - 1]
    assert all(r == [(start[k], ref[k]) for k in kept] for r in recs)
    rt.process([soft[bounds[n_new + 1]:]] * C)
    rc, recs = _read_rt_raw(rt)
    assert rc == 0 and all(r == [(start[k], ref[k]) for k in (n_new + 1, n_new + 2)] for r in recs)
    rt.close()


def test_rt_output_ring_limit_and_recovery():
    """RT_OUT packets may wait unread; one more is lost and reported; the next read succeeds with the packets after it."""
    jb = _jb()
    fb, C = 1200, 33
    n_out = LIMITS["RT_OUT"]
    soft, _, uw_last = fs.rt_many_packets(fb, n_out + 4, seed=9)
    bounds = list(np.nonzero(soft == -1)[0]) + [len(soft)]
    o = restated.OracleRTChannel(fb); o.process(soft); ref = [(u + 2, p["bytes"].tobytes()) for u, p in zip(uw_last, o.packets())]; o.close()
    assert len(ref) == n_out + 4
    half = n_out // 2 + 1                                        # fewer new packets per call than the slots allow
    rt = jb.RTChannelBatch(C, fb)
    rt.process([soft[:bounds[half]]] * C); rt.process([soft[bounds[half]:bounds[n_out]]] * C)
    rc, recs = _read_rt_raw(rt)
    assert rc == 0 and all(r == ref[:n_out] for r in recs)      # exactly full
    rt.close()
    rt = jb.RTChannelBatch(C, fb)
    rt.process([soft[:bounds[half]]] * C); rt.process([soft[bounds[half]:bounds[n_out + 1]]] * C)   # one more unread
    rc, recs = _read_rt_raw(rt)
    assert rc == E_OVERFLOW and all(r == ref[:n_out] for r in recs)
    rt.process([soft[bounds[n_out + 1]:]] * C)
    rc, recs = _read_rt_raw(rt)
    assert rc == 0 and all(r == ref[n_out + 1:] for r in recs)
    rt.close()


def _c_stream():
    """the recording's soft bits followed by its frames once more (enough frames for the queue and the output ring) ->
    (soft, ends): ends[k] is the length of the prefix whose last value completes frame k, a sync bit + 4096 + 1"""
    src = fs.c_source()
    t0 = fs.c_sync_points(src)[0]
    src = np.concatenate([src, src[t0 - 120:]])
    syncs = fs.c_sync_points(src)
    coarse, step = [], 50                                        # the oracle's frames, located to within 50 values
    o = restated.OracleCChannel()
    n = 0
    for a in range(0, len(src), step):
        o.process(src[a:a + step])
        k = int(restated.lib().jor_cchan_frame_count(o.h))
        coarse += [min(a + step, len(src))] * (k - n); n = k
    o.close()
    ends = []
    for e in coarse:
        hit = [t + 4097 for t in syncs if e - step < t + 4097 <= e]
        assert len(hit) == 1
        ends.append(hit[0])
    return src, ends


def _frames(recs):
    g = np.array(recs)
    s = g[:, :48].reshape(-1, 3, 16)
    return s[:, :, :12], s[:, :, 12].astype(np.int32), g[:, 48:348], g[:, 348:352].copy().view(np.int32).reshape(-1)


def test_cchannel_queue_limit_and_recovery():
    """CC_QUEUE frames may complete in one call. That many plus the start of the next in one call decode as the oracle
    decodes them (the next finishes in the following call); one more in one call is lost, the read reports it, and the read
    after that succeeds with what the oracle decodes from the same stream without the lost frame."""
    jb = _jb()
    src, end = _c_stream()
    Q = LIMITS["CC_QUEUE"]
    C = 33
    o = restated.OracleCChannel(); o.process(src); su, ok, voice = o.take_frames(); o.close()
    assert len(su) == len(end) >= Q + 4
    # capacity: frames 0 .. Q-1 and the start of frame Q in one call
    cc = jb.CChannelBatch(C)
    a = end[Q] - 1500
    assert end[Q - 1] < a
    calls = [a] + [840] * (-(-(len(src) - a) // 840))
    got = [[] for _ in range(C)]
    p = 0
    for n in calls:
        cc.process([src[p:p + n]] * C); p += n
        rc, recs = _read_cc_raw(cc)
        assert rc == 0
        for c in range(C):
            got[c] += list(recs[c])
    cc.close()
    for c in range(C):
        gs, gok, gv, gfr = _frames(got[c])
        assert np.array_equal(gs, su) and np.array_equal(gok, ok) and np.array_equal(gv, voice)
        assert np.array_equal(gfr, np.arange(len(su)))
    # one past: frames 0 .. Q complete in one call; frame Q is lost
    cc = jb.CChannelBatch(C)
    cc.process([src[:end[Q]]] * C)
    rc, recs = _read_cc_raw(cc)
    assert rc == E_OVERFLOW and all(len(r) == Q for r in recs)
    rest = [[] for _ in range(C)]
    p = end[Q]
    while p < len(src):
        cc.process([src[p:p + 840]] * C); p += 840
        rc, recs = _read_cc_raw(cc)
        assert rc == 0
        for c in range(C):
            rest[c] += list(recs[c])
    cc.close()
    # the oracle without frame Q: from the value after frame Q-1 to the value that completes frame Q (its preamble and body;
    # an even count, so both arms keep their roles)
    assert (end[Q] - end[Q - 1]) % 2 == 0
    o = restated.OracleCChannel(); o.process(np.concatenate([src[:end[Q - 1]], src[end[Q]:]]))
    su2, ok2, voice2 = o.take_frames(); o.close()
    assert len(su2) == len(su) - 1
    for c in range(C):
        gs, gok, gv, gfr = _frames(rest[c])
        assert np.array_equal(gs, su2[Q:]) and np.array_equal(gok, ok2[Q:]) and np.array_equal(gv, voice2[Q:])
        assert np.array_equal(gfr, np.arange(Q, len(su2)))


def test_cchannel_output_ring_limit_and_recovery():
    """CC_OUT frames may wait unread; one more is lost and reported; the next read succeeds with the frames after it."""
    jb = _jb()
    src, end = _c_stream()
    n_out = LIMITS["CC_OUT"]
    o = restated.OracleCChannel(); o.process(src); su, ok, voice = o.take_frames(); o.close()
    assert len(su) >= n_out + 3
    C = 33
    stops = list(range(2, n_out + 1, 3))                         # fewer frames per call than the queue takes
    if stops[-1] != n_out:
        stops.append(n_out)
    cc = jb.CChannelBatch(C)
    p = 0
    for k in stops:                                              # n_out + 1 frames unread
        cc.process([src[p:end[k]]] * C); p = end[k]
    rc, recs = _read_cc_raw(cc)
    assert rc == E_OVERFLOW and all(len(r) == n_out for r in recs)
    for r in recs:
        gs, gok, gv, gfr = _frames(r)
        assert np.array_equal(gs, su[:n_out]) and np.array_equal(gok, ok[:n_out]) and np.array_equal(gv, voice[:n_out])
    cc.process([src[p:]] * C)
    rc, recs = _read_cc_raw(cc)
    assert rc == 0
    for r in recs:
        gs, gok, gv, gfr = _frames(r)
        assert np.array_equal(gs, su[n_out + 1:]) and np.array_equal(gok, ok[n_out + 1:]) and np.array_equal(gv, voice[n_out + 1:])
        assert np.array_equal(gfr, np.arange(n_out + 1, len(su)))
