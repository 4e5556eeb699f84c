"""GPU tests of the C-ABI boundary itself (pytest -m gpu): error returns of every create path, several demodulator
modes alive on one GPU at once (the reference keeps all four demodulators alive, JAERO/mainwindow.cpp:198-237),
queue limits of the frame layer, the ingest router's back-pressure."""
import ctypes
import struct

import numpy as np
import pytest

from conftest import has_cuda, load_excerpt
from oracle import restated

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]


def _import():
    import jaero_b200
    return jaero_b200


def _raw_create(jb, kind, n_channels, fb, Fs, fft_power=14, lockingbw=10500.0):
    s = jb.Settings(kind, fft_power, 8000.0, lockingbw, float(fb), float(Fs), 0.65, 0, 0, 0, 1)
    h = ctypes.c_void_p()
    rc = jb.lib().jaero_batch_create(ctypes.byref(s), n_channels, None, 0, ctypes.byref(h))
    if rc == 0:
        jb.lib().jaero_batch_destroy(h)
    return rc, jb.lib().jaero_last_error().decode()


def test_every_create_error_branch_returns_an_error():
    """Each early exit of jaero_batch_create / jaero_burst_*_create must come back as a negative code with a message and
    leave the process alive (round 1 aborted here: the create guard freed the object a second time)."""
    jb = _import()
    OQ, MSK = jb.KIND_OQPSK, jb.KIND_MSK
    cases = [
        (OQ, 2, 10500, 44100, 14),      # AGC window (4*Fs) fine, fractional delays of T/4, T/8 not representable -> "unsupported"
        (OQ, 2, 10500, 48001, 14),      # AGC / EbNo windows not a multiple of 32 samples
        (OQ, 2, 10500, 192000, 14),     # T/4 = 9.14 samples: delay line longer than the kernels keep
        (MSK, 2, 100, 48000, 13),       # 2*SPS = 960 taps > MAX_TAPS
        (MSK, 2, 600, 48010, 13),       # AGC window not a multiple of 32
        (OQ, 0, 10500, 48000, 14),      # n_channels = 0
        (OQ, 2, 10500, 48000, 9),       # coarsefreqest_fft_power out of range
        (OQ, 2, -1, 48000, 14),         # fb <= 0
        (7, 2, 10500, 48000, 14),       # unknown kind
    ]
    for kind, n, fb, Fs, power in cases:
        rc, msg = _raw_create(jb, kind, n, fb, Fs, power)
        assert rc < 0 and msg, (kind, n, fb, Fs, power, rc, msg)
    for _ in range(3):                   # repeated failures do not corrupt the allocator
        rc, _m = _raw_create(jb, OQ, 2, 10500, 44100)
        assert rc < 0
    with pytest.raises(jb.JaeroError):
        jb.BurstMskBatch(2, fb=1200, Fs=44100)
    with pytest.raises(jb.JaeroError):
        jb.BurstMskBatch(2, fb=300)
    with pytest.raises(jb.JaeroError):
        jb.BurstOqpskBatch(2, fb=8400)
    with pytest.raises(jb.JaeroError):
        jb.PChannelBatch(2, 8400)
    with pytest.raises(jb.JaeroError):
        jb.RTChannelBatch(2, 8400)
    with pytest.raises(jb.JaeroError):
        jb.ViterbiBatch(2, 23)
    # and a good create still works afterwards
    rc, msg = _raw_create(jb, OQ, 2, 10500, 48000)
    assert rc == 0, msg


def test_four_demodulator_modes_alive_at_once(golden):
    """MSK-600, OQPSK-10.5k, burst MSK and burst OQPSK batches created up front and written in an interleaved order: each
    must give exactly the stream it gives alone (= the oracle's). The matched-filter taps are per batch (kernel parameter
    block); a process-global tap table would hand the last-created mode's taps to all of them."""
    jb = _import()
    names = ["msk_600", "oqpsk_10500", "burst_msk_1200_a", "burst_oqpsk_10500"]
    secs = {"msk_600": 8, "oqpsk_10500": 4, "burst_msk_1200_a": 10, "burst_oqpsk_10500": 6}
    objs, pcms, accs, oracles = {}, {}, {}, {}
    for nm in names:                                            # create ALL first
        case = golden[nm]
        pcm = load_excerpt(case.get("excerpt", nm))[:48000 * secs[nm]]
        pcms[nm] = np.stack([pcm, (pcm.astype(np.int32) * 2 // 3).astype(np.int16)])
        kw = dict(case["kw"])
        if case["kind"] == "burst_msk":
            objs[nm] = jb.BurstMskBatch(2, **kw)
        elif case["kind"] == "burst_oqpsk":
            objs[nm] = jb.BurstOqpskBatch(2, **kw)
        else:
            objs[nm] = jb.DemodBatch(case["kind"], 2, **kw)
        accs[nm] = [[], []]
        oracles[nm] = [restated.OracleDemod(case["kind"], **kw) for _ in range(2)]
    chunk = 4800
    nmax = max(p.shape[1] for p in pcms.values())
    for k, a in enumerate(range(0, nmax, chunk)):
        order = names if k % 2 == 0 else names[::-1]           # interleaved, alternating order
        for nm in order:
            x = pcms[nm][:, a:a + chunk]
            if x.shape[1] == 0:
                continue
            objs[nm].write(x)
            for c, s in enumerate(objs[nm].read_softbits()):
                accs[nm][c].append(s)
    for nm in names:
        objs[nm].close()
        for c in range(2):
            o = oracles[nm][c]
            for a in range(0, pcms[nm].shape[1], chunk):
                o.write(pcms[nm][c, a:a + chunk])
            so = o.take_soft(); sg = np.concatenate(accs[nm][c])
            assert len(so) == len(sg) and len(so) > 100, nm
            assert np.array_equal(so < 0, sg < 0) and np.array_equal(so >= 128, sg >= 128), nm
            assert np.abs(so.astype(int) - sg.astype(int)).max(initial=0) <= 1, nm


def test_two_msk_rates_alive_at_once(golden):
    """MSK 600 (160 taps) and MSK 1200 (80 taps) share every kernel and differ only in parameters."""
    jb = _import()
    pcm = load_excerpt("msk_600")[:48000 * 6]
    kw6 = dict(golden["msk_600"]["kw"])
    kw12 = dict(kw6, fb=1200, lockingbw=1800)
    b6 = jb.DemodBatch("msk", 1, **kw6)
    b12 = jb.DemodBatch("msk", 1, **kw12)
    o6 = restated.OracleDemod("msk", **kw6); o12 = restated.OracleDemod("msk", **kw12)
    g6, g12 = [], []
    for a in range(0, len(pcm), 6000):
        x = pcm[None, a:a + 6000]
        b12.write(x); b6.write(x)
        g6.append(b6.read_softbits()[0]); g12.append(b12.read_softbits()[0])
        o6.write(pcm[a:a + 6000]); o12.write(pcm[a:a + 6000])
    st6, st12 = b6.status()[0], b12.status()[0]
    b6.close(); b12.close()
    for g, o, st in ((g6, o6, st6), (g12, o12, st12)):
        so = o.take_soft(); sg = np.concatenate(g)
        assert len(so) == len(sg) and np.array_equal(so >= 128, sg >= 128)
        os_ = o.state()
        for key in ("mixer2_freq", "mse", "agc", "st_wtptr"):
            assert abs(st[key] - os_[key]) <= 1e-6 * max(abs(os_[key]), 1e-9), key
        assert st["softbits"] == len(so)                        # jaero_status.softbits counts what was emitted


def test_pchannel_takes_a_full_soft_ring_and_flags_anything_beyond():
    """One process call may hand over a whole demodulator ring (2 s at 10.5k = 4.2 blocks + the carried partial block):
    same SUs as feeding the oracle; a host call that delivers more than the queue holds raises JAERO_E_OVERFLOW on the
    next read instead of returning corrupted signal units."""
    jb = _import()
    from jaero_b200 import synth
    C = 2
    pcm = np.stack([synth.oqpsk_pchannel_pcm(14, fc=8000.0, seed=5 + c, ebn0_db=12.0) for c in range(C)])
    kw = dict(fb=10500, freq_center=8000.0, lockingbw=10500, fft_power=14, signalthreshold=0.65)
    b = jb.DemodBatch("oqpsk", C, **kw)
    pc = jb.PChannelBatch(C, 10500)
    od = [restated.OracleDemod("oqpsk", **kw) for _ in range(C)]
    op = [restated.OraclePChannel(10500) for _ in range(C)]
    got = [[], []]
    step = 47000                                                 # just under one second per write ...
    for k, a in enumerate(range(0, pcm.shape[1], step)):
        b.write(pcm[:, a:a + step])
        for c in range(C):
            od[c].write(pcm[c, a:a + step])
        if k % 2 == 1:                                           # ... frame layer only every second write: ~20.5k soft bits per call
            pc.process_batch(b)
            for c in range(C):
                op[c].process(od[c].take_soft()); od[c].set_dcd(op[c].dcd)
            for c, r in enumerate(pc.read_sus()):
                got[c].append(r)
    for c in range(C):
        gb = np.concatenate([g[0] for g in got[c]]); gok = np.concatenate([g[1] for g in got[c]])
        rb, rok, _ = op[c].take_sus()
        assert np.array_equal(gb, rb) and np.array_equal(gok, rok) and rok.sum() > 50
    b.close()
    # beyond the queue: 40 000 soft values in one host call (the queue holds floor(21064/4992)+2 = 6 blocks)
    soft = [np.full(40000, 200, dtype=np.int16) for _ in range(C)]
    pc.process_softbits(soft)
    with pytest.raises(jb.JaeroError, match="overflow"):
        pc.read_sus()
    pc.close()


def test_ingest_router_refuses_a_message_that_does_not_fit():
    jb = _import()
    r = jb.IngestRouter(["CHAN0", "CHAN1"], 48000, capacity_samples=1000)
    rate = struct.pack("<I", 48000)
    x = np.arange(600, dtype=np.int16).tobytes()
    assert r.message(b"CHAN0", rate, x) == 0
    with pytest.raises(jb.JaeroError, match="full"):
        r.message(b"CHAN0", rate, x)                             # 1200 > 1000: refused as a whole, nothing filed
    assert r.message(b"CHAN1", rate, x) == 1
    assert r.available == 600                                    # channel 0 still holds exactly the first message
    r.close()


def _gap_stream(name, secs_a, secs_gap, secs_b, seed=3):
    """recording, then low-level noise (the carrier disappears), then the recording again"""
    pcm = load_excerpt(name)
    rng = np.random.default_rng(seed)
    gap = np.round(rng.normal(0, 300.0, size=48000 * secs_gap)).astype(np.int16)
    return np.concatenate([pcm[:48000 * secs_a], gap, pcm[48000 * secs_a:48000 * (secs_a + secs_b)]])


def test_write_batch_is_the_reference_wiring_oqpsk(golden):
    """jaero_pchannel_write_batch = the demodulator and the AeroL connected as JAERO/mainwindow.cpp:198-237,432,508 connects
    them (direct connections): DCD read by FreqOffsetEstimateSlot reflects every soft bit emitted before that sample, and a
    SignalStatus(false) is a LostSignal before any later soft bit. Oracle: the restated demodulator with the restated AeroL
    hooked into its emits (OraclePChannel.wire). A carrier drop in the middle exercises LostSignal and the re-acquisition."""
    jb = _import()
    kw = dict(golden["oqpsk_10500"]["kw"])
    x = _gap_stream("oqpsk_10500", 5, 3, 5)
    pcm2 = np.stack([x, (x.astype(np.int32) * 2 // 3).astype(np.int16)])
    b = jb.DemodBatch("oqpsk", 2, **kw)
    pc = jb.PChannelBatch(2, 10500)
    got = [[], []]
    sizes = [4800, 7000, 1234, 48000, 10000]
    a = 0; k = 0
    while a < pcm2.shape[1]:
        n = min(sizes[k % len(sizes)], pcm2.shape[1] - a)
        pc.write_batch(b, pcm2[:, a:a + n]); a += n; k += 1
        if a % 48000 < n:                                       # the 1 s DCD timer
            pc.tick(b)
        for c, r in enumerate(pc.read_sus()):
            got[c].append(r)
    st = b.status(); dcd, tot, okc = pc.stats()
    b.close(); pc.close()
    for c in range(2):
        od = restated.OracleDemod("oqpsk", **kw); op = restated.OraclePChannel(10500); op.wire(od)
        a = 0; k = 0
        while a < pcm2.shape[1]:
            n = min(sizes[k % len(sizes)], pcm2.shape[1] - a)
            od.write(pcm2[c, a:a + n]); a += n; k += 1
            if a % 48000 < n:
                op.update_dcd(); od.set_dcd(op.dcd)
        rb, rok, _ = op.take_sus()
        gb = np.concatenate([g[0] for g in got[c]]); gok = np.concatenate([g[1] for g in got[c]])
        assert np.array_equal(gb, rb) and np.array_equal(gok, rok) and rok.sum() > 100
        o = od.state()
        assert st[c]["n_sig_false"] == o["n_sig_false"] and st[c]["n_sig_true"] == o["n_sig_true"] and o["n_sig_false"] >= 5
        assert dcd[c] == int(op.dcd)
        for key in ("mixer2_freq", "mse", "agc"):
            assert abs(st[c][key] - o[key]) <= 1e-6 * max(abs(o[key]), 1e-9), key


def test_lost_signal_entry_point(golden):
    """jaero_pchannel_lost_signal == AeroL::LostSignal (aerol.h:921-931): frame counter parked, DCD and its countdown cleared,
    the demodulator told at once; decoding resumes at the next unique word exactly as the oracle's does."""
    jb = _import()
    kw = dict(golden["oqpsk_10500"]["kw"])
    pcm = load_excerpt("oqpsk_10500")[:48000 * 9]
    pcm2 = np.stack([pcm, pcm])
    b = jb.DemodBatch("oqpsk", 2, **kw); pc = jb.PChannelBatch(2, 10500)
    od = restated.OracleDemod("oqpsk", **kw); op = restated.OraclePChannel(10500)
    got = []
    for k, a in enumerate(range(0, pcm2.shape[1], 4800)):
        b.write(pcm2[:, a:a + 4800]); pc.process_batch(b)
        od.set_dcd(op.dcd); od.write(pcm[a:a + 4800]); op.process(od.take_soft())
        if k == 50:
            pc.lost_signal(b, channel=0)                        # channel 0 only; channel 1 carries on
            op.lost_signal(); od.set_dcd(op.dcd)
            assert pc.stats()[0].tolist() == [0, 1] and b.status()[0]["dcd"] == 0 and b.status()[1]["dcd"] == 1
        got.append(pc.read_sus())
    rb, rok, _ = op.take_sus()
    g0 = np.concatenate([g[0][0] for g in got]); ok0 = np.concatenate([g[0][1] for g in got])
    g1 = np.concatenate([g[1][0] for g in got])
    assert np.array_equal(g0, rb) and np.array_equal(ok0, rok)
    assert len(g1) > len(g0)                                    # the frame in flight on channel 0 was dropped, as in the reference
    b.close(); pc.close()


def test_write_batch_msk_signal_units(golden):
    """The same wiring for MSK 1200 (cfg 2 signal). The MSK timing loop reads DCD every sample (mskdemodulator.cpp:387-405), the
    device path switches its gain at the next estimator trigger (<= 2048 samples later than the reference's emit-granular
    switch): decoded signal units and CRC flags still have to come out identical."""
    jb = _import()
    from jaero_b200 import synth
    kw = dict(fb=1200, freq_center=2000.0, lockingbw=1800, fft_power=13, signalthreshold=0.5, afc=False)
    pcm = np.tile(synth.msk_pchannel_pcm(4, fc=2013.0, seed=41, ebn0_db=9.0, fb=1200.0, phase=0.7, delay=9), 4)
    b = jb.DemodBatch("msk", 1, **kw); pc = jb.PChannelBatch(1, 1200)
    od = restated.OracleDemod("msk", **kw); op = restated.OraclePChannel(1200); op.wire(od)
    got = []
    for k, a in enumerate(range(0, len(pcm), 9600)):
        pc.write_batch(b, pcm[None, a:a + 9600]); od.write(pcm[a:a + 9600])
        if k % 5 == 4:
            pc.tick(b); op.update_dcd(); od.set_dcd(op.dcd)
        got.append(pc.read_sus()[0])
    rb, rok, _ = op.take_sus()
    gb = np.concatenate([g[0] for g in got]); gok = np.concatenate([g[1] for g in got])
    assert np.array_equal(gok, rok) and np.array_equal(gb[gok.astype(bool)], rb[rok.astype(bool)]) and rok.sum() >= 60
    b.close(); pc.close()


def _split_vectors(soft, T):
    """The burst demodulators' emits: an optional start-of-burst marker followed by exactly T values (they clear the buffer,
    push -1, then add pairs until >= T: burstmskdemodulator.cpp:735-739, burstoqpskdemodulator.cpp)."""
    out, i = [], 0
    while i < len(soft):
        n = T + (1 if soft[i] < 0 else 0)
        out.append(soft[i:i + n]); i += n
    return out


@pytest.mark.parametrize("name", ["burst_msk_1200_a", "burst_oqpsk_10500"])
def test_rt_vector_mode_drops_the_rest_of_the_vector_like_the_reference(golden, name):
    """jaero_rt_set_vector_mode: AeroL::Decode returns in the middle of a soft-bit vector when the burst time-out fires
    (aerol.cpp:2018-2027). Device path (soft bits never leave the GPU) against the oracle fed vector by vector."""
    jb = _import()
    case = golden[name]
    pcm = load_excerpt(name)
    oq = case["kind"] == "burst_oqpsk"
    T = 32 if oq else 12
    b = (jb.BurstOqpskBatch if oq else jb.BurstMskBatch)(1, **case["kw"])
    rt = jb.RTChannelBatch(1, case["kw"]["fb"]); rt.set_vector_mode(True)
    got = []
    for a in range(0, len(pcm), 48000):
        b.write(pcm[None, a:a + 48000]); rt.process_burst(b)
        got += rt.read_packets()[0]
    tr, bad, dcd = rt.stats()
    b.close(); rt.close()
    o = restated.OracleDemod(case["kind"], **case["kw"]); ort = restated.OracleRTChannel(case["kw"]["fb"])
    nvec = 0
    for a in range(0, len(pcm), 48000):
        o.write(pcm[a:a + 48000])
        for v in _split_vectors(o.take_soft(), T):
            ort.process(v, vector_semantics=True); nvec += 1
    ref = ort.packets()
    assert nvec > 50 and len(ref) == len(got) and len(ref) >= 1 and tr[0] == ort.trials
    for r, g in zip(ref, got):
        assert r["type"] == g["type"] and r["nsus"] == g["nsus"] and np.array_equal(r["bytes"], g["bytes"])
    # host-supplied soft bits: every call is one vector
    streams = __import__("conftest").synthetic_r_packet_stream(1200, (np.arange(17) * 5 % 256).astype(np.uint8))
    rt2 = jb.RTChannelBatch(1, 1200); rt2.set_vector_mode(True); ort2 = restated.OracleRTChannel(1200)
    for a in range(0, len(streams), 40):
        rt2.process([streams[a:a + 40]]); ort2.process(streams[a:a + 40], vector_semantics=True)
    g2 = rt2.read_packets()[0]; r2 = ort2.packets()
    rt2.close()
    assert len(g2) == len(r2) and all(np.array_equal(x["bytes"], y["bytes"]) for x, y in zip(g2, r2))


def test_status_telemetry_peak_volume_and_scatter_points(golden):
    """PeakVolume (max |sample| since the previous read-out) and the decimated ScatterPoints in jaero_status."""
    jb = _import()
    kw = dict(golden["oqpsk_10500"]["kw"])
    pcm = load_excerpt("oqpsk_10500")[:48000 * 4]
    pcm2 = np.stack([pcm, (pcm // 2).astype(np.int16), np.zeros_like(pcm)])
    b = jb.DemodBatch("oqpsk", 3, **kw)
    b.write(pcm2[:, :100000])
    st = b.status()
    for c in range(3):
        assert st[c]["peak_volume"] == np.abs(pcm2[c, :100000].astype(int)).max() / 32768.0
    b.write(pcm2[:, 100000:100001])                                    # the read-out restarted the maximum
    assert b.status()[0]["peak_volume"] == abs(int(pcm2[0, 100000])) / 32768.0
    b.write(pcm2[:, 100001:])
    st = b.status()
    pts = np.array(st[0]["scatter"][:]).reshape(2, 2)
    assert np.all(np.abs(np.abs(pts) - 1.0) < 0.6)                      # locked OQPSK constellation points sit near (+-1, +-1)
    assert list(st[2]["scatter"][:]) != list(st[0]["scatter"][:])
    b.close()


def test_regrouping_never_changes_results(golden):
    """The 10500 bps kernel may seat channels in any lane (the library regroups them by symbol-timing phase for speed): soft
    bits and loop state must be bit-identical whatever the seating and whenever it changes - random permutations in the middle
    of the stream, phase regrouping on request, and the library's own schedule alone."""
    jb = _import()
    kw = dict(golden["oqpsk_10500"]["kw"])
    pcm = load_excerpt("oqpsk_10500")[:48000 * 5]
    C = 70
    rng = np.random.default_rng(7)
    variants = np.stack([pcm, (pcm.astype(np.int32) * 2 // 3).astype(np.int16), np.roll(pcm, 5), np.roll(pcm, 123), pcm[::-1].copy()])
    idx = rng.integers(0, 5, size=C)
    pcm2 = np.ascontiguousarray(variants[idx])

    def run(mode):
        b = jb.DemodBatch("oqpsk", C, **kw)
        acc = [[] for _ in range(C)]
        step = 90000 if mode == "long_writes" else 7000                 # long_writes: the scheduled seating (epoch 34) falls between two launches inside the second call
        for k, a in enumerate(range(0, pcm2.shape[1], step)):
            if mode == "random" and k % 3 == 1:
                b.regroup(rng.permutation(C))
            if mode == "phase" and k == 20:
                b.regroup()
            b.write(pcm2[:, a:a + step])
            if k % 4 == 3 or mode == "long_writes":
                for c, s in enumerate(b.read_softbits()):
                    acc[c].append(s)
        for c, s in enumerate(b.read_softbits()):
            acc[c].append(s)
        st = b.status()
        b.close()
        return [np.concatenate(x) for x in acc], st

    ref, st_ref = run("scheduled")            # the library's own seating check only: epoch 34 of the ~58 (the next is at 66)
    for mode in ("random", "phase", "long_writes"):
        got, st = run(mode)
        for c in range(C):
            assert np.array_equal(got[c], ref[c]), (mode, c)
            for key in ("mixer2_wtptr", "st_wtptr", "mse", "agc", "ebno", "mixer2_freq"):
                assert st[c][key] == st_ref[c][key], (mode, c, key)
    so, sto = restated.OracleDemod("oqpsk", **kw), None
    so.write(variants[idx[C - 1]])
    assert np.array_equal(so.take_soft() >= 128, ref[C - 1] >= 128)
