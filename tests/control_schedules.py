"""Run-time control schedules for the continuous demodulators: CenterFreqChangedSlot, setAFC, setSQL, setCPUReduce and
DataCarrierDetect calls at chosen sample indices of the committed recordings, placed so that every branch of the centre
change and every way the flags are read is reached (tests/test_demod_controls_cpu.py checks that they are).

An event is (sample_index, [(name, *args), ...], tag): oracle.restated.write_plan cuts the writes at each event and makes
its calls before the write that starts there. `tag` names the branch the event is there for."""

# recording -> (kind, create-time settings, seconds by which the carrier is locked)
RECORDINGS = {
    "oqpsk_10500": ("oqpsk", dict(fb=10500, freq_center=5760, lockingbw=10500, fft_power=14, signalthreshold=0.65, afc=True), 0.5),
    "oqpsk_8400": ("oqpsk", dict(fb=8400, freq_center=8000, lockingbw=10500, fft_power=14, signalthreshold=0.65, afc=True), 3.4),
    "msk_600": ("msk", dict(fb=600, freq_center=1000, lockingbw=900, fft_power=13, signalthreshold=0.5, afc=True), 2.6),
    "msk_1200": ("msk", dict(fb=1200, freq_center=2000, lockingbw=1800, fft_power=13, signalthreshold=0.5, afc=True), 1.8),
}
# synthetic streams (the 8000 bps single-warp kernel has no recording): name -> (kind, settings, seconds to lock)
SYNTHETIC = {
    "oqpsk_8000": ("oqpsk", dict(fb=8000, freq_center=6000, lockingbw=8000, fft_power=14, signalthreshold=0.65, afc=True), 0.5),
}
FS = 48000


def synthetic_stream(name):
    """6 s of random 8000 bps OQPSK at 6 kHz, Eb/N0 12 dB (the stream of test_oqpsk_parity_below_8400_bps)"""
    assert name == "oqpsk_8000"
    import numpy as np
    from jaero_b200 import synth
    rng = np.random.default_rng(8000)
    env = synth.oqpsk_envelope(rng.integers(0, 2, size=8000 * 6, dtype=np.uint8), 8000.0)
    return synth.to_passband_int16(env, 6000.0, ebn0_db=12.0, fb=8000.0, rng=rng)


def trigger_every(kw, cpu_reduce=False):
    """samples between coarse-estimator triggers (oqpskdemodulator.cpp:415): the ring's trigger samples are k * this - 1"""
    n = 1 << kw["fft_power"]
    return n if cpu_reduce else n // 4


def schedule(kind, kw, n, t_lock):
    """The event list for a stream of n samples whose carrier (at freq_center) is locked after t_lock seconds.

    Positions are epoch-relative: 'bef' is one sample before a trigger sample, 'aft' the sample right after one, 'mid'
    halfway between two. Every centre change empties the estimator ring in the middle of an epoch or at its edge."""
    T = trigger_every(kw)
    fc0, lbw, fb = float(kw["freq_center"]), float(kw["lockingbw"]), float(kw["fb"])
    span = n - int(t_lock * FS)

    def at(frac, where):
        k = max(1, int(round((t_lock * FS + frac * span) / T)))
        return {"bef": k * T - 2, "aft": k * T, "mid": k * T + T // 2}[where]

    def after(pos, sec, where):                 # the first such position at least `sec` seconds after pos
        k = -(-(pos + int(sec * FS) + 2) // T)
        return {"bef": k * T - 2, "aft": k * T, "mid": k * T + T // 2}[where]

    ev = []
    if kind == "msk":                        # the MSK AFC acts only with DCD up (mskdemodulator.cpp:498)
        ev.append((at(0.0, "aft"), [("set_dcd", 1)], ""))
    ev += [
        (at(0.01, "bef"), [("set_afc", 0)], "afc_off_locked"),
        (at(0.03, "mid"), [("set_center_freq", fc0 + min(37.0, lbw / 20)), ("set_sql", 1)], "inside,sql_locked"),
        (at(0.05, "aft"), [("set_center_freq", fc0 + 1.25 * lbw)], "below"),
        (at(0.07, "mid"), [("set_center_freq", fc0)], "above"),
        (at(0.09, "bef"), [("set_afc", 1), ("set_center_freq", fc0)], "follow"),
        (at(0.11, "aft"), [("set_center_freq", 1.0)], "clamp_low"),
        (at(0.12, "mid"), [("set_center_freq", 30000.0)], "clamp_high"),
    ]
    # the MSE (a 400 / 600-symbol mean) takes a while to rise above the threshold once the carrier is lost
    u = after(ev[-1][0], 0.35, "aft")
    ev += [
        (u, [("set_sql", 1)], "sql_unlocked"),
        (after(u, 0.1, "bef"), [("set_center_freq", -250.0)], "negative"),
        (after(u, 0.3, "aft"), [("set_center_freq", fc0)], "follow"),
        (after(u, 0.6, "mid"), [("set_sql", 0)], ""),
    ]
    # AFC toggled while it pulls: DCD up (so that the OQPSK estimator no longer steers mixer2, oqpskdemodulator.cpp:642),
    # mixer_center moved 40 Hz below the locked mixer2 with the AFC off, then the AFC on, off inside its countdown, and on
    k1 = at(0.40, "bef")
    ev += [
        (k1, [("set_dcd", 1), ("set_afc", 0), ("set_center_freq", fc0 - min(40.0, lbw / 20))], "offset_locked"),
        (k1 + 2 * T + 2, [("set_afc", 1)], "afc_on_pulling"),
        (k1 + 4 * T + 2, [("set_afc", 0)], "afc_off_pulling"),
        (k1 + 6 * T + 1, [("set_afc", 1)], "afc_on_pulling"),
    ]
    # CPU-reduce: on right after a trigger, off again inside the ring run that starts once coarseCounter reaches Fs (the
    # run is trigger_every(cpu_reduce=True) samples long), then on for the rest of the stream
    k0 = at(0.62, "aft")
    off = k0 + FS + trigger_every(kw, True) // 2
    ev += [(k0, [("set_cpu_reduce", 1)], "cpu_reduce_on"),
           (off, [("set_cpu_reduce", 0)], "cpu_reduce_off_in_run"),
           (off - off % T + 6 * T + T // 2, [("set_cpu_reduce", 1)], "cpu_reduce_on")]
    assert all(a < b for (a, _, _), (b, _, _) in zip(ev, ev[1:])) and ev[-1][0] < n, [e[0] for e in ev]
    return ev


def events(ev):
    """the (sample_index, calls) pairs write_plan takes"""
    return [(a, calls) for a, calls, _ in ev]


def recording_schedule(name, n):
    kind, kw, t_lock = RECORDINGS[name] if name in RECORDINGS else SYNTHETIC[name]
    return schedule(kind, kw, n, t_lock)
