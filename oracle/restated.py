"""TEST INFRASTRUCTURE ONLY. ctypes bindings for oracle/_build/libjaero_oracle.so — this repo's CPU
restatement of the reference's hot path (oracle/restated/*.cpp, oracle/correct_restated.c).
Only tests/, bench.py's cpu_baseline / --impl reference legs and __graft_entry__.smoke() may import this."""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libjaero_oracle.so")
_lib = None
STATE_FIELDS = ["mixer2_freq", "mixer2_wtptr", "center_freq", "st_freq", "st_wtptr", "agc", "mse",
                "ebno", "marg", "cfe_est", "n_sig_true", "n_sig_false", "center_wtptr", "st_ref_wtptr"]


BURST_STATE_FIELDS = ["mixer2_freq", "mixer2_wtptr", "center_freq", "st_freq", "st_wtptr", "agc", "mse",
                      "ebno", "vol_gain", "rotator_freq", "n_sig_true", "n_sig_false", "cntr", "startstop"]


def available():
    return os.path.exists(_SO)


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(_SO)
        vp, d, i, l = ctypes.c_void_p, ctypes.c_double, ctypes.c_int, ctypes.c_long
        L.jor_demod_new.restype = vp; L.jor_demod_new.argtypes = [i, d, d, d, d, i, d, i, i, i]
        L.jor_burst_msk_new.restype = vp; L.jor_burst_msk_new.argtypes = [d, d, d, d, d]
        L.jor_burst_oqpsk_new.restype = vp; L.jor_burst_oqpsk_new.argtypes = [d, d, d, d, d]
        L.jor_aux_take.restype = l; L.jor_aux_take.argtypes = [vp, i, vp, l]
        L.jor_write.argtypes = [vp, vp, l]; L.jor_set_dcd.argtypes = [vp, i]
        L.jor_set_center_freq.argtypes = [vp, d]
        L.jor_set_afc.argtypes = [vp, i]; L.jor_set_sql.argtypes = [vp, i]; L.jor_set_cpu_reduce.argtypes = [vp, i]
        L.jor_burst_set_sql.argtypes = [vp, i]
        L.jor_soft_count.restype = l; L.jor_soft_count.argtypes = [vp]
        L.jor_soft_take.restype = l; L.jor_soft_take.argtypes = [vp, vp, l]
        L.jor_cfe_log_take.restype = l; L.jor_cfe_log_take.argtypes = [vp, vp, l, i]
        L.jor_state.argtypes = [vp, vp]; L.jor_free.argtypes = [vp]
        L.jor_rrc_design.argtypes = [d, i, d, d, vp, i]
        L.jor_trig_tables.argtypes = [vp, vp]; L.jor_qround.argtypes = [d]
        L.jor_fft.argtypes = [i, i, vp, vp]
        L.jor_cfe_new.restype = vp; L.jor_cfe_new.argtypes = [i, d, d, d]
        L.jor_cfe_process.restype = d; L.jor_cfe_process.argtypes = [vp, vp, vp, vp]
        L.jor_cfe_bigchange.argtypes = [vp]; L.jor_cfe_free.argtypes = [vp]
        L.jor_deinterleave.argtypes = [vp, i, vp]
        L.jor_viterbi_new.restype = vp; L.jor_viterbi_new.argtypes = [i]
        L.jor_viterbi_decode_continuous.argtypes = [vp, vp, i, vp]; L.jor_viterbi_free.argtypes = [vp]
        L.jor_conv_decode_soft.argtypes = [vp, i, vp]; L.jor_conv_encode.argtypes = [vp, i, vp]
        L.jor_pchan_new.restype = vp; L.jor_pchan_new.argtypes = [i]
        L.jor_pchan_process.argtypes = [vp, vp, i]; L.jor_pchan_update_dcd.argtypes = [vp]
        L.jor_pchan_dcd.argtypes = [vp]; L.jor_pchan_syncs.restype = l; L.jor_pchan_syncs.argtypes = [vp]
        L.jor_pchan_lost_signal.argtypes = [vp]; L.jor_wire_pchan.argtypes = [vp, vp]
        L.jor_pchan_su_count.restype = l; L.jor_pchan_su_count.argtypes = [vp]
        L.jor_pchan_su_take.restype = l; L.jor_pchan_su_take.argtypes = [vp, vp, vp, vp, l]
        L.jor_pchan_free.argtypes = [vp]
        L.jor_crc16.restype = ctypes.c_uint16; L.jor_crc16.argtypes = [vp, i]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


class OracleDemod:
    def __init__(self, kind, fb, Fs=48000.0, freq_center=8000.0, lockingbw=10500.0, fft_power=14,
                 signalthreshold=0.65, afc=False, sql=False, cpureduce=False):
        self.kind = kind
        if kind == "burst_msk":
            self.h = lib().jor_burst_msk_new(fb, Fs, freq_center, lockingbw, signalthreshold)
        elif kind == "burst_oqpsk":
            self.h = lib().jor_burst_oqpsk_new(fb, Fs, freq_center, lockingbw, signalthreshold)
            lib().jor_burst_set_sql(self.h, int(sql))
        else:
            self.h = lib().jor_demod_new(0 if kind == "oqpsk" else 1, fb, Fs, freq_center, lockingbw, fft_power,
                                         signalthreshold, int(afc), int(sql), int(cpureduce))

    def write(self, pcm):
        pcm = np.ascontiguousarray(pcm, dtype=np.int16)
        lib().jor_write(self.h, _p(pcm), len(pcm))

    def set_dcd(self, dcd):
        lib().jor_set_dcd(self.h, int(dcd))

    def set_center_freq(self, hz):
        """CenterFreqChangedSlot (continuous kinds)"""
        lib().jor_set_center_freq(self.h, float(hz))

    def set_afc(self, state):
        """setAFC / setSQL / setCPUReduce (continuous kinds): plain flags, read by the following writes"""
        lib().jor_set_afc(self.h, int(bool(state)))

    def set_sql(self, state):
        lib().jor_set_sql(self.h, int(bool(state)))

    def set_cpu_reduce(self, state):
        lib().jor_set_cpu_reduce(self.h, int(bool(state)))

    def take_soft(self):
        n = lib().jor_soft_count(self.h)
        out = np.zeros(n, dtype=np.int16)
        if n:
            lib().jor_soft_take(self.h, _p(out), n)
        return out

    def take_cfe_log(self, raw=False):
        """the estimate of every coarse-estimator epoch so far: as emitted (FreqOffsetEstimate, gated by emptyingcountdown) or,
        raw=True, freq_offset_est itself (what jaero_status.cfe_est reports). The two logs are drained independently."""
        out = np.zeros(1 << 16, dtype=np.float64)
        n = lib().jor_cfe_log_take(self.h, _p(out), len(out), int(bool(raw)))
        return out[:n].copy()

    def take_aux(self, which, cap=1 << 14):
        """burst kinds: 0 = EbNo of each burst, 1 = trident log (5 values per test), 2 = stream index of the input sample at which
        each trident test ran (the sample that completed the fill), 3 = the trident buffer of each test (tri_sz samples per
        test). Each log is drained independently; at most `cap` values per call."""
        out = np.zeros(cap, dtype=np.float64)
        n = lib().jor_aux_take(self.h, which, _p(out), len(out))
        return out[:n].copy()

    def state(self):
        o = np.zeros(16, dtype=np.float64)
        n = lib().jor_state(self.h, _p(o))
        fields = BURST_STATE_FIELDS if self.kind.startswith("burst") else STATE_FIELDS
        return dict(zip(fields, o[:n]))

    def close(self):
        if self.h:
            lib().jor_free(self.h); self.h = None


class OracleCfe:
    """Restated CoarseFreqEstimate on its own (radix-2 FFT arithmetic of the restatement): setSettings, bigchange,
    ProcessBasebandData. process() -> (emitted estimate, freq_offset_est, y)."""

    def __init__(self, fft_power, lockingbw, fb, Fs=48000.0):
        self.nfft = 1 << fft_power
        self.h = lib().jor_cfe_new(fft_power, lockingbw, fb, Fs)

    def process(self, data):
        d = np.ascontiguousarray(data, dtype=np.complex128)
        assert d.shape == (self.nfft,)
        y = np.zeros(self.nfft, dtype=np.float64)
        raw = ctypes.c_double()
        e = lib().jor_cfe_process(self.h, _p(d), _p(y), ctypes.byref(raw))
        return e, raw.value, y

    def bigchange(self):
        lib().jor_cfe_bigchange(self.h)

    def close(self):
        if self.h:
            lib().jor_cfe_free(self.h); self.h = None


class OracleViterbi:
    def __init__(self, paddinglength=24):
        self.h = lib().jor_viterbi_new(paddinglength)

    def decode_continuous(self, soft):
        soft = np.ascontiguousarray(soft, dtype=np.uint8)
        out = np.zeros(len(soft), dtype=np.int32)
        n = lib().jor_viterbi_decode_continuous(self.h, _p(soft), len(soft), _p(out))
        return out[:n].copy()

    def close(self):
        if self.h:
            lib().jor_viterbi_free(self.h); self.h = None


def conv_encode(msg_bytes):
    msg = np.ascontiguousarray(msg_bytes, dtype=np.uint8)
    enc = np.zeros(2 * (len(msg) + 2) + 8, dtype=np.uint8)
    nbits = lib().jor_conv_encode(_p(msg), len(msg), _p(enc))
    return np.unpackbits(enc)[:nbits]


def conv_decode_soft(soft):
    soft = np.ascontiguousarray(soft, dtype=np.uint8)
    msg = np.zeros(len(soft) // 16 + 8, dtype=np.uint8)
    nbytes = lib().jor_conv_decode_soft(_p(soft), len(soft), _p(msg))
    return np.unpackbits(msg[:nbytes])


def deinterleave(block, cols):
    block = np.ascontiguousarray(block, dtype=np.int32)
    out = np.zeros(64 * cols, dtype=np.uint8)
    lib().jor_deinterleave(_p(block), cols, _p(out))
    return out


class OraclePChannel:
    """Restated AeroL::Decode (continuous P-channel): soft bits -> signal units + CRC flags + DCD."""

    def __init__(self, fb):
        self.h = lib().jor_pchan_new(int(fb))

    def process(self, soft):
        soft = np.ascontiguousarray(soft, dtype=np.int16)
        lib().jor_pchan_process(self.h, _p(soft), len(soft))

    def update_dcd(self):
        lib().jor_pchan_update_dcd(self.h)

    def lost_signal(self):
        """AeroL::LostSignal (aerol.h:925-931)"""
        lib().jor_pchan_lost_signal(self.h)

    def wire(self, demod):
        """Connect a continuous OracleDemod to this AeroL as JAERO/mainwindow.cpp does (direct connections): soft-bit vectors are
        decoded inside write(), DCD and LostSignal feed back at once. take_soft() on the demodulator still returns what was emitted."""
        lib().jor_wire_pchan(demod.h, self.h)

    @property
    def dcd(self):
        return bool(lib().jor_pchan_dcd(self.h))

    @property
    def syncs(self):
        """unique-word syncs so far"""
        return int(lib().jor_pchan_syncs(self.h))

    def take_sus(self):
        n = lib().jor_pchan_su_count(self.h)
        b = np.zeros((n, 12), dtype=np.uint8); ok = np.zeros(n, dtype=np.int32); fr = np.zeros(n, dtype=np.int64)
        if n:
            lib().jor_pchan_su_take(self.h, _p(b), _p(ok), _p(fr), n)
        return b, ok, fr

    def close(self):
        if self.h:
            lib().jor_pchan_free(self.h); self.h = None


class OracleRTChannel:
    """Restated burst branch of AeroL::Decode + RTChannelDeleaveFECScram: soft bits (with -1 markers) -> R / T packets."""

    def __init__(self, fb):
        L = lib()
        L.jor_rt_new.restype = ctypes.c_void_p; L.jor_rt_new.argtypes = [ctypes.c_int]
        L.jor_rt_process.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        L.jor_rt_update_dcd.argtypes = [ctypes.c_void_p]
        L.jor_rt_packet_count.restype = ctypes.c_long; L.jor_rt_packet_count.argtypes = [ctypes.c_void_p]
        L.jor_rt_trials.restype = ctypes.c_long; L.jor_rt_trials.argtypes = [ctypes.c_void_p]
        L.jor_rt_packet.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        L.jor_rt_free.argtypes = [ctypes.c_void_p]
        self.h = L.jor_rt_new(int(fb))

    def process(self, soft, vector_semantics=False):
        soft = np.ascontiguousarray(soft, dtype=np.int16)
        lib().jor_rt_process(self.h, _p(soft), len(soft), int(vector_semantics))

    def update_dcd(self):
        lib().jor_rt_update_dcd(self.h)

    @property
    def trials(self):
        return lib().jor_rt_trials(self.h)

    def packets(self):
        out = []
        for k in range(lib().jor_rt_packet_count(self.h)):
            t = ctypes.c_int(); ns = ctypes.c_int(); bi = ctypes.c_long(); buf = np.zeros(1024, dtype=np.uint8)
            n = lib().jor_rt_packet(self.h, k, ctypes.byref(t), ctypes.byref(ns), ctypes.byref(bi), _p(buf), 1024)
            out.append(dict(type=t.value, nsus=ns.value, bit_index=bi.value, bytes=buf[:n].copy()))
        return out

    def close(self):
        if self.h:
            lib().jor_rt_free(self.h); self.h = None


class OracleCChannel:
    """Restated AeroL::DecodeC (8400 bps C-channel): soft bits -> per frame 3 sub-band signal units (+CRC) and 25 x 12 voice bytes."""

    def __init__(self):
        L = lib()
        L.jor_cchan_new.restype = ctypes.c_void_p
        L.jor_cchan_process.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        L.jor_cchan_update_dcd.argtypes = [ctypes.c_void_p]; L.jor_cchan_lost_signal.argtypes = [ctypes.c_void_p]
        L.jor_cchan_dcd.argtypes = [ctypes.c_void_p]
        L.jor_cchan_frame_count.restype = ctypes.c_long; L.jor_cchan_frame_count.argtypes = [ctypes.c_void_p]
        L.jor_cchan_take.restype = ctypes.c_long; L.jor_cchan_take.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_long]
        L.jor_cchan_free.argtypes = [ctypes.c_void_p]
        self.h = L.jor_cchan_new()

    def process(self, soft):
        soft = np.ascontiguousarray(soft, dtype=np.int16)
        lib().jor_cchan_process(self.h, _p(soft), len(soft))

    def update_dcd(self):
        lib().jor_cchan_update_dcd(self.h)

    def lost_signal(self):
        """AeroL::LostSignal (aerol.h:925-931)"""
        lib().jor_cchan_lost_signal(self.h)

    @property
    def dcd(self):
        return bool(lib().jor_cchan_dcd(self.h))

    def take_frames(self):
        n = lib().jor_cchan_frame_count(self.h)
        su = np.zeros((n, 3, 12), dtype=np.uint8); ok = np.zeros((n, 3), dtype=np.int32); voice = np.zeros((n, 300), dtype=np.uint8)
        if n:
            lib().jor_cchan_take(self.h, _p(su), _p(ok), _p(voice), n)
        return su, ok, voice

    def close(self):
        if self.h:
            lib().jor_cchan_free(self.h); self.h = None


CONTROLS = ("set_center_freq", "set_afc", "set_sql", "set_cpu_reduce", "set_dcd")


def write_plan(n, chunk, events=()):
    """[(start, length, calls)]: n samples written in pieces of `chunk` samples (or of the successive lengths in `chunk` when
    it is a sequence), each piece cut again at every event position. events: [(sample_index, [(name, *args), ...]), ...] with
    names from CONTROLS; an event's calls are made before the write that starts at its sample index."""
    ev = {}
    for at, calls in events or ():
        at = int(at)
        assert 0 <= at < n, at
        assert all(c[0] in CONTROLS for c in calls), calls
        ev.setdefault(at, []).extend(tuple(c) for c in calls)
    sizes = [chunk] * -(-n // chunk) if np.ndim(chunk) == 0 else list(chunk)
    cuts, a = set(ev), 0
    for m in sizes:
        cuts.add(a); a += int(m)
        if a >= n:
            break
    assert a >= n, "the write sizes cover %d of %d samples" % (a, n)
    cuts = sorted(c for c in cuts if c < n) + [n]
    return [(a, b - a, ev.get(a, [])) for a, b in zip(cuts[:-1], cuts[1:])]


def apply_calls(demod, calls):
    """make each (name, *args) call of an event on a demodulator (OracleDemod, RefDemod or DemodBatch)"""
    for name, *args in calls:
        getattr(demod, name)(*args)


def run_demod_job(args):
    """(kind, kw, pcm, chunk[, events]) -> (soft, state, aux): one restated demodulator over one stream, written in pieces of
    `chunk` samples, or of the successive lengths in `chunk` when it is a sequence, with the control calls of `events` made at
    their sample indices (write_plan). aux: the EbNo of each burst (burst kinds) or the emitted coarse estimates. Module-level so that tests can farm channels out to a multiprocessing pool."""
    kind, kw, pcm, chunk = args[:4]
    events = args[4] if len(args) > 4 else ()
    d = OracleDemod(kind, **kw)
    for a, n, calls in write_plan(len(pcm), chunk, events):
        apply_calls(d, calls)
        d.write(pcm[a:a + n])
    soft, st = d.take_soft(), d.state()
    aux = d.take_aux(0) if kind.startswith("burst") else d.take_cfe_log()
    d.close()
    return soft, st, aux
