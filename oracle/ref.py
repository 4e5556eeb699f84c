"""TEST INFRASTRUCTURE ONLY. ctypes bindings for oracle/_ref/libjaero_ref.so — the reference's
own hot-path sources compiled verbatim (oracle/Makefile). Only tests/, bench.py's cpu_baseline /
--impl reference legs and __graft_entry__.smoke() may import this."""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_ref", "libjaero_ref.so")
_lib = None
c_dp = ctypes.POINTER(ctypes.c_double)
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
        for name in ("jref_oqpsk_new", "jref_msk_new"):
            f = getattr(L, name); f.restype = vp; f.argtypes = [d, d, d, d, i, d, i, i, i]
        for name in ("jref_burst_msk_new", "jref_burst_oqpsk_new"):
            f = getattr(L, name); f.restype = vp; f.argtypes = [d, d, d, d, d]
        L.jref_ebno_log_take.restype = l; L.jref_ebno_log_take.argtypes = [vp, vp, l]
        L.jref_write.argtypes = [vp, vp, l]
        L.jref_set_dcd.argtypes = [vp, i]
        if hasattr(L, "jref_set_center_freq"):          # absent from a reference build made before it existed
            L.jref_set_center_freq.argtypes = [vp, d]
            L.jref_set_afc.argtypes = [vp, i]; L.jref_set_sql.argtypes = [vp, i]; L.jref_set_cpu_reduce.argtypes = [vp, i]
        L.jref_soft_count.restype = l; L.jref_soft_count.argtypes = [vp]
        L.jref_soft_take.restype = l; L.jref_soft_take.argtypes = [vp, vp, l]
        L.jref_emit_count.restype = l; L.jref_emit_count.argtypes = [vp]
        L.jref_cfe_log_take.restype = l; L.jref_cfe_log_take.argtypes = [vp, vp, l]
        L.jref_state.argtypes = [vp, vp]
        L.jref_free.argtypes = [vp]
        L.jref_rrc_design.argtypes = [d, i, d, d, vp, i]
        L.jref_trig_tables.argtypes = [vp, vp]
        L.jref_fir.argtypes = [vp, i, vp, vp, l]
        L.jref_qround.argtypes = [d]
        if hasattr(L, "jref_wavetable_script"):         # absent from a reference build made before it existed
            L.jref_wavetable_script.argtypes = [i, i, vp, vp, d, vp]
        L.jref_fft.argtypes = [i, i, vp, vp]
        L.jref_fftr_forward.argtypes = [i, vp, vp]
        L.jref_fftr_inverse.argtypes = [i, vp, vp]
        L.jref_jfastfir_rrc.argtypes = [d, i, d, d, i, vp, l]
        L.jref_cfe_new.restype = vp; L.jref_cfe_new.argtypes = [i, d, d, d]
        L.jref_cfe_process.restype = d; L.jref_cfe_process.argtypes = [vp, vp, vp]
        L.jref_cfe_bigchange.argtypes = [vp]; L.jref_cfe_free.argtypes = [vp]
        L.jref_codec_new.restype = vp; L.jref_codec_new.argtypes = [i]
        L.jref_codec_decode_continuous.argtypes = [vp, vp, i, vp]
        L.jref_codec_decode_soft.argtypes = [vp, vp, i, vp]
        L.jref_codec_free.argtypes = [vp]
        L.jref_golden_jfastfir_len.restype = l
        L.jref_golden_jfastfir_Fs.restype = d; L.jref_golden_jfastfir_fb.restype = d
        L.jref_golden_jfastfir.argtypes = [vp, vp]
        _lib = L
    return _lib


_FASTFIR_SO = os.path.join(_HERE, "_ref", "libjaero_ref_fastfir.so")
_fastfir_lib = None


def fastfir_available():
    return os.path.exists(_FASTFIR_SO)


def fastfir_lib():
    """oracle/_ref/libjaero_ref_fastfir.so (ref_fastfir_driver.cpp): jref_jfastfir(taps_ri, K, nfft, inout_ri, n, writes,
    n_writes) drives the reference's JFastFir piecewise; jref_hilbert_kernel(out_ri) returns QJHilbertFilter's kernel"""
    global _fastfir_lib
    if _fastfir_lib is None:
        L = ctypes.CDLL(_FASTFIR_SO)
        vp, i, l = ctypes.c_void_p, ctypes.c_int, ctypes.c_long
        L.jref_jfastfir.argtypes = [vp, i, i, vp, l, vp, i]
        L.jref_hilbert_kernel.argtypes = [vp]
        _fastfir_lib = L
    return _fastfir_lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def wavetable_script_available():
    return available() and hasattr(lib(), "jref_wavetable_script")


def wavetable_script(op, arg, samplerate):
    """The reference's own WaveTable (DSP.cpp) running one script per row of op / arg [n_lanes, n_ops] (JAERO_OSC_* codes) ->
    log [n_lanes, n_ops, 9]: WTptr, last_WTptr, WTstep, freq, table index, IfHavePassedPoint, FractionOfSampleItPassesBy,
    WTCISValue() re, im (ref_driver.cpp jref_wavetable_script)"""
    op = np.ascontiguousarray(op, dtype=np.int32)
    arg = np.ascontiguousarray(arg, dtype=np.float64)
    assert op.ndim == 2 and op.shape == arg.shape
    log = np.zeros(op.shape + (9,), dtype=np.float64)
    lib().jref_wavetable_script(op.shape[0], op.shape[1], _p(op), _p(arg), float(samplerate), _p(log))
    return log


class RefDemod:
    """One verbatim reference demodulator. kind: 'oqpsk' | 'msk'.
    NB OQPSK keeps function-local statics: ONE instance per process."""

    def __init__(self, kind, fb, Fs=48000.0, freq_center=8000.0, lockingbw=10500.0, fft_power=14,
                 signalthreshold=0.65, afc=False, sql=False, cpureduce=False):
        L = lib()
        if kind in ("burst_msk", "burst_oqpsk"):
            new = L.jref_burst_msk_new if kind == "burst_msk" else L.jref_burst_oqpsk_new
            self.h = new(fb, Fs, freq_center, lockingbw, signalthreshold)
        else:
            new = L.jref_oqpsk_new if kind == "oqpsk" else L.jref_msk_new
            self.h = new(fb, Fs, freq_center, lockingbw, fft_power, signalthreshold, int(afc), int(sql), int(cpureduce))
        self.kind = kind

    def write(self, pcm):
        pcm = np.ascontiguousarray(pcm, dtype=np.int16)
        lib().jref_write(self.h, _p(pcm), len(pcm))

    def set_dcd(self, dcd):
        lib().jref_set_dcd(self.h, int(dcd))

    def set_center_freq(self, hz):
        """the reference's own CenterFreqChangedSlot / setAFC / setSQL / setCPUReduce (continuous kinds)"""
        lib().jref_set_center_freq(self.h, float(hz))

    def set_afc(self, state):
        lib().jref_set_afc(self.h, int(bool(state)))

    def set_sql(self, state):
        lib().jref_set_sql(self.h, int(bool(state)))

    def set_cpu_reduce(self, state):
        lib().jref_set_cpu_reduce(self.h, int(bool(state)))

    def take_soft(self):
        n = lib().jref_soft_count(self.h)
        out = np.zeros(n, dtype=np.int16)
        if n:
            lib().jref_soft_take(self.h, _p(out), n)
        return out

    def take_cfe_log(self):
        out = np.zeros(1 << 16, dtype=np.float64)
        n = lib().jref_cfe_log_take(self.h, _p(out), len(out))
        return out[:n].copy()

    def take_ebno_log(self):
        out = np.zeros(4096, dtype=np.float64)
        n = lib().jref_ebno_log_take(self.h, _p(out), len(out))
        return out[:n].copy()

    def state(self):
        o = np.zeros(16, dtype=np.float64)
        n = lib().jref_state(self.h, _p(o))
        fields = STATE_FIELDS if not self.kind.startswith("burst") else BURST_STATE_FIELDS
        return dict(zip(fields, o[:n]))

    def close(self):
        if self.h:
            lib().jref_free(self.h); self.h = None


class RefCodec:
    """JConvolutionalCodec (jconvolutionalcodec.cpp) over the restated libcorrect."""

    def __init__(self, paddinglength=24):
        self.h = lib().jref_codec_new(paddinglength)

    def decode_continuous(self, soft):
        soft = np.ascontiguousarray(soft, dtype=np.uint8)
        out = np.zeros(len(soft), dtype=np.int32)
        n = lib().jref_codec_decode_continuous(self.h, _p(soft), len(soft), _p(out))
        return out[:n].copy()

    def decode_soft(self, soft):
        soft = np.ascontiguousarray(soft, dtype=np.uint8)
        out = np.zeros(len(soft), dtype=np.int32)
        n = lib().jref_codec_decode_soft(self.h, _p(soft), len(soft), _p(out))
        return out[:n].copy()

    def close(self):
        if self.h:
            lib().jref_codec_free(self.h); self.h = None


def run_demod_job(args):
    """Process-pool worker: (kind, kwargs, pcm, chunk, dcd_schedule[, events]) -> (soft, state, cfe_log).
    dcd_schedule: list of (sample_index, dcd) applied at chunk boundaries (index must be a multiple of chunk).
    events: control calls at sample indices, as restated.write_plan takes them; the writes are cut at each of them."""
    from oracle.restated import apply_calls, write_plan
    kind, kw, pcm, chunk, dcd_schedule = args[:5]
    events = list(args[5]) if len(args) > 5 and args[5] else []
    events += [(int(a), [("set_dcd", int(v))]) for a, v in (dcd_schedule or [])]
    d = RefDemod(kind, **kw)
    for a, n, calls in write_plan(len(pcm), chunk, events):
        apply_calls(d, calls)
        d.write(pcm[a:a + n])
    out = (d.take_soft(), d.state(), d.take_cfe_log())
    d.close()
    return out


class RefReasm:
    """The reference's own RISUData / ISUData / ParserISU / ACARSDefragmenter (JAERO/aerol.cpp:4-487), compiled
    verbatim into oracle/_ref/libjaero_ref_reasm.so by oracle/Makefile (ref_reasm_driver.cpp)."""

    _lib = None

    @classmethod
    def lib(cls):
        if cls._lib is None:
            L = ctypes.CDLL(os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libjaero_ref_reasm.so"))
            L.jref_reasm_new.restype = ctypes.c_void_p
            for f in ("jref_reasm_free", "jref_reasm_reset", "jref_reasm_short_frame"):
                getattr(L, f).argtypes = [ctypes.c_void_p]
            L.jref_reasm_su.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int]
            L.jref_reasm_r.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int]
            L.jref_reasm_pending.argtypes = [ctypes.c_void_p]
            L.jref_reasm_pop.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
            cls._lib = L
        return cls._lib

    @staticmethod
    def available():
        return os.path.exists(os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libjaero_ref_reasm.so"))

    def __init__(self):
        self.h = self.lib().jref_reasm_new()

    def reset(self):
        self.lib().jref_reasm_reset(self.h)

    def short_frame(self):
        self.lib().jref_reasm_short_frame(self.h)

    def push_su(self, su, burstmode=False):
        return self.lib().jref_reasm_su(self.h, bytes(bytearray(su[:10])), int(burstmode))

    def push_r(self, info, burstmode=True):
        return self.lib().jref_reasm_r(self.h, bytes(bytearray(info[:17])), int(burstmode))

    def pop_all(self):
        out = []
        meta = (ctypes.c_uint * 16)(); cap = 1 << 16; text = (ctypes.c_ubyte * cap)()
        while True:
            n = self.lib().jref_reasm_pop(self.h, meta, text, cap)
            if n < 0:
                break
            out.append(reasm_record(list(meta), bytes(text[:n])))
        return out

    def close(self):
        if self.h:
            self.lib().jref_reasm_free(self.h); self.h = None


def reasm_record(m, t):
    """meta/text layout shared by the reference driver and the oracle: see ref_reasm_driver.cpp jref_reasm_pop."""
    o = 0
    label = t[o:o + m[11]]; o += m[11]
    reg = t[o:o + m[12]]; o += m[12]
    msg = t[o:o + m[13]]; o += m[13]
    ud = t[o:o + m[14]]
    return dict(kind=m[0], aesid=m[1], gesid=m[2], qno=m[3], refno=m[4], seqno=m[5], nooct=m[6], mode=m[7], tak=m[8], bi=m[9],
                nonacars=bool(m[10] & 1), downlink=bool(m[10] & 2), valid=bool(m[10] & 4), hastext=bool(m[10] & 8),
                moretocome=bool(m[10] & 16), label=label.hex(), reg=reg.hex(), message=msg.hex(), userdata=ud.hex())
