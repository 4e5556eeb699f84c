"""Decode audio recordings of JAERO carriers into ACARS messages as parallel time segments.

JAERO's own input is audio: one carrier per recording, SSB-demodulated by the radio software, at 48 kHz or 44.1 kHz.
AudioDecoder joins the library's stages for such recordings: the rate converter (Resampler) brings them to the demodulators'
48 kHz, the mode identifier (Identifier, identify) finds each one's bit rate and carrier centre where they are not given, and
RecordingDecoder's segment engine demodulates each recording as parallel time segments, one DemodBatch per mode, and stitches
them into one message stream per recording. Every per-sample step runs in the library's kernels; the host copies each second
of input once and reads back the decoded bytes.
"""
import math

import numpy as np

from . import CHANNEL_SETTINGS, Identifier, JaeroError, Reassembler, Resampler, identify, lib, resample_plan
from .receiver import P_MODES, _Raw
from .recording import MODES, _ordered, _SegmentEngine, _Segments, layout

OUT_RATE = 48000


class AudioDecoder(_SegmentEngine):
    """Decodes audio recordings of continuous JAERO carriers (one carrier per recording, int16 PCM at sample_rate) on one GPU.

      sample_rate: the recordings' rate, any whole-hertz rate Resampler accepts; other rates than 48 kHz are converted on the
                   device by one Resampler whose rows are the recordings, fed in lockstep, a whole second per write, with
                   zeros past each recording's end;
      modes, centers_hz: per recording its mode ("msk600", "msk1200", "oqpsk10500", "oqpsk8400") and the audio frequency of its
                   carrier in Hz; one value for every recording or a list with one entry per recording; None identifies it;
      identify_seconds: the recordings whose mode or centre is not given are identified from their first identify_seconds of
                   48 kHz PCM (all of it if shorter) by one Identifier; a given value always wins over the identified one;
      block_seconds, segment_seconds, lead_seconds, max_channels: RecordingDecoder's (layout() lists the checks);
      emit_sus: also return every CRC-valid P-channel signal unit;
      device, stream: the CUDA device, and a cudaStream_t as an int (None: a new torch CUDA stream).
    Every setting is checked before the device is used; a bad one raises ValueError naming it.

    decode(recordings) takes a list of 1-D int16 host arrays (np.memmap is fine), any lengths, and may be called once. Each
    recording is zero-padded to a whole block. A recording whose mode is identified as "unknown" is not decoded; the others
    are grouped by mode into DemodBatch channels (CHANNEL_SETTINGS' kind, fb and lockingbw, the default thresholds, the
    recording's centre as freq_center, AFC on), each cut into segments as RecordingDecoder cuts a carrier, with the P-channel
    frame layer and one Reassembler per recording at 600, 1200 and 10 500 bps and the C-channel layer at 8400 bps. A segment
    whose owned stretch starts at or after its recording's end is dead: its records are dropped and it counts as neither late
    nor unlocked; a live segment's records are dropped from its recording's end on.

    Events are Receiver's dicts (acars, su with emit_sus, cframe) with carrier the recording's index in the list given to
    decode(), center_hz its audio centre and input_seconds the end of the emitting block in seconds of that recording, ordered
    by input_seconds, then carrier. carriers(), unplanned() and stats() report the plan and the counts.

    Burst (R/T) recordings are not decoded: modes refuses burst modes, and a burst recording may be identified as a continuous
    mode. Use as a context manager, or call close()."""

    def __init__(self, sample_rate, modes=None, centers_hz=None, identify_seconds=4.0, block_seconds=0.1, segment_seconds=10,
                 lead_seconds=None, max_channels=4096, emit_sus=False, device=0, stream=None):
        try:
            ok = not isinstance(sample_rate, bool) and float(sample_rate) > 0 and float(sample_rate) == int(float(sample_rate))
        except (TypeError, ValueError, OverflowError):
            ok = False
        if not ok:
            raise ValueError("AudioDecoder: sample_rate must be a positive whole number of hertz, got %r" % (sample_rate,))
        rate = int(float(sample_rate))
        ratio = (1, 1)
        if rate != OUT_RATE:
            lib()                                                 # a library that is not built is not a bad rate
            try:
                plan = resample_plan(rate, OUT_RATE, 0.45 * min(rate, OUT_RATE))
            except JaeroError as e:
                raise ValueError("AudioDecoder: sample_rate %d Hz cannot be converted to 48 kHz: %s" % (rate, e)) from None
            ratio = (plan["L"], plan["M"])
        try:
            self.geometry = layout(rate, block_seconds, segment_seconds, lead_seconds, max_channels, owner="AudioDecoder",
                                   ratio=ratio)
        except ValueError as e:
            msg = str(e)
            if not any(k in msg for k in ("segment_seconds", "lead_seconds", "max_channels", "block_seconds")):
                msg = msg.replace("AudioDecoder: ", "AudioDecoder: block_seconds: ", 1)     # the block grid's rules
            raise ValueError(msg) from None
        try:
            ok = float(identify_seconds) > 0 and math.isfinite(float(identify_seconds))
        except (TypeError, ValueError):
            ok = False
        if not ok:
            raise ValueError("AudioDecoder: identify_seconds must be a positive number of seconds, got %r" % (identify_seconds,))
        for m in _values(modes):
            _check_mode(m)
        for c in _values(centers_hz):
            _check_center(c)
        self.sample_rate, self.segment_seconds, self.identify_seconds = rate, int(segment_seconds), float(identify_seconds)
        self.block_n = int(round(float(block_seconds) * rate))
        self.modes, self.centers_hz = modes, centers_hz
        self.emit_sus, self.device, self._stream_arg = bool(emit_sus), int(device), stream
        self._groups, self._carriers, self._reasm, self._unplanned = [], [], [], []
        self._n_in = np.zeros(0, dtype=np.int64)
        self._clipped = np.zeros(0, dtype=np.int64)
        self._read = 0
        self._used = False

    # ---------------------------------------------------------------------------------------------------------- decode
    def decode(self, recordings):
        """recordings: a list of 1-D int16 host arrays, one carrier each -> every event of every recording"""
        if self._used:
            raise ValueError("AudioDecoder: decode() was already called; new recordings need a new AudioDecoder")
        if isinstance(recordings, np.ndarray) or not isinstance(recordings, (list, tuple)):
            raise ValueError("AudioDecoder: recordings must be a list of 1-D int16 arrays, got %s" % type(recordings).__name__)
        recs = []
        for i, r in enumerate(recordings):
            a = r if isinstance(r, np.ndarray) else np.asarray(r)
            if a.ndim != 1 or a.dtype != np.int16:
                raise ValueError("AudioDecoder: recording %d must be 1-D int16 PCM, got %s of shape %s" % (i, a.dtype, a.shape))
            if a.size == 0:
                raise ValueError("AudioDecoder: recording %d is empty" % i)
            recs.append(a)
        if not recs:
            raise ValueError("AudioDecoder: recordings is empty")
        modes = _per_recording("modes", self.modes, len(recs))
        centers = _per_recording("centers_hz", self.centers_hz, len(recs))
        self._used = True
        import torch
        self._torch = torch
        self._dev = torch.device("cuda", self.device)
        if self._stream_arg is None:
            self._ts = torch.cuda.Stream(device=self._dev)
        else:
            self._ts = torch.cuda.ExternalStream(int(self._stream_arg), device=self._dev)
        self.stream = self._ts.cuda_stream
        with torch.cuda.stream(self._ts):
            return _ordered(self._run(recs, modes, centers))

    def _run(self, recs, modes, centers):
        torch, rate, R = self._torch, self.sample_rate, len(recs)
        per_s = OUT_RATE                                          # 48 kHz samples per second of input
        self._n_in = np.array([len(r) for r in recs], dtype=np.int64)
        geo = next(iter(self.geometry.values()))
        ends = -(-self._n_in // self.block_n)                     # per recording: its blocks, the last one zero-padded
        who = [c for c in range(R) if modes[c] is None or centers[c] is None]
        ident_n = min(int(round(self.identify_seconds * per_s)), int(ends[who].max()) * geo.m) if who else 0
        kept = -(-ident_n // per_s)                               # seconds kept on the device while identifying
        rs = ident = None
        try:
            if rate != OUT_RATE:
                rs = Resampler(rate, R, device=self.device)
                rs.set_stream(self.stream)
            head = None
            if who:
                head = torch.empty((R, kept * per_s), dtype=torch.int16, device=self._dev)
                for s in range(kept):
                    head[:, s * per_s:(s + 1) * per_s].copy_(self._second(recs, s, rs))
                rows = head[who]
                ident = Identifier(float(OUT_RATE), len(who), device=self.device)
                ident.set_stream(self.stream)
                step = geo.m
                for a in range(0, ident_n, step):
                    k = min(step, ident_n - a)
                    ident.write_device(rows.data_ptr() + 2 * a, k, rows.stride(0))
                sq, frames = ident.read()
                found = {c: identify(sq[k], float(OUT_RATE), frames) for k, c in enumerate(who)}
            else:
                found = {}
            self._plan(R, modes, centers, found, ends)
            # whole-second writes up to the end of the longest decoded recording; the undecoded ones are not read further
            last = max((int(g.ends.max()) for g in self._groups), default=0)
            ev = []
            self._read = max(kept, -(-last // geo.per))
            for s in range(-(-last // geo.per)):
                pcm = head[:, s * per_s:(s + 1) * per_s] if s < kept else self._second(recs, s, rs)
                for g in self._groups:
                    ev += self._feed(g, pcm)
            head = None
            if rs is not None:
                _, self._clipped = rs.stats()
            else:
                self._clipped = np.zeros(R, dtype=np.int64)
            for g in self._groups:
                if g.fill:
                    ev += self._chunk(g, final=True)
            return ev
        finally:
            for o in (ident, rs):
                if o is not None:
                    o.close()

    def _second(self, recs, s, rs):
        """second s of every recording, zero-filled past its end, as 48 kHz device PCM [recordings, 48000]"""
        torch, n = self._torch, self.sample_rate
        buf = np.zeros((len(recs), n), dtype=np.int16)
        for c, r in enumerate(recs):
            piece = r[s * n:(s + 1) * n]
            buf[c, :len(piece)] = piece
        x = torch.from_numpy(buf).to(self._dev)
        if rs is None:
            return x
        rs.write_device(x.data_ptr(), n, n)
        p, m, stride = rs.output()
        if m != OUT_RATE:
            raise RuntimeError("AudioDecoder: a second of input gave %d samples at 48 kHz, not %d" % (m, OUT_RATE))
        return torch.as_tensor(_Raw(p, len(recs) * stride, "<i2"), device=self._dev).view(len(recs), stride)[:, :m]

    def _feed(self, g, pcm):
        """appends one second of the group's rows, up to the end of its longest recording; decodes every chunk that fills"""
        left = int(g.ends.max()) * g.geo.m - (g.g0 * g.geo.seg * g.geo.m + g.fill)
        k = min(pcm.shape[1], left)
        if k <= 0:
            return []
        rows = pcm[g.rows_t, :k]
        ev, a = [], 0
        while a < k:
            a += self._take(g, rows[:, a:])
            if self._due(g):
                ev += self._chunk(g, final=False)
        return ev

    def _plan(self, R, modes, centers, found, ends):
        self._carriers, self._reasm, self._unplanned = [None] * R, [None] * R, []
        rows = {}
        for c in range(R):
            r = found.get(c)
            mode = modes[c] if modes[c] is not None else r["mode"]
            center = centers[c] if centers[c] is not None else r["carrier_hz"]
            d = dict(mode=mode, center_hz=float(center), mode_given=modes[c] is not None,
                     center_given=centers[c] is not None, ident_score_db=None if r is None else max(r["score_db"].values()),
                     ident_margin_db=None if r is None else r["margin_db"])
            if mode == "unknown":
                self._unplanned.append(dict(d, index=c, reason="unknown mode"))
                continue
            self._carriers[c] = d
            rows.setdefault(mode, []).append(c)
        for mode in MODES:
            if mode not in rows:
                continue
            idx = rows[mode]
            s = CHANNEL_SETTINGS[mode]
            kw = dict(kind=s["kind"], fb=s["fb"], lockingbw=s["lockingbw"], afc=True,
                      freq_center=[self._carriers[c]["center_hz"] for c in idx])
            g = _Segments(mode, idx, kw, self.geometry[mode], ends=ends[idx])
            g.rows_t = self._torch.as_tensor(idx, dtype=self._torch.int64, device=self._dev)
            self._groups.append(g)
            for c in idx:
                self._reasm[c] = Reassembler() if mode in P_MODES else None
        z = lambda: np.zeros(R, dtype=np.int64)
        self._su_total, self._su_bad, self._messages, self._frames = z(), z(), z(), z()

    def _event_seconds(self, c, t):
        return min((t + 1) * self.block_n, int(self._n_in[c])) / self.sample_rate

    # ---------------------------------------------------------------------------------------------------------- state
    def carriers(self):
        """the decoded recordings, by index: mode, center_hz, mode_given and center_given (False: identified), the identifier's
        best score and margin (None when nothing was identified), and dcd and ebno at the end of the recording's last segment"""
        return sorted(super().carriers(), key=lambda c: c["index"])

    def unplanned(self):
        """the recordings not decoded, with index and reason ("unknown mode") and what the identifier found"""
        return list(self._unplanned)

    def stats(self):
        """read_seconds: the whole seconds of input read (uploaded, and converted at other rates than 48 kHz); per recording
        its length in seconds and the rate converter's clipped samples (over the seconds converted: the
        first identify_seconds, and up to the end of the longest decoded recording); per decoded recording the signal
        units, CRC failures, ACARS records and C-channel frames, and RecordingDecoder's boundary and lock counts; per mode
        group RecordingDecoder's segment, chunk, width and PCM buffer figures"""
        per = {}
        for c, d in enumerate(self._carriers):
            if d is not None:
                per[c] = dict(carrier=c, mode=d["mode"], center_hz=d["center_hz"], sus=int(self._su_total[c]),
                              crc_failures=int(self._su_bad[c]), messages=int(self._messages[c]), cframes=int(self._frames[c]))
        groups = self._segment_stats(per, self.segment_seconds)
        recordings = [dict(index=c, seconds=int(n) / self.sample_rate,
                           resample_clipped=int(self._clipped[c]) if c < len(self._clipped) else 0)
                      for c, n in enumerate(self._n_in)]
        return dict(sample_rate=self.sample_rate, read_seconds=self._read, recordings=recordings,
                    carriers=[per[c] for c in sorted(per)], groups=groups)

    def close(self):
        for g in self._groups:
            g.close()
        self._groups = []
        for r in self._reasm:
            if r is not None:
                r.close()
        self._reasm = []

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _values(v):
    """the entries of a per-recording setting: one value, or a list"""
    return list(v) if isinstance(v, (list, tuple)) else [v]


def _check_mode(m):
    if m is None or m in MODES:
        return
    if isinstance(m, str) and "burst" in m.lower():
        raise ValueError("AudioDecoder: modes: %r is a burst (R/T) mode; burst recordings are not supported, only the continuous "
                         "modes %s" % (m, ", ".join(MODES)))
    raise ValueError("AudioDecoder: modes: %r is not one of the continuous modes %s (burst modes are not supported)"
                     % (m, ", ".join(MODES)))


def _check_center(c):
    if c is None:
        return
    try:
        ok = not isinstance(c, bool) and 0 < float(c) < OUT_RATE / 2
    except (TypeError, ValueError):
        ok = False
    if not ok:
        raise ValueError("AudioDecoder: centers_hz must be audio frequencies in (0, 24000) Hz or None, got %r" % (c,))


def _per_recording(name, v, n):
    if isinstance(v, (list, tuple)):
        if len(v) != n:
            raise ValueError("AudioDecoder: %s has %d entries for %d recordings" % (name, len(v), n))
        return list(v)
    return [v] * n
