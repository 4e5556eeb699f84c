"""Decode audio recordings of R/T burst carriers into R/T packets and ACARS messages as parallel time segments.

Half of JAERO's recordings are of burst carriers: an aircraft's R and T channels, where each packet is one short burst at 600,
1200 or 10 500 bps. BurstAudioDecoder joins the library's stages for such recordings, one carrier per recording: the rate
converter (Resampler) brings them to 48 kHz, the mode identifier (Identifier, identify) finds each one's bit rate where it is
not given, and each recording is cut into time segments that run side by side as channels of one burst demodulator batch
(BurstMskBatch, BurstOqpskBatch) with the R/T packet layer (RTChannelBatch.process_burst) behind it, as RecordingDecoder cuts
a continuous carrier. The segments' packets are stitched into one packet stream per recording, which feeds its Reassembler.
Every per-sample step runs in the library's kernels; the host copies each second of input once and reads back the packets.
"""
import inspect
import math

import numpy as np

from . import (BurstMskBatch, BurstOqpskBatch, Identifier, JaeroError, Reassembler, Resampler, RTChannelBatch, identify, lib,
               resample_plan)
from .receiver import _Events, _Raw
from .recording import MODES as CONTINUOUS_MODES
from .recording import Geometry, _ordered, _whole_seconds, stitch

OUT_RATE = 48000
BURST_MODES = ("burst_msk600", "burst_msk1200", "burst_oqpsk10500")
FB = {"burst_msk600": 600, "burst_msk1200": 1200, "burst_oqpsk10500": 10500}
# the identifier's rates that have a burst mode (8400 bps has none)
FROM_IDENT = {"msk600": "burst_msk600", "msk1200": "burst_msk1200", "oqpsk10500": "burst_oqpsk10500"}
# identify()'s threshold: a recording whose best burst rate scores below it is "unknown"
IDENT_THRESHOLD_DB = inspect.signature(identify).parameters["threshold_db"].default

# What a segment must have seen for a packet it emits to be the straight chain's, from the library's constants:
# - the R/T layer's time-out: a burst is dropped total_number_of_bits after its start, fb x 3 bits at 600 and 1200 bps and
#   fb bits at 10 500 bps (capi.cu, jaero_rt_create), so no packet is emitted later than 3 s and 1 s after its burst began;
# - the trident fill that finds the burst: TRI_SAMPLES 48 kHz samples before the demodulator knows of it (capi.cu,
#   burst_create: 224, 200 and 288 symbols);
# - the emission lag: a packet is read after the write that completes it, at most one internal chunk, BURST_CHUNK samples
#   (burst.cuh), when a block is at most that long;
# - the burst front's AGC, a moving average over agc_len = 1 s of samples (capi.cu, burst_create), which a cold start fills
#   from zeros: the gain that feeds the burst detector is the chain's once the segment has run that long;
# - the R/T layer's carrier-detect hold: a unique word sets datacdcountdown to 12 (rtchannel.cu) and each 1 s tick takes 3
#   off (frame_stages.cuh, dcd_tick), so carrier detect stays up for up to 4 s after a sync. While it is up, and the bit
#   counter is inside a packet, the next burst's unique word is not searched for, so a burst within 4 s of the previous
#   sync is decoded only if the segment saw that sync too.
TIMEOUT_SECONDS = {"burst_msk600": 3, "burst_msk1200": 3, "burst_oqpsk10500": 1}
TRI_SAMPLES = {"burst_msk600": 17920, "burst_msk1200": 8000, "burst_oqpsk10500": 2633}
BURST_CHUNK = 16384
AGC_SECONDS = 1
DCD_HOLD_SECONDS = 4
# Seconds a segment starts before the stretch it owns: the sum above, rounded up to whole seconds. 600 bps: 3 + (17920 +
# 16384) / 48000 + 1 + 4 = 8.71 s -> 9; 1200 bps: 3 + (8000 + 16384) / 48000 + 1 + 4 = 8.51 s -> 9; 10 500 bps: 1 + (2633 +
# 16384) / 48000 + 1 + 4 = 6.40 s -> 7. A run of bursts each within 4 s of the one before links a packet to syncs further
# back than any lead; there a segment, which starts with carrier detect down, can decode a packet the chain's held carrier
# detect skips, or skip one the chain decodes.
DEFAULT_BURST_LEAD_SECONDS = {mode: int(math.ceil(TIMEOUT_SECONDS[mode] + (TRI_SAMPLES[mode] + BURST_CHUNK) / OUT_RATE
                                                  + AGC_SECONDS + DCD_HOLD_SECONDS)) for mode in BURST_MODES}


def burst_layout(input_rate, block_seconds, segment_seconds, lead_seconds=None, max_channels=4096, ratio=(1, 1),
                 owner="BurstAudioDecoder"):
    """Checks the segment settings of burst recordings -> {mode: Geometry}.

    Segment boundaries, starts and leads are whole seconds and a second is a whole number of blocks, each giving the same whole
    number of 48 kHz samples (ratio: the rate converter's (interpolation, decimation)), so every segment runs on the block
    grid and the R/T layer's 1 s tick grid. A block gives at most BURST_CHUNK samples at 48 kHz, so a packet is read at most
    one internal chunk after its burst ends. The guard, how long a segment runs past the stretch it owns, is that emission lag
    plus one block, and a segment is longer than two guards, so the windows around neighbouring boundaries do not meet.
    lead_seconds: None (DEFAULT_BURST_LEAD_SECONDS), seconds for every mode, or a dict of seconds by mode over the defaults.
    ValueError otherwise, its text headed by `owner`."""
    L, D = ratio
    rate = int(float(input_rate))
    try:
        b = float(block_seconds)
    except (TypeError, ValueError):
        b = float("nan")
    if not 0 < b <= 1.0:
        raise ValueError(owner + ": block_seconds must be in (0, 1], got %r" % (block_seconds,))
    if isinstance(max_channels, bool) or not isinstance(max_channels, (int, np.integer)) or max_channels < 1:
        raise ValueError(owner + ": max_channels must be a positive whole number, got %r" % (max_channels,))
    seg_s = _whole_seconds(owner, "segment_seconds", segment_seconds)
    if seg_s < 1:
        raise ValueError(owner + ": segment_seconds must be at least 1, got %r" % (segment_seconds,))
    block_n = int(round(b * rate))
    if block_n < 1 or rate % block_n:
        raise ValueError(owner + ": block_seconds: a second of input (%d samples) is not a whole number of %r s blocks (%d "
                         "samples)" % (rate, block_seconds, block_n))
    if block_n * L % D:
        raise ValueError(owner + ": block_seconds: a %r s block (%d samples) does not give a whole number of 48 kHz samples "
                         "at %d Hz (%d x %d / %d)" % (block_seconds, block_n, rate, block_n, L, D))
    per, m = rate // block_n, block_n * L // D
    if m > BURST_CHUNK:
        raise ValueError(owner + ": block_seconds %r gives %d samples at 48 kHz, more than one burst demodulator chunk (%d)"
                         % (block_seconds, m, BURST_CHUNK))
    if lead_seconds is None:
        leads = dict(DEFAULT_BURST_LEAD_SECONDS)
    elif isinstance(lead_seconds, dict):
        unknown = sorted(set(lead_seconds) - set(BURST_MODES))
        if unknown:
            raise ValueError(owner + ": lead_seconds for unknown mode(s) %s" % ", ".join(map(str, unknown)))
        leads = dict(DEFAULT_BURST_LEAD_SECONDS, **lead_seconds)
    else:
        leads = {mode: lead_seconds for mode in BURST_MODES}
    guard = -(-BURST_CHUNK // m) + 1
    if seg_s * per <= 2 * guard + 2:
        raise ValueError(owner + ": segment_seconds %r is too short: a segment must be longer than two guards of %.2f s (one "
                         "burst demodulator chunk and one block)" % (segment_seconds, guard / per))
    return {mode: Geometry(mode, per, m, seg_s * per, _whole_seconds(owner, "lead_seconds", leads[mode]) * per, guard,
                           int(max_channels)) for mode in BURST_MODES}


def packet_keys(rows, recs):
    """Per packet a key that is equal for two packets only when they are of the same row and have the same type, number of
    signal units and bytes: stitch() takes it as the packet's carrier, so only copies of one packet are matched.
    rows: per packet its row; recs: per packet (type, nsus, bytes)."""
    ids = {}
    return np.array([ids.setdefault((int(r),) + (int(q[0]), int(q[1]), bytes(q[2])), len(ids)) for r, q in zip(rows, recs)],
                    dtype=np.int64)


def stitch_packets(rows, recs, seg, t, starts, guard, ends=None):
    """Which packets of consecutive segments of the same rows make one stream.

    rows, seg, t: per packet its row, its segment (an index into starts) and the block it was emitted in; recs: per packet
    (type, nsus, bytes). Around each boundary b = starts[s + 1], two packets of s and s + 1 are one packet when they have the
    same row, type, nsus and bytes and were emitted at most one block apart, one of them within [b - guard, b + guard]: the
    copy emitted in its own segment's owned stretch is kept, otherwise s's copy. A packet within that window without such a
    partner is kept; every other packet is kept when it was emitted in its segment's owned stretch. This is stitch() with
    packet_keys() as the carrier, so bursts closer together than three blocks are told apart by their content (identical
    packets of one segment must still be three blocks apart). ends: None, or per packet the block its row's signal ends at; a
    boundary at or after it is not one of that row's. -> stitch()'s (keep, matched, unmatched)"""
    return stitch(packet_keys(rows, recs), seg, t, starts, guard, ends)


class _Group:
    """One mode's recordings: their rows (index: their recording indices, in row order), per row the block its signal ends at,
    the 48 kHz PCM not decoded yet, P[row, t] (int16 on the device, from the first block of segment g0's window on), the
    packets held back for the next chunk's stitch and the counts stats() reports"""

    def __init__(self, mode, index, geo, ends):
        self.mode, self.index, self.geo = mode, np.asarray(index, dtype=np.int64), geo
        self.n = len(self.index)
        self.ends = np.asarray(ends, dtype=np.int64)
        self.S = geo.segments_per_chunk(self.n)
        # the most PCM a chunk holds: a whole chunk, or the longest row with the last segment's window past its end
        self.cap = min(geo.chunk_blocks(self.S), int(self.ends.max()) + geo.seg + geo.guard) * geo.m
        self.P, self.fill, self.g0 = None, 0, 0
        self.chunks = self.segments = self.width = self.pcm_peak = 0
        self.held = None
        z = lambda: np.zeros(self.n, dtype=np.int64)
        self.matched, self.unmatched, self.crc_failures = z(), z(), z()

    def close(self):
        self.P = None


class BurstAudioDecoder(_Events):
    """Decodes audio recordings of R/T burst carriers (one carrier per recording, int16 PCM at sample_rate) on one GPU.

      sample_rate: the recordings' rate, any whole-hertz rate Resampler accepts; other rates than 48 kHz are converted on the
                   device by one Resampler whose rows are the recordings, a whole second per write, with zeros past each
                   recording's end;
      modes:       per recording "burst_msk600", "burst_msk1200" or "burst_oqpsk10500"; one value for every recording or a
                   list with one entry per recording; None identifies it;
      identify_seconds: the recordings whose mode is not given are identified from their first identify_seconds of 48 kHz PCM
                   (all of it if shorter) by one Identifier: the burst rate with the best identify() score, or "unknown" when
                   that score is below identify()'s threshold. Bursts are sparse, so the default is a minute;
      block_seconds: the decoding step; a second is a whole number of blocks;
      segment_seconds, lead_seconds: the stretch each demodulator channel owns, and how long before it the channel starts
                   (None: DEFAULT_BURST_LEAD_SECONDS by mode; seconds; or a dict by mode), whole seconds (burst_layout lists
                   the checks);
      max_channels: the widest batch; a mode group of R recordings runs S = max_channels // R segments per chunk;
      emit_packets: also return every R/T packet;
      device, stream: the CUDA device, and a cudaStream_t as an int for the rate converter, identifier and PCM copies (None: a
                   new torch CUDA stream).
    Every setting is checked before the device is used; a bad one raises ValueError naming it.

    decode(recordings) takes a list of 1-D int16 host arrays (np.memmap is fine), any lengths, and may be called once. Each
    recording is zero-padded to a whole block. A recording identified as "unknown" is not decoded; the others are grouped by
    mode. Each group's recordings are cut into segments as RecordingDecoder cuts a carrier, and a chunk of S segments per
    recording runs as one burst demodulator batch of recordings x S channels with the batch classes' default settings (one
    batch serves carriers at any centre: the trident search covers the band and re-centres on every burst) and one
    RTChannelBatch of the same width, block by block, ticked once per second of signal. The packets of neighbouring segments
    are stitched (stitch_packets) into one stream per recording, which feeds the recording's Reassembler: R packets with
    push_r(downlink=True), T packets with push_t_packet. A segment whose owned stretch starts at or after its recording's end
    is dead and its packets are dropped, as are a live segment's from its recording's end on.

    Events are Receiver's dicts with carrier the recording's index, center_hz the identified audio centre (None when the mode
    was given; for information only) and input_seconds the end of the emitting block in seconds of that recording, ordered by
    input_seconds, then carrier. Kinds: "acars" (Receiver's fields) and, with emit_packets, "rtpacket": type ("R" or "T"),
    nsus and bytes. carriers(), unplanned() and stats() report the plan and the counts. Use as a context manager, or call
    close()."""

    def __init__(self, sample_rate, modes=None, identify_seconds=60.0, block_seconds=0.1, segment_seconds=10, lead_seconds=None,
                 max_channels=4096, emit_packets=False, device=0, stream=None):
        try:
            ok = not isinstance(sample_rate, bool) and float(sample_rate) > 0 and float(sample_rate) == int(float(sample_rate))
        except (TypeError, ValueError, OverflowError):
            ok = False
        if not ok:
            raise ValueError("BurstAudioDecoder: sample_rate must be a positive whole number of hertz, got %r" % (sample_rate,))
        rate = int(float(sample_rate))
        ratio = (1, 1)
        if rate != OUT_RATE:
            lib()                                                 # a library that is not built is not a bad rate
            try:
                plan = resample_plan(rate, OUT_RATE, 0.45 * min(rate, OUT_RATE))
            except JaeroError as e:
                raise ValueError("BurstAudioDecoder: sample_rate %d Hz cannot be converted to 48 kHz: %s" % (rate, e)) from None
            ratio = (plan["L"], plan["M"])
        self.geometry = burst_layout(rate, block_seconds, segment_seconds, lead_seconds, max_channels, ratio)
        try:
            ok = float(identify_seconds) > 0 and math.isfinite(float(identify_seconds))
        except (TypeError, ValueError):
            ok = False
        if not ok:
            raise ValueError("BurstAudioDecoder: identify_seconds must be a positive number of seconds, got %r"
                             % (identify_seconds,))
        for m in (list(modes) if isinstance(modes, (list, tuple)) else [modes]):
            _check_mode(m)
        self.sample_rate, self.segment_seconds, self.identify_seconds = rate, int(segment_seconds), float(identify_seconds)
        self.block_n = int(round(float(block_seconds) * rate))
        self.modes = modes
        self.emit_packets, self.device, self._stream_arg = bool(emit_packets), int(device), stream
        self._groups, self._carriers, self._reasm, self._unplanned = [], [], [], []
        self._n_in = np.zeros(0, dtype=np.int64)
        self._clipped = np.zeros(0, dtype=np.int64)
        self._read = 0
        self._used = False

    # ---------------------------------------------------------------------------------------------------------- decode
    def decode(self, recordings):
        """recordings: a list of 1-D int16 host arrays, one burst carrier each -> every event of every recording"""
        if self._used:
            raise ValueError("BurstAudioDecoder: decode() was already called; new recordings need a new BurstAudioDecoder")
        if isinstance(recordings, np.ndarray) or not isinstance(recordings, (list, tuple)):
            raise ValueError("BurstAudioDecoder: recordings must be a list of 1-D int16 arrays, got %s"
                             % type(recordings).__name__)
        recs = []
        for i, r in enumerate(recordings):
            a = r if isinstance(r, np.ndarray) else np.asarray(r)
            if a.ndim != 1 or a.dtype != np.int16:
                raise ValueError("BurstAudioDecoder: recording %d must be 1-D int16 PCM, got %s of shape %s" % (i, a.dtype, a.shape))
            if a.size == 0:
                raise ValueError("BurstAudioDecoder: recording %d is empty" % i)
            recs.append(a)
        if not recs:
            raise ValueError("BurstAudioDecoder: recordings is empty")
        if isinstance(self.modes, (list, tuple)):
            if len(self.modes) != len(recs):
                raise ValueError("BurstAudioDecoder: modes has %d entries for %d recordings" % (len(self.modes), len(recs)))
            modes = list(self.modes)
        else:
            modes = [self.modes] * len(recs)
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
            return _ordered(self._run(recs, modes))

    def _run(self, recs, modes):
        torch, rate, R = self._torch, self.sample_rate, len(recs)
        per_s = OUT_RATE
        self._n_in = np.array([len(r) for r in recs], dtype=np.int64)
        geo = next(iter(self.geometry.values()))
        ends = -(-self._n_in // self.block_n)                     # per recording: its blocks, the last one zero-padded
        who = [c for c in range(R) if modes[c] is None]
        ident_n = min(int(round(self.identify_seconds * per_s)), int(ends[who].max()) * geo.m) if who else 0
        kept = -(-ident_n // per_s)                               # seconds kept on the device while identifying
        rs = ident = None
        try:
            if rate != OUT_RATE:
                rs = Resampler(rate, R, device=self.device)
                rs.set_stream(self.stream)
            head = None
            found = {}
            if who:
                head = torch.empty((R, kept * per_s), dtype=torch.int16, device=self._dev)
                for s in range(kept):
                    head[:, s * per_s:(s + 1) * per_s].copy_(self._second(recs, s, rs))
                rows = head[who]
                ident = Identifier(float(OUT_RATE), len(who), device=self.device)
                ident.set_stream(self.stream)
                for a in range(0, ident_n, geo.m):
                    k = min(geo.m, ident_n - a)
                    ident.write_device(rows.data_ptr() + 2 * a, k, rows.stride(0))
                sq, frames = ident.read()
                found = {c: identify(sq[k], float(OUT_RATE), frames) for k, c in enumerate(who)}
            self._plan(R, modes, found, ends)
            # whole-second writes up to the end of the longest decoded recording; the undecoded ones are not read further
            last = max((int(g.ends.max()) for g in self._groups), default=0)
            ev = []
            self._read = max(kept, -(-last // geo.per))
            for s in range(-(-last // geo.per)):
                pcm = head[:, s * per_s:(s + 1) * per_s] if s < kept else self._second(recs, s, rs)
                for g in self._groups:
                    ev += self._feed(g, pcm)
            head = None
            self._clipped = rs.stats()[1] if rs is not None else np.zeros(R, dtype=np.int64)
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
            raise RuntimeError("BurstAudioDecoder: a second of input gave %d samples at 48 kHz, not %d" % (m, OUT_RATE))
        return torch.as_tensor(_Raw(p, len(recs) * stride, "<i2"), device=self._dev).view(len(recs), stride)[:, :m]

    def _plan(self, R, modes, found, ends):
        self._carriers, self._reasm, self._unplanned = [None] * R, [None] * R, []
        rows = {}
        for c in range(R):
            r = found.get(c)
            d = dict(mode=modes[c], mode_given=modes[c] is not None, center_hz=None, ident_score_db=None)
            if r is not None:
                best = max(FROM_IDENT, key=lambda k: r["score_db"][k])
                score = float(r["score_db"][best])
                d.update(center_hz=float(r["carrier_hz"]), ident_score_db=score,
                         mode=FROM_IDENT[best] if score >= IDENT_THRESHOLD_DB else "unknown")
            if d["mode"] == "unknown":
                self._unplanned.append(dict(d, index=c, reason="unknown mode"))
                continue
            self._carriers[c] = d
            rows.setdefault(d["mode"], []).append(c)
        for mode in BURST_MODES:
            if mode in rows:
                self._groups.append(_Group(mode, rows[mode], self.geometry[mode], ends[rows[mode]]))
                self._groups[-1].rows_t = self._torch.as_tensor(rows[mode], dtype=self._torch.int64, device=self._dev)
                for c in rows[mode]:
                    self._reasm[c] = Reassembler()
        z = lambda: np.zeros(R, dtype=np.int64)
        self._packets, self._messages = z(), z()

    # ---------------------------------------------------------------------------------------------------------- chunks
    def _feed(self, g, pcm):
        """appends one second of the group's rows, up to the end of its longest recording; decodes every chunk that fills"""
        geo = g.geo
        left = int(g.ends.max()) * geo.m - (g.g0 * geo.seg * geo.m + g.fill)
        k = min(pcm.shape[1], left)
        if k <= 0:
            return []
        rows = pcm[g.rows_t, :k]
        ev, a, full = [], 0, geo.chunk_blocks(g.S) * geo.m
        while a < k:
            if g.P is None:
                g.P = self._torch.empty((g.n, g.cap), dtype=self._torch.int16, device=self._dev)
                g.pcm_peak = max(g.pcm_peak, g.P.numel() * 2)
            z = min(k - a, full - g.fill)
            g.P[:, g.fill:g.fill + z].copy_(rows[:, a:a + z])
            g.fill += z
            a += z
            if g.fill >= full:
                ev += self._chunk(g, final=False)
        return ev

    def _chunk(self, g, final):
        """Demodulates the segments g.g0 .. g.g0 + S - 1 of every row of g as one burst batch with its R/T layer, stitches their
        packets (with those held back from the previous chunk) and forms the events of every packet not held back for the next
        chunk. A chunk before the last runs every segment over its whole window; the last one has every segment whose owned
        stretch starts before its row's end, each running its window or up to the end, and the last one to the end. Segments
        run in lockstep: one whose PCM has ended is fed zeros while the others go on, and its packets are dropped."""
        torch, geo, m = self._torch, g.geo, g.geo.m
        blocks = g.fill // m                                      # every row holds whole blocks
        if final:
            S = min(g.S, geo.final_segments(blocks))
            J = max(min(geo.window, blocks), blocks - (S - 1) * geo.seg)
            g.P[:, g.fill:((S - 1) * geo.seg + J) * m].zero_()
        else:
            S, J = g.S, geo.window
        end, alive = geo.rows(g.g0, S, blocks, g.ends)            # per row and segment: local blocks that hold PCM, live
        C = g.n * S
        g.width = max(g.width, C)
        g.segments += int(alive.sum())
        # per channel the local blocks it owns: from its start (segment 0: the recording's start) to the next segment's start,
        # or to the end for the chunk's last segment of the recording's last chunk; never past its PCM
        gs = g.g0 + np.arange(S)
        own_lo = np.where(gs > 0, geo.lead, 0)[None, :].repeat(g.n, 0)
        own_hi = np.minimum(np.where(final & (np.arange(S) == S - 1), J, geo.lead + geo.seg)[None, :], end)
        own_lo, own_hi, live_rows = own_lo.reshape(-1), own_hi.reshape(-1), alive.reshape(-1)
        cuts = {int(x) for x in own_lo} | {int(x) for x in own_hi if 0 < x <= J} | {J}
        Batch = BurstOqpskBatch if g.mode == "burst_oqpsk10500" else BurstMskBatch
        demod = rt = None
        pk_ch, pk_j, pk_rec = [], [], []
        try:
            demod = Batch(C, fb=float(FB[g.mode]), device=self.device)
            rt = RTChannelBatch(C, FB[g.mode], device=self.device)
            out = np.empty((C, 8, RTChannelBatch.RECORD), dtype=np.uint8)
            counts = np.zeros(C, dtype=np.int32)
            x = torch.empty(C * m, dtype=torch.int16, device=self._dev)
            P, bad0, j0 = g.P, np.zeros(C, dtype=np.int64), 0
            for j in range(J):
                src = P.as_strided((g.n, S, m), (P.stride(0), geo.seg * m, 1), P.storage_offset() + j * m)
                x.view(g.n, S, m).copy_(src)
                self._ts.synchronize()                            # the burst batch runs on its own stream
                demod.write_device(x.data_ptr(), m, m)
                rt.process_burst(demod)                           # returns with the batch done reading x
                if (j + 1) % geo.per == 0:
                    rt.tick()
                rt.read_packets_raw(out, counts)
                counts[~((j < end) & alive).reshape(-1)] = 0
                for ch in np.flatnonzero(counts):
                    for k in range(counts[ch]):
                        hdr = out[ch, k, :16].view(np.int32)
                        pk_rec.append((int(hdr[0]), int(hdr[1]), out[ch, k, 16:16 + int(hdr[2])].tobytes()))
                        pk_ch.append(ch); pk_j.append(j)
                if j + 1 in cuts:                                 # CRC failures in each channel's owned blocks
                    bad = rt.stats()[1].astype(np.int64)
                    owned = live_rows & (own_lo <= j0) & (j + 1 <= own_hi)
                    np.add.at(g.crc_failures, np.arange(C)[owned] // S, (bad - bad0)[owned])
                    bad0, j0 = bad, j + 1
        finally:
            for o in (rt, demod):
                if o is not None:
                    o.close()
        ch = np.asarray(pk_ch, dtype=np.int64)
        gsp = g.g0 + ch % S
        tab = dict(row=ch // S, gs=gsp, t=gsp * geo.seg + np.asarray(pk_j, dtype=np.int64), rec=pk_rec)
        if g.held is not None:
            tab = {k: (g.held[k] + tab[k] if k == "rec" else np.concatenate([g.held[k], tab[k]])) for k in tab}
        ev = self._stitched(g, tab, S, final)
        if not final:
            keep = g.fill - S * geo.seg * m                       # the next chunk's first window: [b - lead, b + guard)
            g.P[:, :keep] = g.P[:, S * geo.seg * m:g.fill].clone()
            g.fill, g.g0 = keep, g.g0 + S
        else:
            g.fill, g.P = 0, None
        g.chunks += 1
        return ev

    def _stitched(self, g, tab, S, final):
        geo = g.geo
        row, gs, t, rec = tab["row"], tab["gs"], tab["t"], tab["rec"]
        base, last = g.g0 - (g.held is not None), g.g0 + S - 1
        keep, matched, unmatched = stitch_packets(row, rec, gs - base, t, [geo.start(s) for s in range(base, last + 1)],
                                                  geo.guard, g.ends[row])
        hold = np.zeros(len(t), dtype=bool)
        if not final:                       # packets the next chunk's first segment may also have: stitched with it instead
            hold = (gs == last) & (t >= geo.start(last + 1) - geo.guard - 1)
        np.add.at(g.matched, row[matched & keep & ~hold], 1)
        np.add.at(g.unmatched, row[unmatched & ~hold], 1)
        g.held = None if final else dict(row=row[hold], gs=gs[hold], t=t[hold], rec=[r for r, h in zip(rec, hold) if h])
        sel = np.flatnonzero(keep & ~hold)
        sel = sel[np.lexsort((t[sel], row[sel]))]                 # stable: a block's packets stay in the order read
        ev = []
        for i in sel:
            c = int(g.index[row[i]])
            sec = min((int(t[i]) + 1) * self.block_n, int(self._n_in[c])) / self.sample_rate
            ev += self._packet(c, rec[i], sec)
        return ev

    def _packet(self, c, rec, t):
        """one stitched packet of recording c, emitted by input second t: counted and pushed to the recording's Reassembler ->
        its "rtpacket" (with emit_packets) and "acars" events"""
        kind, nsus, info = rec
        self._packets[c] += 1
        ev = []
        if self.emit_packets:
            ev.append(self._event("rtpacket", c, t, type="R" if kind == 1 else "T", nsus=nsus, bytes=info))
        rs = self._reasm[c]
        if kind == 1:
            rs.push_r(info, downlink=True)
        else:
            rs.push_t_packet(info, nsus)
        for r in rs.pop_all():
            r["record_kind"], r["acars_mode"] = r.pop("kind"), r.pop("mode")
            self._messages[c] += 1
            ev.append(self._event("acars", c, t, **r))
        return ev

    # ---------------------------------------------------------------------------------------------------------- state
    def carriers(self):
        """the decoded recordings, by index: mode, mode_given (False: identified), and what the identifier found, center_hz and
        the chosen rate's score (None when the mode was given)"""
        return [dict(d, index=c) for c, d in enumerate(self._carriers) if d is not None]

    def unplanned(self):
        """the recordings not decoded, with index and reason ("unknown mode") and what the identifier found"""
        return list(self._unplanned)

    def stats(self):
        """read_seconds: the whole seconds of input read; per recording its length in seconds and the rate converter's clipped
        samples; per decoded recording its packets, R/T CRC failures in the stretches its segments own, ACARS records, and the
        packets matched at segment boundaries (each kept copy once) and kept there without a partner; per mode group its
        recordings, segments decoded, segments per chunk, chunks, widest batch, segment, lead and guard lengths and the PCM
        buffer's peak size"""
        per, groups = {}, []
        for g in self._groups:
            groups.append(dict(mode=g.mode, recordings=g.n, segments=g.segments, segments_per_chunk=g.S, chunks=g.chunks,
                               batch_width=g.width, segment_seconds=self.segment_seconds, lead_seconds=g.geo.lead // g.geo.per,
                               guard_seconds=g.geo.guard / g.geo.per, pcm_bytes_peak=g.pcm_peak))
            for r, c in enumerate(g.index):
                c = int(c)
                per[c] = dict(index=c, mode=g.mode, packets=int(self._packets[c]), crc_failures=int(g.crc_failures[r]),
                              messages=int(self._messages[c]), boundary_matches=int(g.matched[r]), unmatched=int(g.unmatched[r]))
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


def _check_mode(m):
    if m is None or m in BURST_MODES:
        return
    if m in CONTINUOUS_MODES:
        raise ValueError("BurstAudioDecoder: modes: %r is a continuous mode; continuous recordings are decoded by AudioDecoder"
                         % (m,))
    raise ValueError("BurstAudioDecoder: modes: %r is not one of the burst modes %s" % (m, ", ".join(BURST_MODES)))
