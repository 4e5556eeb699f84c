"""Decode a recorded band's carriers as parallel time segments and stitch them into one message stream per carrier.

A carrier's demodulator state depends only on the last few seconds of its signal, so one carrier's recording can be cut into
segments that are demodulated side by side, as channels of one DemodBatch: each segment starts a lead early, from a cold start,
so it is locked by the time the stretch it owns begins, and runs a guard past its end, so the frame that straddles the boundary
is decoded whole by both neighbours. The demodulator batches then run at the widths they were built for instead of a few
channels wide. RecordingDecoder is Receiver with that change: the same acquisition, plan, down-converters, events and counts;
the down-converters' output is kept on the device until a chunk of segments is due, and the frames of neighbouring segments
are stitched on the host (stitch) into the stream Receiver would have decoded.
"""
import math

import numpy as np

from . import CChannelBatch, DemodBatch, Ddc, PChannelBatch, rate_ratio
from .receiver import P_MODES, Receiver, _Events, _Raw

MODES = ("msk600", "msk1200", "oqpsk10500", "oqpsk8400")
FRAME_SECONDS = {"msk600": 2.0, "msk1200": 1.0, "oqpsk10500": 0.5, "oqpsk8400": 4096 / 8400.0}
# Seconds a segment starts before the stretch it owns: at least twice the longest time from a cold start to the first
# CRC-valid frame measured on the synthetic band of tests/test_gpu_recording.py (5.2, 3.1 and 2.6 s at 600, 1200 and
# 10 500 bps; at 8400 bps 5.0 s from the start of the recording's signal, DESIGN.md section 5), rounded up to whole seconds.
DEFAULT_LEAD_SECONDS = {"msk600": 11, "msk1200": 7, "oqpsk10500": 6, "oqpsk8400": 10}


class Geometry:
    """One mode's segment grid, counted in the receiver's blocks from the start of the recording.

    per: blocks per second; m: PCM samples per block; seg, lead, guard: the segment, lead and guard lengths; window: the blocks
    one segment demodulates (lead + seg + guard). Segment g demodulates blocks [g seg, g seg + window) and owns the blocks from
    start(g) to start(g + 1): start(0) = 0 (the recording's first segment has no lead), start(g) = g seg + lead. A chunk of S
    segments is one batch of carriers x S channels."""

    def __init__(self, mode, per, m, seg, lead, guard, max_channels):
        self.mode, self.per, self.m, self.seg, self.lead, self.guard = mode, per, m, seg, lead, guard
        self.window = lead + seg + guard
        self.max_channels = max_channels

    def segments_per_chunk(self, n_carriers):
        """S: as many segments per carrier as keep the batch within max_channels (one, if the carriers alone exceed it)"""
        return max(1, self.max_channels // n_carriers)

    def start(self, g):
        return 0 if g == 0 else g * self.seg + self.lead

    def chunk_blocks(self, S):
        """blocks a chunk of S segments reads, from its first segment's first block"""
        return (S - 1) * self.seg + self.window

    def rows(self, g0, S, blocks, ends=None):
        """The grid of a chunk of S segments from segment g0 whose PCM holds `blocks` blocks from g0's first block -> (end,
        alive), both [rows, S]: end the local blocks each segment has PCM for, alive whether its owned stretch starts before its
        row's end. ends: None when every row runs to the end of the PCM (one row), else per row the block its signal ends at"""
        local = np.arange(S) * self.seg
        if ends is None:
            return (blocks - local)[None, :], np.ones((1, S), dtype=bool)
        ends = np.asarray(ends, dtype=np.int64)
        end = np.minimum(blocks, ends[:, None] - g0 * self.seg) - local[None, :]
        alive = np.array([self.start(g0 + s) for s in range(S)])[None, :] < ends[:, None]
        return end, alive

    def final_segments(self, blocks):
        """segments of the last chunk when `blocks` blocks remain from its first segment's first block: every segment whose
        owned stretch starts before the end (at least one); the last one owns everything after its start"""
        return 1 + max(0, -(-(blocks - self.lead) // self.seg) - 1)


def layout(input_rate, block_seconds, segment_seconds, lead_seconds=None, max_channels=4096, owner="RecordingDecoder",
           ratio=None):
    """Checks the segment settings against Receiver's block grid -> {mode: Geometry}.

    Segment boundaries, starts and leads are whole seconds, a second is a whole number of blocks and every block gives the same
    number of 48 kHz samples (block samples x interpolation divisible by decimation), so every segment runs on Receiver's block
    grid and its 1 s DCD-tick grid. A block is at most a quarter of the shortest frame, so frames match by time without
    ambiguity, and a segment is longer than two guards, so the windows around neighbouring boundaries do not meet. lead_seconds:
    None (DEFAULT_LEAD_SECONDS), seconds for every mode, or a dict of seconds by mode over the defaults. ValueError otherwise,
    its text headed by `owner`, the class the settings were given to. ratio: the (interpolation, decimation) that brings
    input_rate to 48 kHz, when it is not the down-converter's rate_ratio (the rate converter allows larger ones)."""
    L, D = rate_ratio(input_rate) if ratio is None else ratio
    rate = int(float(input_rate))
    if not 0 < float(block_seconds) <= 1.0:
        raise ValueError(owner + ": block_seconds must be in (0, 1], got %r" % (block_seconds,))
    if isinstance(max_channels, bool) or not isinstance(max_channels, (int, np.integer)) or max_channels < 1:
        raise ValueError(owner + ": max_channels must be a positive whole number, got %r" % (max_channels,))
    seg_s = _whole_seconds(owner, "segment_seconds", segment_seconds)
    if seg_s < 1:
        raise ValueError(owner + ": segment_seconds must be at least 1, got %r" % (segment_seconds,))
    block_n = int(round(float(block_seconds) * rate))
    if block_n < 1 or rate % block_n:
        raise ValueError(owner + ": a second of input (%d samples) is not a whole number of %r s blocks (%d samples)"
                         % (rate, block_seconds, block_n))
    if block_n * L % D:
        raise ValueError(owner + ": a %r s block (%d samples) does not give a whole number of 48 kHz samples at %d Hz "
                         "(%d x %d / %d)" % (block_seconds, block_n, rate, block_n, L, D))
    shortest = min(FRAME_SECONDS.values())
    if block_n / rate > shortest / 4 + 1e-12:
        raise ValueError(owner + ": block_seconds %r is longer than a quarter of the shortest frame (%.4f s at 8400 bps), "
                         "so frames could not be matched by time" % (block_seconds, shortest))
    if lead_seconds is None:
        leads = dict(DEFAULT_LEAD_SECONDS)
    elif isinstance(lead_seconds, dict):
        unknown = sorted(set(lead_seconds) - set(MODES))
        if unknown:
            raise ValueError(owner + ": lead_seconds for unknown mode(s) %s" % ", ".join(unknown))
        leads = dict(DEFAULT_LEAD_SECONDS, **lead_seconds)
    else:
        leads = {mode: lead_seconds for mode in MODES}
    per, m = rate // block_n, block_n * L // D
    out = {}
    for mode in MODES:
        lead = _whole_seconds(owner, "lead_seconds", leads[mode])
        guard = int(math.ceil(FRAME_SECONDS[mode] * per - 1e-9)) + 1
        if seg_s * per <= 2 * guard + 2:
            raise ValueError(owner + ": segment_seconds %r is too short for %s: a segment must be longer than two guards "
                             "of %.2f s (its longest frame and one block)" % (segment_seconds, mode, guard / per))
        out[mode] = Geometry(mode, per, m, seg_s * per, lead * per, guard, int(max_channels))
    return out


def _whole_seconds(owner, name, v):
    try:
        f = float(v)
    except (TypeError, ValueError):
        raise ValueError(owner + ": %s must be a whole number of seconds, got %r" % (name, v)) from None
    if not (f >= 0 and f == int(f)):
        raise ValueError(owner + ": %s must be a whole number of seconds, got %r" % (name, v))
    return int(f)


def stitch(car, seg, t, starts, guard, ends=None):
    """Which frames of consecutive segments of the same carriers make one stream.

    car, seg, t: per frame its carrier, its segment (an index into starts) and the block it was emitted in. starts[s]: the first
    block segment s owns; segment 0 owns everything before starts[1] and the last segment everything from its start on. Around
    each boundary b = starts[s + 1], a frame of s and one of s + 1 emitted at most one block apart, one of them within
    [b - guard, b + guard], are the same frame: the copy emitted inside its own segment's owned stretch is kept, or s's copy when
    both or neither are. A frame within that window without such a partner is kept. Every other frame is kept when it was
    emitted in its segment's owned stretch. Frames of one segment must be at least three blocks apart.
    ends: None, or per frame the block its carrier's signal ends at; a boundary at or after it is not one of that carrier's, so
    the segment before it is the carrier's last.
    -> (keep, matched, unmatched): boolean masks; matched marks both copies of a matched frame, unmatched the partnerless frames
    kept in a window."""
    car, seg, t = (np.asarray(x, dtype=np.int64).reshape(-1) for x in (car, seg, t))
    starts = np.asarray(starts, dtype=np.int64)
    n, ns = len(t), len(starts)
    none = np.zeros(n, dtype=bool)
    if n == 0:
        return none, none.copy(), none.copy()
    far = np.int64(1) << 50
    nxt = starts[np.minimum(seg + 1, ns - 1)]
    has_next = seg < ns - 1
    if ends is not None:
        has_next &= nxt < np.asarray(ends, dtype=np.int64).reshape(-1)
    lo = np.where(seg > 0, starts[seg], -far)
    hi = np.where(has_next, nxt, far)
    in_lw = (seg > 0) & (np.abs(t - lo) <= guard)
    in_rw = has_next & (np.abs(t - hi) <= guard)
    keep = (t >= lo) & (t < hi)
    # partner of each frame of s near its right boundary: the first frame of s + 1 at t - 1 or later
    span = int(t.max()) + 3
    key = (car * ns + seg) * span + t + 1
    order = np.argsort(key, kind="stable")
    ks = key[order]
    cand = np.flatnonzero(has_next & (np.abs(t - hi) <= guard + 1))
    pos = np.searchsorted(ks, (car[cand] * ns + seg[cand] + 1) * span + t[cand])
    j = order[np.minimum(pos, n - 1)]
    ok = ((pos < n) & (car[j] == car[cand]) & (seg[j] == seg[cand] + 1) & (np.abs(t[j] - t[cand]) <= 1)
          & (in_rw[cand] | in_lw[j]))
    i, j = cand[ok], j[ok]
    j, first = np.unique(j, return_index=True)
    i = i[first]
    b = hi[i]
    take_j = (t[j] >= b) & ~(t[i] < b)
    keep[i], keep[j] = ~take_j, take_j
    matched = none.copy()
    matched[i] = matched[j] = True
    unmatched = (in_lw | in_rw) & ~matched
    keep |= unmatched
    return keep, matched, unmatched


class _Segments:
    """One mode group of the segment engine: its rows (index: their carrier indices, in row order), the PCM not decoded yet,
    P[row, t] (int16 on the device, from the first block of segment g0's window on), the frames held back for the next chunk's
    stitch, and the counts stats() reports. ends: None when every row runs to the end of the input, else per row the block its
    signal ends at. ddc: RecordingDecoder's down-converter for the group, fed every block as in Receiver"""

    def __init__(self, mode, index, demod_kw, geo, ends=None):
        self.mode, self.index, self.geo = mode, np.asarray(index, dtype=np.int64), geo
        self.n, self.first = len(self.index), int(self.index[0])
        self.ends = None if ends is None else np.asarray(ends, dtype=np.int64)
        self.ddc = None
        self.demod_kw = dict(demod_kw)
        self.S = geo.segments_per_chunk(self.n)
        self.P, self.fill, self.g0 = None, 0, 0
        self.chunks = self.width = self.pcm_peak = 0
        self.held = None
        self.status = [dict(dcd=0, ebno=0.0)] * self.n
        z = lambda: np.zeros(self.n, dtype=np.int64)
        self.matched, self.unmatched, self.late, self.unlocked, self.lock_blocks = z(), z(), z(), z(), z()

    def close(self):
        if self.ddc is not None:
            self.ddc.close(); self.ddc = None
        self.P = None


class _SegmentEngine(_Events):
    """Decodes mode groups (_Segments) of 48 kHz device PCM as parallel time segments: _take appends a group's PCM, _chunk
    demodulates a chunk of segments once it is due, stitches their frames and forms the events. Needs self._groups,
    self._torch, self._dev, self.device, self.stream and _event_seconds(carrier, block), besides what _Events needs."""

    def _take(self, g, rows):
        """appends device PCM rows [g.n, k] to g.P, up to where the next chunk is due -> the samples taken"""
        k = min(rows.shape[1], g.geo.chunk_blocks(g.S) * g.geo.m - g.fill)
        self._reserve(g, g.fill + k)
        g.P[:, g.fill:g.fill + k].copy_(rows[:, :k])
        g.fill += k
        return k

    def _due(self, g):
        return g.fill >= g.geo.chunk_blocks(g.S) * g.geo.m

    def _reserve(self, g, need):
        """P holds at least `need` samples per carrier: it grows by doubling up to one chunk's PCM"""
        cap = 0 if g.P is None else g.P.shape[1]
        if need <= cap:
            return
        full = g.geo.chunk_blocks(g.S) * g.geo.m
        new = self._torch.empty((g.n, min(full, max(need, 2 * cap, 16 * g.geo.per * g.geo.m))), dtype=self._torch.int16,
                                device=self._dev)
        if g.fill:
            new[:, :g.fill].copy_(g.P[:, :g.fill])
        g.P = new
        g.pcm_peak = max(g.pcm_peak, new.numel() * 2)

    # ---------------------------------------------------------------------------------------------------------- chunks
    def _chunk(self, g, final):
        """Demodulates the segments g.g0 .. g.g0 + S - 1 of every row of g as one batch, stitches their frames (with those
        held back from the previous chunk) and forms the events of every frame not held back for the next chunk.

        A chunk before the last runs every segment over its whole window. The last chunk has every segment whose owned stretch
        starts before the end of the input; each runs its window or up to the end, whichever comes first, and the last one
        to the end. Segments run in lockstep, so one whose PCM has ended is fed zeros while the others go on, and its records
        from then on are dropped. Where a segment's last block is short, the block is written in two parts, so that segment's
        last write ends where the input ends, as Receiver's does. Where rows end at different blocks (g.ends), a segment whose
        owned stretch starts at or after its row's end is dead: it runs on zeros and all its records are dropped."""
        torch, geo, m = self._torch, g.geo, g.geo.m
        blocks = -(-g.fill // m)
        if final:
            S = min(g.S, geo.final_segments(blocks))
            J = max(min(geo.window, blocks), blocks - (S - 1) * geo.seg)
            self._reserve(g, ((S - 1) * geo.seg + J) * m)
            g.P[:, g.fill:((S - 1) * geo.seg + J) * m].zero_()
        else:
            S, J = g.S, geo.window
        part = g.fill - (blocks - 1) * m                          # samples in the input's last block (m if it is whole)
        end, alive = geo.rows(g.g0, S, blocks, g.ends)            # per row and segment: local blocks that hold PCM, live
        end, alive = np.broadcast_to(end, (g.n, S)), np.broadcast_to(alive, (g.n, S))
        # per row: its last live segment and the block after which its status is read (-1: no live segment)
        s_last = S - 1 - np.argmax(alive[:, ::-1], axis=1)
        at = np.where(alive.any(axis=1), np.minimum(end[np.arange(g.n), s_last], J) - 1, -1)
        C = g.n * S
        g.width = max(g.width, C)
        kw = dict(g.demod_kw, n_channels=C)
        if np.ndim(kw.get("freq_center", 0)):                    # a centre per row: the same for each of its segments
            kw["freq_center"] = np.repeat(np.asarray(kw["freq_center"], dtype=np.float64), S)
        demod = layer = None
        recs, chans, js = [], [], []
        try:
            demod = DemodBatch(device=self.device, **kw)
            demod.set_stream(self.stream)
            if g.mode in P_MODES:
                layer = PChannelBatch(C, g.demod_kw["fb"], device=self.device)
                out, width = np.empty((C, layer.su_cap, 16), dtype=np.uint8), 16
                read = layer.read_sus_raw
            else:
                layer = CChannelBatch(C, device=self.device)
                out, width = np.empty((C, 8, CChannelBatch.RECORD), dtype=np.uint8), CChannelBatch.RECORD
                read = layer.read_frames_raw
            counts = np.zeros(C, dtype=np.int32)
            x = torch.empty(C * m, dtype=torch.int16, device=self._dev)
            P = g.P

            def step(j, a, z, live):
                """samples [a, z) of local block j for every channel; keeps the records of the segments in `live`"""
                src = P.as_strided((g.n, S, z - a), (P.stride(0), geo.seg * m, 1), P.storage_offset() + j * m + a)
                x[:C * (z - a)].view(g.n, S, z - a).copy_(src)
                demod.write_device(x.data_ptr(), z - a, z - a)
                layer.process_batch(demod)
                if z == m and (j + 1) % geo.per == 0:
                    layer.tick(demod)
                read(out, counts)
                counts[~live.reshape(-1)] = 0
                k = int(counts.sum())
                if k:
                    recs.append(out[np.arange(out.shape[1])[None, :] < counts[:, None]])
                    chans.append(np.repeat(np.arange(C), counts))
                    js.append(np.full(k, j, dtype=np.int64))

            def status(j):
                rows = np.flatnonzero(at == j)
                if len(rows):
                    st = demod.status()
                    g.status = list(g.status)
                    for c in rows:
                        g.status[c] = st[c * S + s_last[c]]

            for j in range(J):
                live, whole = (j < end) & alive, (j < end - 1) & alive
                if part < m and (live & ~whole).any():
                    # some segment's PCM ends inside this block
                    step(j, 0, part, live)
                    status(j)
                    if whole.any():
                        step(j, part, m, whole)
                else:
                    step(j, 0, m, live)
                    status(j)
        finally:
            for o in (layer, demod):
                if o is not None:
                    o.close()
        # the chunk's records, in the order they were read: row, global segment, emission block
        rec = np.concatenate(recs) if recs else np.zeros((0, width), dtype=np.uint8)
        ch = np.concatenate(chans) if chans else np.zeros(0, dtype=np.int64)
        j = np.concatenate(js) if js else np.zeros(0, dtype=np.int64)
        car, gs = ch // S, g.g0 + ch % S
        tab = dict(rec=rec, car=car, gs=gs, t=gs * geo.seg + j)
        self._locks(g, tab, S, alive)
        if g.held is not None:
            tab = {k: np.concatenate([g.held[k], tab[k]]) for k in tab}
        ev = self._stitched(g, tab, S, final)
        if not final:
            keep = g.fill - S * geo.seg * m                       # the next chunk's first window: [b - lead, b + guard)
            g.P[:, :keep] = g.P[:, S * geo.seg * m:g.fill].clone()
            g.fill, g.g0 = keep, g.g0 + S
        else:
            g.fill, g.P = 0, None
        g.chunks += 1
        return ev

    def _frame_index(self, g, tab):
        """per record the index of its frame, and per frame whether it holds a CRC-valid unit"""
        rec = tab["rec"]
        if g.mode in P_MODES:
            fno = rec[:, 14].astype(np.int64) | (rec[:, 15].astype(np.int64) << 8)
            valid = rec[:, 12] != 0
        else:
            fno = np.arange(len(rec), dtype=np.int64)
            valid = (rec[:, 12] != 0) | (rec[:, 28] != 0) | (rec[:, 44] != 0)
        n = len(rec)
        new = np.ones(n, dtype=bool)
        if n:
            new[1:] = (tab["car"][1:] != tab["car"][:-1]) | (tab["gs"][1:] != tab["gs"][:-1]) | (tab["t"][1:] != tab["t"][:-1]) \
                | (fno[1:] != fno[:-1])
        fid = np.cumsum(new) - 1
        heads = np.flatnonzero(new)
        fvalid = np.logical_or.reduceat(valid, heads) if n else np.zeros(0, dtype=bool)
        return fid, heads, fvalid

    def _locks(self, g, tab, S, alive):
        """late locks, segments that never locked and the longest time to the first CRC-valid frame, per row, for the chunk's
        segments (late and unlocked count only live segments with a lead)"""
        fid, heads, fvalid = self._frame_index(g, tab)
        h = heads[fvalid]
        car, gs, t = tab["car"][h], tab["gs"][h], tab["t"][h]
        o = np.lexsort((t, gs, car))
        car, gs, t = car[o], gs[o], t[o]
        first = np.ones(len(t), dtype=bool)
        first[1:] = (car[1:] != car[:-1]) | (gs[1:] != gs[:-1])
        car, gs, t = car[first], gs[first], t[first]
        geo = g.geo
        np.maximum.at(g.lock_blocks, car, t - gs * geo.seg + 1)
        late = (gs > 0) & (t >= gs * geo.seg + geo.lead)
        np.add.at(g.late, car[late], 1)
        with_lead = (alive & (g.g0 + np.arange(S) > 0)[None, :]).sum(axis=1)
        g.unlocked += with_lead - np.bincount(car[gs > 0], minlength=g.n)

    def _stitched(self, g, tab, S, final):
        geo = g.geo
        fid, heads, _ = self._frame_index(g, tab)
        car_f, gs_f, t_f = tab["car"][heads], tab["gs"][heads], tab["t"][heads]
        base, last = g.g0 - (g.held is not None), g.g0 + S - 1
        keep, matched, unmatched = stitch(car_f, gs_f - base, t_f, [geo.start(s) for s in range(base, last + 1)], geo.guard,
                                          None if g.ends is None else g.ends[car_f])
        hold = np.zeros(len(heads), dtype=bool)
        if not final:                       # frames the next chunk's first segment may also have: stitched with it instead
            hold = (gs_f == last) & (t_f >= geo.start(last + 1) - geo.guard - 1)
        np.add.at(g.matched, car_f[matched & keep & ~hold], 1)
        np.add.at(g.unmatched, car_f[unmatched & ~hold], 1)
        g.held = None if final else {k: v[hold[fid]] for k, v in tab.items()}
        sel = (keep & ~hold)[fid]
        rec, car, t = tab["rec"][sel], tab["car"][sel], tab["t"][sel]
        o = np.lexsort((t, car))                                  # stable: each frame's records stay in order
        rec, car, t = rec[o], car[o], t[o]
        ev = []
        if not len(t):
            return ev
        cut = np.flatnonzero((car[1:] != car[:-1]) | (t[1:] != t[:-1])) + 1
        for a, z in zip(np.concatenate([[0], cut]), np.concatenate([cut, [len(t)]])):
            c = int(g.index[car[a]])
            sec = self._event_seconds(c, int(t[a]))
            r = rec[a:z]
            if g.mode in P_MODES:
                ev += self._units(c, r, sec)
            else:
                su = r[:, :48].reshape(-1, 3, 16)
                ev += self._cframes(c, su[:, :, :12], su[:, :, 12], r[:, 48:348], r[:, 348:352].copy().view(np.int32).reshape(-1),
                                    sec)
        return ev

    # ---------------------------------------------------------------------------------------------------------- state
    def carriers(self):
        out = []
        for g in self._groups:
            for ch, st in enumerate(g.status):
                c = int(g.index[ch])
                out.append(dict(self._carriers[c], index=c, dcd=bool(st["dcd"]), ebno=st["ebno"]))
        return out

    def _segment_stats(self, per, segment_seconds):
        """per group: the segments per chunk, chunks, widest batch, segment, lead and guard lengths and PCM buffer sizes; adds
        each row's boundary counts, late locks, unlocked segments and lock_seconds to per[carrier index]"""
        groups = []
        for g in self._groups:
            groups.append(dict(mode=g.mode, carriers=g.n, segments_per_chunk=g.S, chunks=g.chunks, batch_width=g.width,
                               segment_seconds=segment_seconds, lead_seconds=g.geo.lead // g.geo.per,
                               guard_seconds=g.geo.guard / g.geo.per,
                               pcm_bytes=0 if g.P is None else int(g.P.numel()) * 2, pcm_bytes_peak=g.pcm_peak))
            for ch in range(g.n):
                per[int(g.index[ch])].update(boundary_matches=int(g.matched[ch]), unmatched=int(g.unmatched[ch]),
                                             late_locks=int(g.late[ch]), unlocked_segments=int(g.unlocked[ch]),
                                             lock_seconds=int(g.lock_blocks[ch]) / g.geo.per)
        return groups


class RecordingDecoder(_SegmentEngine, Receiver):
    """Decodes every continuous carrier of a recorded band (cu8 or cs16 IQ at any whole-hertz rate) as parallel time segments.

    The constructor takes Receiver's arguments plus:
      segment_seconds: the stretch of each carrier one demodulator channel owns (whole seconds);
      lead_seconds: how long before its stretch a segment starts (None: DEFAULT_LEAD_SECONDS by mode; seconds; or a dict by mode);
      max_channels: the widest demodulator batch; each mode group cuts S = max_channels // carriers segments per chunk.
    layout() lists the checks on them.

    Acquisition and down-conversion are Receiver's. Each mode group keeps its Ddc's output on the device; once it holds a chunk
    (S segments, plus the lead and guard of the next boundary), one DemodBatch of carriers x S channels and its frame layer
    decode every segment of the chunk at once, block by block and ticked once per second as Receiver does, and stitch() joins
    the segments' frames. flush() decodes the rest. Events are Receiver's, with input_seconds the end of the block the frame was
    emitted in; each call returns them ordered by input_seconds, then carrier. A chunk's events come when it is decoded, so the
    latency is up to one chunk (S x segment_seconds plus the lead and guard). flush() ends the recording.

    stats() adds per group the segments per chunk, the chunks decoded and the widest batch, and per carrier the frames matched at
    boundaries, the partnerless frames kept there, late locks (segments with a lead whose first CRC-valid frame was emitted in
    or after their owned stretch, where signal units can be lost), unlocked segments (segments with a lead that gave no
    CRC-valid frame at all) and lock_seconds, the longest time from a segment's start to its first CRC-valid frame. carriers()
    reports each carrier's DCD and Eb/N0 at the end of the last segment decoded. The PCM buffer is freed when flush() has
    decoded the last chunk."""

    def __init__(self, input_rate, fmt, acquire_seconds=4.0, block_seconds=0.1, device=0, stream=None, scan_nfft=1 << 16,
                 emit_sus=False, segment_seconds=10, lead_seconds=None, max_channels=4096, **find_params):
        self.geometry = layout(input_rate, block_seconds, segment_seconds, lead_seconds, max_channels)
        self.segment_seconds = int(segment_seconds)
        self._ended = False
        super().__init__(input_rate, fmt, acquire_seconds=acquire_seconds, block_seconds=block_seconds, device=device,
                         stream=stream, scan_nfft=scan_nfft, emit_sus=emit_sus, **find_params)

    # ---------------------------------------------------------------------------------------------------------- input
    def write(self, iq):
        self._open()
        return _ordered(super().write(iq))

    def write_device(self, ptr, n_iq):
        self._open()
        return _ordered(super().write_device(ptr, n_iq))

    def flush(self):
        """Decodes the rest of the recording and ends it -> new events"""
        if self._ended:
            return []
        ev = super().flush()
        with self._torch.cuda.stream(self._ts):
            for g in self._groups:
                if g.fill:
                    ev += self._chunk(g, final=True)
        self._ended = True
        return _ordered(ev)

    def _open(self):
        if self._ended:
            raise ValueError("RecordingDecoder: the recording was flushed; a new recording needs a new RecordingDecoder")

    def _new_group(self, mode, plan, first):
        g = _Segments(mode, range(first, first + len(plan["carriers"])), plan["demod"], self.geometry[mode])
        g.ddc = Ddc(device=self.device, **plan["ddc"])
        g.ddc.set_stream(self.stream)
        return g

    def _event_seconds(self, c, t):
        return min((t + 1) * self.block_n, self._n_in) / self.input_rate

    # ---------------------------------------------------------------------------------------------------------- blocks
    def _block(self, ptr, n):
        torch = self._torch
        for g in self._groups:
            g.ddc.write_device(ptr, n, self.fmt)
            p, m, stride = g.ddc.output()
            if n == self.block_n and m != g.geo.m:
                raise RuntimeError("RecordingDecoder: a block gave %d PCM samples, not %d" % (m, g.geo.m))
            if m:
                rows = torch.as_tensor(_Raw(p, g.n * stride, "<i2"), device=self._dev).view(g.n, stride)
                self._take(g, rows[:, :m])                        # a chunk is due only after a whole block: it takes all m
        self._n_in += n
        self._blocks += 1
        ev = []
        for g in self._groups:
            if self._due(g):
                ev += self._chunk(g, final=False)
        return ev

    # ---------------------------------------------------------------------------------------------------------- state
    def stats(self):
        st = super().stats()
        st["groups"] = self._segment_stats(st["carriers"], self.segment_seconds)
        return st


def _ordered(ev):
    return sorted(ev, key=lambda e: (e["input_seconds"], e["carrier"]))
