"""One receiver for a whole band: wideband SDR IQ in, ACARS messages, signal units and C-channel frames out.

Receiver joins the existing stages without changing any of them: the carrier scanner (Scanner, find_carriers), the mode
identifier (probe_carriers), the planner (channel_plan), the down-converter (Ddc), the continuous demodulators (DemodBatch), the
P- and C-channel frame layers and the message layer (Reassembler). Per block the host only passes device pointers between
the stages and reads back the decoded bytes; every per-sample step is one of the library's kernels.
"""
import numpy as np

from . import (IQ_CU8, CChannelBatch, DemodBatch, Ddc, PChannelBatch, Reassembler, Scanner, _host_iq, _iq_format,
               channel_plan, find_carriers, probe_carriers, rate_ratio)

FIND_PARAMS = ("threshold_db", "floor_window_hz", "floor_quantile", "min_width_hz", "dc_guard_hz")
P_MODES = ("msk600", "msk1200", "oqpsk10500")          # P-channel frame layer; oqpsk8400 gets the C-channel layer


class _Raw:
    """A device buffer given as a pointer, for torch.as_tensor (the CUDA array interface)"""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = dict(shape=(int(n),), typestr=typestr, data=(int(ptr), False), strides=None, version=2)


class _Group:
    """The stages of one mode: a Ddc, a DemodBatch and its frame layer, fed from the same IQ blocks"""

    def __init__(self, mode, plan, first, device, stream):
        self.mode, self.first, self.n = mode, first, len(plan["carriers"])
        self.ddc = self.demod = self.layer = None
        self.ddc = Ddc(device=device, **plan["ddc"])
        self.demod = DemodBatch(device=device, **plan["demod"])
        self.ddc.set_stream(stream); self.demod.set_stream(stream)
        if mode in P_MODES:
            self.layer = PChannelBatch(self.n, plan["demod"]["fb"], device=device)
            self.su_out = np.empty((self.n, self.layer.su_cap, 16), dtype=np.uint8)
            self.su_counts = np.zeros(self.n, dtype=np.int32)
        else:
            self.layer = CChannelBatch(self.n, device=device)

    def close(self):
        for o in (self.layer, self.demod, self.ddc):
            if o is not None:
                o.close()


class _Events:
    """Event formation shared by the decoders: a carrier's signal-unit records or C-channel frames -> its events, counted per
    carrier. Needs self._carriers (carrier index -> dict with mode and center_hz), self._reasm (its Reassembler, P-channel
    carriers), self.emit_sus and the counters self._su_total, self._su_bad, self._messages and self._frames."""

    def _event(self, kind, c, t, **fields):
        car = self._carriers[c]
        return dict(kind=kind, carrier=c, center_hz=car["center_hz"], mode=car["mode"], input_seconds=t, **fields)

    def _units(self, c, recs, t):
        """carrier c's signal-unit records (read_sus_raw rows), decoded by input second t: counted, the CRC-valid ones pushed to
        the carrier's Reassembler -> their "su" (with emit_sus) and "acars" events"""
        ev = []
        ok = recs[:, 12] != 0
        self._su_total[c] += len(recs); self._su_bad[c] += int((~ok).sum())
        rs = self._reasm[c]
        for r in recs[ok]:
            su = r[:12].tobytes()
            if self.emit_sus:
                ev.append(self._event("su", c, t, su=su, index=int(r[13]), frame=int(r[14]) | (int(r[15]) << 8)))
            rs.push_su(su)
        for rec in rs.pop_all():
            rec["record_kind"], rec["acars_mode"] = rec.pop("kind"), rec.pop("mode")
            self._messages[c] += 1
            ev.append(self._event("acars", c, t, **rec))
        return ev

    def _cframes(self, c, su, ok, voice, frame, t):
        """carrier c's C-channel frames (read_frames arrays), decoded by input second t: counted -> their "cframe" events"""
        ev = []
        for k in range(len(frame)):
            self._frames[c] += 1; self._su_total[c] += 3; self._su_bad[c] += int((ok[k] == 0).sum())
            ev.append(self._event("cframe", c, t, sus=[x.tobytes() for x in su[k]], crc_ok=[bool(x) for x in ok[k]],
                                  voice=voice[k].tobytes(), frame=int(frame[k])))
        return ev


class Receiver(_Events):
    """Decodes every continuous carrier of one wideband SDR IQ stream (cu8 or cs16 at any whole-hertz rate) on one GPU.

    Acquisition: the first acquire_seconds of IQ feed a Scanner (scan_nfft points) and are kept in one device buffer. Then
    find_carriers (find_params: its thresholds) on the mean spectrum, probe_carriers on the kept IQ and channel_plan give the
    carriers; per mode one Ddc, one DemodBatch and its frame layer are built on the receiver's CUDA stream (a P-channel layer for
    600, 1200 and 10 500 bps with one Reassembler per carrier, the C-channel layer for 8400 bps), and the kept IQ is decoded
    first, so nothing sent during acquisition is lost. Burst carriers are not planned and no channel is ever retuned.

    Steady state, per block of block_seconds: each Ddc down-converts the block straight from its one device copy, the
    demodulators read the Ddc's output rows, the frame layers run, and once per whole second of input the layers' 1 s DCD tick
    runs (paced by signal time). The CRC-valid P-channel signal units go to their carrier's Reassembler.

    write / write_device / flush return the new events, a list of dicts. Every event has kind, carrier (index into carriers()),
    center_hz, mode and input_seconds: the input consumed at the end of the block that produced the event. input_seconds is
    block-granular: it says which block decoded the event, not at which sample the event was sent. Kinds:
      "acars":  the fields of Reassembler.pop_all, with its record kind as record_kind (0 message, 1 error) and the ACARS mode
                character as acars_mode;
      "su":     a CRC-valid P-channel signal unit (only with emit_sus=True): su (12 bytes), index (in its frame), frame;
      "cframe": a C-channel frame: sus (three 12-byte signal units), crc_ok (three flags), voice (300 bytes), frame.

    stream: a cudaStream_t as an int, or None for a new torch CUDA stream. IQ given to write_device must be ready in that stream's
    order. Use as a context manager, or call close()."""

    def __init__(self, input_rate, fmt, acquire_seconds=4.0, block_seconds=0.1, device=0, stream=None, scan_nfft=1 << 16,
                 emit_sus=False, **find_params):
        self.fmt = fmt
        self._f = _iq_format(fmt)
        self.interpolation, self.decimation = rate_ratio(input_rate)
        self.input_rate = float(input_rate)
        self._rate = int(self.input_rate)
        unknown = sorted(set(find_params) - set(FIND_PARAMS))
        if unknown:
            raise TypeError("Receiver: unknown find_carriers parameter(s) %s" % ", ".join(unknown))
        if not float(acquire_seconds) > 0:
            raise ValueError("Receiver: acquire_seconds must be positive, got %r" % (acquire_seconds,))
        if not 0 < float(block_seconds) <= 1.0:
            raise ValueError("Receiver: block_seconds must be in (0, 1], got %r" % (block_seconds,))
        self.block_n = int(round(float(block_seconds) * self.input_rate))
        if self.block_n * self.interpolation < self.decimation:
            raise ValueError("Receiver: a block of %r s is shorter than one %g Hz output sample of the down-converter"
                             % (block_seconds, self.input_rate * self.interpolation / self.decimation))
        self.acquire_n = max(1, int(round(float(acquire_seconds) * self.input_rate)))
        self.emit_sus, self.find_params, self.device = bool(emit_sus), dict(find_params), int(device)
        self._groups, self._carriers, self._unplanned, self._reasm = [], [], [], []
        self._scanner = self._acq = self._stage = None
        import torch
        self._torch = torch
        self._dev = torch.device("cuda", self.device)
        if stream is None:
            self._ts = torch.cuda.Stream(device=self._dev)
        else:
            self._ts = torch.cuda.ExternalStream(int(stream), device=self._dev)
        self.stream = self._ts.cuda_stream
        self._dtype = torch.uint8 if self._f == IQ_CU8 else torch.int16
        self._typestr = "|u1" if self._f == IQ_CU8 else "<i2"
        self._bytes = 2 if self._f == IQ_CU8 else 4                  # bytes per IQ sample
        with torch.cuda.stream(self._ts):
            self._acq = torch.empty(2 * self.acquire_n, dtype=self._dtype, device=self._dev)
            self._stage = torch.empty(2 * self.block_n, dtype=self._dtype, device=self._dev)
        self._scanner = Scanner(self.input_rate, scan_nfft, device=self.device)
        self._scanner.set_stream(self.stream)
        self._n_acq = 0                  # IQ samples kept so far
        self._pending = 0                # IQ samples of the next block waiting in the staging buffer
        self._n_in = 0                   # IQ samples decoded (whole blocks, and the last partial block after flush)
        self._ticks = self._blocks = 0
        self.acquired = False

    # ---------------------------------------------------------------------------------------------------------- input
    def write(self, iq):
        """iq: interleaved host I, Q (uint8 for cu8, int16 for cs16), any length. -> new events"""
        iq, _ = _host_iq(iq, self.fmt)
        if iq.size == 0:
            return []
        torch = self._torch
        with torch.cuda.stream(self._ts):                            # one upload, ordered before everything that reads it
            dev = torch.from_numpy(iq).to(self._dev)
            return self._consume(dev.data_ptr(), iq.size // 2)

    def write_device(self, ptr, n_iq):
        """The same from device memory: n_iq interleaved I, Q samples at ptr, ready in the receiver's stream order"""
        if int(n_iq) <= 0:
            return []
        with self._torch.cuda.stream(self._ts):
            return self._consume(int(ptr), int(n_iq))

    def flush(self):
        """Decodes what is still short of a block (at the end of a stream). A stream that ended during acquisition is planned from
        the IQ it had. -> new events"""
        ev = []
        with self._torch.cuda.stream(self._ts):
            if not self.acquired and self._n_acq:
                ev += self._finish_acquisition()
            if self._pending:
                n, self._pending = self._pending, 0
                ev += self._block(self._stage.data_ptr(), n)
        return ev

    def _copy(self, dst, dst_at, ptr, n):
        """n IQ samples from ptr to dst[dst_at:], on the receiver's stream"""
        src = self._torch.as_tensor(_Raw(ptr, 2 * n, self._typestr), device=self._dev)
        dst[2 * dst_at:2 * (dst_at + n)].copy_(src)

    def _consume(self, ptr, n):
        ev, a = [], 0
        if not self.acquired:
            a = min(n, self.acquire_n - self._n_acq)
            self._copy(self._acq, self._n_acq, ptr, a)
            self._scanner.write_device(self._acq.data_ptr() + self._n_acq * self._bytes, a, self.fmt)
            self._n_acq += a
            if self._n_acq < self.acquire_n:
                return ev
            ev += self._finish_acquisition()
        if a < n:
            ev += self._feed(ptr + a * self._bytes, n - a)
        return ev

    def _feed(self, ptr, n):
        """steady state: whole blocks straight from ptr, the pieces around them through the staging buffer"""
        ev, a = [], 0
        if self._pending:
            a = min(n, self.block_n - self._pending)
            self._copy(self._stage, self._pending, ptr, a)
            self._pending += a
            if self._pending < self.block_n:
                return ev
            self._pending = 0
            ev += self._block(self._stage.data_ptr(), self.block_n)
        while n - a >= self.block_n:
            ev += self._block(ptr + a * self._bytes, self.block_n)
            a += self.block_n
        if a < n:
            self._copy(self._stage, 0, ptr + a * self._bytes, n - a)
            self._pending = n - a
        return ev

    # ---------------------------------------------------------------------------------------------------- acquisition
    def _finish_acquisition(self):
        self.acquired = True
        mean, _, _ = self._scanner.read()
        self._scanner.close(); self._scanner = None
        found = find_carriers(mean, self.input_rate, **self.find_params)
        probed = probe_carriers(found, self.input_rate, (self._acq.data_ptr(), self._n_acq), self.fmt,
                                interpolation=self.interpolation, decimation=self.decimation, stream=self.stream,
                                device=self.device)
        plans, self._unplanned = channel_plan(probed, self.input_rate, self.decimation, self.interpolation)
        for mode in sorted(plans, key=lambda m: plans[m]["carriers"][0]["center_hz"]):
            g = self._new_group(mode, plans[mode], len(self._carriers))
            self._groups.append(g)
            for c in plans[mode]["carriers"]:
                self._carriers.append(dict(c, mode=mode))
                self._reasm.append(Reassembler() if mode in P_MODES else None)
        k = len(self._carriers)
        self._su_total, self._su_bad = np.zeros(k, dtype=np.int64), np.zeros(k, dtype=np.int64)
        self._messages, self._frames = np.zeros(k, dtype=np.int64), np.zeros(k, dtype=np.int64)
        acq, n, self._acq = self._acq, self._n_acq, None
        ev = self._feed(acq.data_ptr(), n)                            # the acquisition window, decoded like any other IQ
        del acq                                                        # freed in stream order: the blocks above come first
        return ev

    def _new_group(self, mode, plan, first):
        return _Group(mode, plan, first, self.device, self.stream)

    # ---------------------------------------------------------------------------------------------------------- blocks
    def _block(self, ptr, n):
        for g in self._groups:
            g.ddc.write_device(ptr, n, self.fmt)
            p, m, stride = g.ddc.output()
            if m:
                g.demod.write_device(p, m, stride)
                g.layer.process_batch(g.demod)
        self._n_in += n
        self._blocks += 1
        due = self._n_in // self._rate - self._ticks                 # JAERO's 1 s DCD timer, paced by signal time
        for _ in range(due):
            for g in self._groups:
                g.layer.tick(g.demod)
        self._ticks += due
        return self._read()

    def _read(self):
        ev, t = [], self._n_in / self.input_rate
        for g in self._groups:
            if g.mode in P_MODES:
                out, counts = g.layer.read_sus_raw(g.su_out, g.su_counts)
                for ch in np.flatnonzero(counts):
                    ev += self._units(g.first + int(ch), out[ch, :counts[ch]], t)
            else:
                for ch, (su, ok, voice, frame) in enumerate(g.layer.read_frames()):
                    ev += self._cframes(g.first + ch, su, ok, voice, frame, t)
        return ev

    # ---------------------------------------------------------------------------------------------------------- state
    def carriers(self):
        """the planned carriers, in the order of the events' carrier index: channel_plan's carrier dicts (mode, center_hz, snr_db,
        ...) plus dcd and ebno from the demodulators (empty before acquisition completes)"""
        out = []
        for g in self._groups:
            for ch, st in enumerate(g.demod.status()):
                out.append(dict(self._carriers[g.first + ch], index=g.first + ch, dcd=bool(st["dcd"]), ebno=st["ebno"]))
        return out

    def unplanned(self):
        """channel_plan's leftovers, each with the reason it was left: "unknown mode", "at DC" or "band edge" """
        out = []
        for c in self._unplanned:
            if c["mode"] not in ("msk600", "msk1200", "oqpsk8400", "oqpsk10500"):
                why = "unknown mode"
            elif c["flags"] & 1:
                why = "at DC"
            else:
                why = "band edge"
            out.append(dict(c, reason=why))
        return out

    def stats(self):
        """blocks and seconds decoded; per planned carrier the signal units read, their CRC failures, ACARS records, C-channel
        frames and the clipped samples of its down-converter channel"""
        per = []
        for g in self._groups:
            _, clipped = g.ddc.stats()
            for ch in range(g.n):
                c = g.first + ch
                per.append(dict(carrier=c, mode=g.mode, center_hz=self._carriers[c]["center_hz"], sus=int(self._su_total[c]),
                                crc_failures=int(self._su_bad[c]), messages=int(self._messages[c]), cframes=int(self._frames[c]),
                                ddc_clipped=int(clipped[ch])))
        return dict(blocks=self._blocks, seconds=self._n_in / self.input_rate, acquired=self.acquired,
                    acquire_seconds=self.acquire_n / self.input_rate, carriers=per)

    def close(self):
        for g in self._groups:
            g.close()
        self._groups = []
        for r in self._reasm:
            if r is not None:
                r.close()
        self._reasm = []
        if self._scanner is not None:
            self._scanner.close(); self._scanner = None
        self._acq = self._stage = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def jsonable(event):
    """An event with its bytes as text, for JSON: ACARS text, label and registration as latin-1 strings, signal units and voice
    as hex"""
    out = {}
    for k, v in event.items():
        if isinstance(v, bytes):
            v = v.decode("latin-1") if k in ("text", "label", "reg") else v.hex()
        elif isinstance(v, list):
            v = [x.hex() if isinstance(x, bytes) else x for x in v]
        elif isinstance(v, np.generic):
            v = v.item()
        out[k] = v
    return out
