"""Decode every continuous carrier of a wideband SDR IQ recording or pipe into ACARS messages (jaero_b200.Receiver).

    python tools/receive.py --rate 2400000 --format cu8 [--acquire 4] [--block 0.1] [--sus] [--segment SECONDS] FILE|-

FILE is raw interleaved IQ (cu8: unsigned 8-bit as rtl_sdr writes it; cs16: signed 16-bit little-endian); `-` reads standard
input, e.g. `rtl_sdr -f 1545.0e6 -s 2.4e6 - | python tools/receive.py --rate 2400000 --format cu8 -`. One JSON object per event
goes to standard output as it is decoded (bytes as text: ACARS text, label and registration as latin-1, signal units and voice
as hex). At the end of the input the plan (the carriers decoded and the ones left unplanned, with the reason) and the
statistics go to standard error as JSON.

--segment SECONDS decodes a recording with jaero_b200.RecordingDecoder instead: each carrier is cut into segments of that many
seconds that are demodulated side by side, so events come out a chunk of segments at a time (at the latest at the end of the
input) rather than as the input arrives. The output has the same form.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rate", required=True, help="IQ sample rate, whole hertz")
    ap.add_argument("--format", required=True, help="cu8 or cs16")
    ap.add_argument("--acquire", type=float, default=4.0, help="seconds of IQ to find and identify the carriers in (default 4)")
    ap.add_argument("--block", type=float, default=0.1, help="seconds of IQ per decoding step (default 0.1)")
    ap.add_argument("--sus", action="store_true", help="also print every CRC-valid P-channel signal unit")
    ap.add_argument("--segment", type=float, default=None,
                    help="decode as parallel segments of this many whole seconds (RecordingDecoder); for recordings")
    ap.add_argument("--device", type=int, default=0, help="CUDA device (default 0)")
    ap.add_argument("input", help="raw IQ file, or - for standard input")
    a = ap.parse_args(argv)
    try:
        rate = float(a.rate)
    except ValueError:
        ap.error("--rate must be a number of hertz, got %r" % a.rate)
    if not (rate > 0 and rate == int(rate)):
        ap.error("--rate must be a positive whole number of hertz, got %r" % a.rate)
    if a.format not in ("cu8", "cs16"):
        ap.error("--format must be cu8 or cs16, got %r" % a.format)
    from jaero_b200 import rate_ratio
    try:
        rate_ratio(rate)
    except ValueError as e:
        ap.error(str(e))
    if not a.acquire > 0:
        ap.error("--acquire must be positive")
    if not 0 < a.block <= 1.0:
        ap.error("--block must be in (0, 1] seconds")
    if a.block * 48000.0 < 1.0:
        ap.error("--block is shorter than one 48 kHz sample")
    if a.segment is not None:
        from jaero_b200.recording import layout
        try:
            layout(rate, a.block, a.segment)
        except ValueError as e:
            ap.error("--segment: %s" % str(e).replace("RecordingDecoder: ", ""))
    a.rate = rate
    return a


def main(argv=None):
    import numpy as np
    from jaero_b200.receiver import Receiver, jsonable
    from jaero_b200.recording import RecordingDecoder
    a = parse_args(argv)
    dtype = np.uint8 if a.format == "cu8" else np.dtype("<i2")
    item = 2 * np.dtype(dtype).itemsize                          # bytes per IQ sample
    chunk = max(1, int(a.rate * a.block)) * item
    src = sys.stdin.buffer if a.input == "-" else open(a.input, "rb")
    out = sys.stdout

    def emit(events):
        for e in events:
            out.write(json.dumps(jsonable(e)) + "\n")
        if events:
            out.flush()

    rest = bytearray()
    kw = dict(acquire_seconds=a.acquire, block_seconds=a.block, device=a.device, emit_sus=a.sus)
    if a.segment is None:
        rx = Receiver(a.rate, a.format, **kw)
    else:
        rx = RecordingDecoder(a.rate, a.format, segment_seconds=a.segment, **kw)
    with rx:
        while True:
            buf = src.read(chunk)
            if not buf:
                break
            buf = rest + buf                                         # writable: torch uploads it without a warning
            n = len(buf) - len(buf) % item                           # whole IQ samples; a pipe may split one
            rest = buf[n:]
            if n:
                emit(rx.write(np.frombuffer(buf, dtype=dtype, count=n // np.dtype(dtype).itemsize)))
        emit(rx.flush())
        report = dict(carriers=[jsonable(c) for c in rx.carriers()],
                      unplanned=[jsonable(c) for c in rx.unplanned()], stats=rx.stats())
        sys.stderr.write(json.dumps(report, indent=1) + "\n")
    if src is not sys.stdin.buffer:
        src.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
