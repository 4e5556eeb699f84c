"""Decode audio recordings of R/T burst carriers into R/T packets and ACARS messages (jaero_b200.BurstAudioDecoder).

    python tools/decode_bursts.py [--mode M] [--channel N] [--rate HZ] [--segment S] [--identify S] [--block S] [--packets]
                                  [--device D] FILE...

Each FILE holds one burst carrier, SSB-demodulated by the radio software: a WAV file of 16-bit PCM (mono, or the --channel of
a stereo file) at its own rate, or raw signed 16-bit little-endian mono PCM, whose rate --rate gives (decode_audio.py's
reader). Files of the same sample rate are decoded together by one BurstAudioDecoder, each as parallel segments of --segment
seconds. --mode gives every file's mode (burst_msk600, burst_msk1200, burst_oqpsk10500); without it each file's burst rate is
identified from its first --identify seconds. One JSON object per event goes to standard output, with the file's name added
as "file" (ACARS text, label and registration as latin-1, packet bytes as hex). The plan and the statistics go to standard
error as JSON, one report per sample rate.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from decode_audio import AudioFileError, read_audio  # noqa: E402

FLAGS = (("sample_rate", "--rate"), ("segment_seconds", "--segment"), ("block_seconds", "--block"),
         ("identify_seconds", "--identify"), ("modes", "--mode"))


def _flag(msg):
    for name, flag in FLAGS:
        if name in msg:
            return flag
    return None


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--mode", default=None, help="every file's mode: burst_msk600, burst_msk1200 or burst_oqpsk10500 "
                                                 "(default: identify)")
    ap.add_argument("--channel", type=int, default=0, help="channel of a stereo WAV to decode (default 0)")
    ap.add_argument("--rate", default=None, help="sample rate of raw files, whole hertz")
    ap.add_argument("--segment", type=float, default=10, help="seconds each demodulator channel owns (default 10)")
    ap.add_argument("--identify", type=float, default=60.0, help="seconds to identify the burst rate from (default 60)")
    ap.add_argument("--block", type=float, default=0.1, help="seconds of audio per decoding step (default 0.1)")
    ap.add_argument("--packets", action="store_true", help="also print every R/T packet")
    ap.add_argument("--device", type=int, default=0, help="CUDA device (default 0)")
    ap.add_argument("files", nargs="+", metavar="FILE", help="WAV or raw 16-bit PCM file")
    a = ap.parse_args(argv)
    rate = None
    if a.rate is not None:
        try:
            rate = float(a.rate)
        except ValueError:
            ap.error("--rate must be a number of hertz, got %r" % a.rate)
        if not (rate > 0 and rate == int(rate)):
            ap.error("--rate must be a positive whole number of hertz, got %r" % a.rate)
        rate = int(rate)
    if a.channel < 0:
        ap.error("--channel must be 0 or more, got %d" % a.channel)
    a.audio = []
    for path in a.files:
        try:
            a.audio.append((path,) + read_audio(path, rate, a.channel))
        except AudioFileError as e:
            ap.error(str(e))
        except OSError as e:
            ap.error("%s: %s" % (path, e.strerror or e))
    from jaero_b200 import BurstAudioDecoder
    a.decoders = {}
    for fs in sorted({fs for _, _, fs in a.audio}):
        try:
            a.decoders[fs] = BurstAudioDecoder(fs, **_settings(a))
        except ValueError as e:
            msg = str(e).replace("BurstAudioDecoder: ", "")
            flag = _flag(msg)
            ap.error("%s%s" % ("" if flag is None else flag + ": ", msg))
    return a


def _settings(a):
    return dict(modes=a.mode, identify_seconds=a.identify, block_seconds=a.block, segment_seconds=a.segment,
                emit_packets=a.packets, device=a.device)


def main(argv=None):
    from jaero_b200.receiver import jsonable
    a = parse_args(argv)
    out = sys.stdout
    for fs, dec in a.decoders.items():
        files = [(path, pcm) for path, pcm, r in a.audio if r == fs]
        with dec:
            for e in dec.decode([pcm for _, pcm in files]):
                out.write(json.dumps(dict(jsonable(e), file=files[e["carrier"]][0])) + "\n")
            out.flush()
            name = lambda d: dict(jsonable(d), file=files[d["index"]][0])
            report = dict(sample_rate=fs, files=[p for p, _ in files], carriers=[name(c) for c in dec.carriers()],
                          unplanned=[name(c) for c in dec.unplanned()], stats=dec.stats())
            sys.stderr.write(json.dumps(report, indent=1) + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
