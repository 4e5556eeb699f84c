"""Decode audio recordings of JAERO carriers into ACARS messages (jaero_b200.AudioDecoder).

    python tools/decode_audio.py [--mode M] [--center HZ] [--channel N] [--rate HZ] [--segment S] [--identify S] [--block S]
                                 [--sus] [--device D] FILE...

Each FILE holds one carrier, SSB-demodulated by the radio software:
- a WAV file of 16-bit PCM, mono or stereo (--channel picks the channel, default 0), at its own sample rate;
- or raw signed 16-bit little-endian mono PCM, whose rate --rate gives.
Other WAV encodings (8-bit, 24-bit, float, compressed) are refused with a message naming what the file has.

Files of the same sample rate are decoded together by one AudioDecoder, each as parallel segments of --segment seconds. --mode
and --center give every file's mode (msk600, msk1200, oqpsk10500, oqpsk8400) and carrier frequency in Hz; without them each
file's mode and carrier are identified from its first --identify seconds. One JSON object per event goes to standard output,
with the file's name added as "file" (bytes as text: ACARS text, label and registration as latin-1, signal units and voice as
hex). The plan (the files decoded and those left undecoded, with the reason) and the statistics go to standard error as JSON,
one report per sample rate.
"""
import argparse
import json
import os
import sys
import wave

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FLAGS = (("sample_rate", "--rate"), ("segment_seconds", "--segment"), ("lead_seconds", "--segment"), ("block_seconds", "--block"),
         ("identify_seconds", "--identify"), ("modes", "--mode"), ("centers_hz", "--center"), ("max_channels", "--segment"))


class AudioFileError(ValueError):
    """a file this tool cannot read, with the reason"""


def read_audio(path, rate=None, channel=0):
    """-> (1-D int16 PCM, sample rate). A file that starts with a RIFF header is read as WAV (16-bit PCM, mono, or the given
    channel of a multi-channel file); any other file as raw signed 16-bit little-endian mono at `rate`, through np.memmap."""
    import numpy as np
    with open(path, "rb") as fh:
        magic = fh.read(4)
    if magic == b"RIFF":
        try:
            w = wave.open(path, "rb")
        except wave.Error as e:
            raise AudioFileError("%s: the WAV's encoding is not PCM (%s); only 16-bit PCM WAV is read" % (path, e)) from None
        with w:
            width, nch, fs, n = w.getsampwidth(), w.getnchannels(), w.getframerate(), w.getnframes()
            if width != 2:
                raise AudioFileError("%s: the WAV has %d-bit samples; only 16-bit PCM WAV is read" % (path, 8 * width))
            if not 0 <= channel < nch:
                raise AudioFileError("%s: the WAV has %d channel(s); --channel %d does not exist" % (path, nch, channel))
            data = np.frombuffer(w.readframes(n), dtype="<i2")
        pcm = data.reshape(-1, nch)[:, channel]
        return np.ascontiguousarray(pcm, dtype=np.int16), fs
    if rate is None:
        raise AudioFileError("%s is not a WAV file: raw 16-bit PCM needs --rate" % path)
    if os.path.getsize(path) < 2:
        raise AudioFileError("%s: no samples" % path)
    pcm = np.memmap(path, dtype="<i2", mode="r", shape=(os.path.getsize(path) // 2,))
    return pcm.view(np.int16), rate


def _flag(msg):
    for name, flag in FLAGS:
        if name in msg:
            return flag
    return None


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--mode", default=None, help="every file's mode: msk600, msk1200, oqpsk10500 or oqpsk8400 (default: identify)")
    ap.add_argument("--center", type=float, default=None, help="every file's carrier frequency, Hz (default: identify)")
    ap.add_argument("--channel", type=int, default=0, help="channel of a stereo WAV to decode (default 0)")
    ap.add_argument("--rate", default=None, help="sample rate of raw files, whole hertz")
    ap.add_argument("--segment", type=float, default=10, help="seconds each demodulator channel owns (default 10)")
    ap.add_argument("--identify", type=float, default=4.0, help="seconds to identify the mode and carrier from (default 4)")
    ap.add_argument("--block", type=float, default=0.1, help="seconds of audio per decoding step (default 0.1)")
    ap.add_argument("--sus", action="store_true", help="also print every CRC-valid P-channel signal unit")
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
    from jaero_b200 import AudioDecoder
    a.decoders = {}
    for fs in sorted({fs for _, _, fs in a.audio}):
        try:
            a.decoders[fs] = AudioDecoder(fs, **_settings(a))
        except ValueError as e:
            msg = str(e).replace("AudioDecoder: ", "")
            flag = _flag(msg)
            ap.error("%s%s" % ("" if flag is None else flag + ": ", msg))
    return a


def _settings(a):
    return dict(modes=a.mode, centers_hz=a.center, identify_seconds=a.identify, block_seconds=a.block, segment_seconds=a.segment,
                emit_sus=a.sus, device=a.device)


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
