"""Build the native-rate (44.1 kHz) fixtures and what the rate converter + demodulator chain decodes from them.

Needs the reference's recordings (/root/reference/samples) and the restated oracle (make -C oracle oracle). Writes
  tests/golden/oqpsk_10500_44k1_excerpt.npz        int16 @44.1 kHz, 0-12 s of 10.5k_sample.ogg (the window of oqpsk_10500)
  tests/golden/burst_oqpsk_10500_44k1_excerpt.npz  int16 @44.1 kHz, 0-8 s of 10.5k_burst_sample.mp3 (that of burst_oqpsk_10500)
  tests/golden/native_rate_manifest.json           source, rate, length and SHA-256 of each excerpt
  tests/golden/native_rate_outputs.json            the excerpts resampled to 48 kHz by the numpy reference of the rate converter
                                                    (tests/resample_reference.py) and decoded by the restated oracle: the
                                                    continuous excerpt's CRC-valid signal units, the burst excerpt's R/T packets
The decoding loops are those of the GPU tests: 4800-sample writes at 48 kHz (4410 at 44.1 kHz), DCD fed back to the demodulator
at every write and the frame layer's DCD updated once a second. The same loops run over the 48 kHz fixtures of the same windows,
and the tool reports whether both rates decode the same signal units and packets.
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from audio_decode import decode_mono  # noqa: E402
from make_fixtures import to_i16  # noqa: E402
import jaero_b200  # noqa: E402
import resample_reference as rr  # noqa: E402
from oracle import restated  # noqa: E402

REF = "/root/reference/samples"
GOLD = os.path.join(ROOT, "tests", "golden")
RATE = 44100
CHUNK = 4800                                     # 48 kHz samples per write; 4410 at 44.1 kHz
ITEMS = {
    "oqpsk_10500_44k1": ("10.5k_sample.ogg", 12.0, "oqpsk_10500"),
    "burst_oqpsk_10500_44k1": ("10.5k_burst_sample.mp3", 8.0, "burst_oqpsk_10500"),
}


def resample_48k(x):
    p = jaero_b200.resample_plan(RATE, 48000, 0.45 * RATE)
    pcm, _, clipped = rr.resample_reference(x[None, :], p["h"], p["L"], p["M"])
    return pcm[0], int(clipped[0])


def decode_sus(pcm, kw):
    """restated OQPSK demodulator -> P-channel, DCD fed back per write; CRC-valid signal units as hex strings"""
    od = restated.OracleDemod("oqpsk", **kw)
    op = restated.OraclePChannel(kw["fb"])
    for a in range(0, len(pcm), CHUNK):
        od.set_dcd(op.dcd); od.write(pcm[a:a + CHUNK]); op.process(od.take_soft())
        if (a + CHUNK) % 48000 < CHUNK:
            op.update_dcd()
    su, ok, _ = op.take_sus()
    od.close(); op.close()
    return [bytes(s).hex() for s, k in zip(su, ok) if k]


def decode_rt(pcm, kw):
    """restated burst OQPSK demodulator -> R/T layer, DCD updated once a second; packets as the golden files record them"""
    od = restated.OracleDemod("burst_oqpsk", **kw)
    ort = restated.OracleRTChannel(kw["fb"])
    for k, a in enumerate(range(0, len(pcm), CHUNK)):
        od.write(pcm[a:a + CHUNK]); ort.process(od.take_soft())
        if k % 10 == 9:
            ort.update_dcd()
    out = [dict(type=q["type"], nsus=q["nsus"], n_bytes=int(len(q["bytes"])), sha256=hashlib.sha256(q["bytes"].tobytes()).hexdigest())
           for q in ort.packets()]
    od.close(); ort.close()
    return out


def main():
    golden = json.load(open(os.path.join(GOLD, "expected_outputs.json")))
    manifest, outputs = {}, {}
    for name, (fn, secs, twin) in ITEMS.items():
        f, _ = decode_mono(os.path.join(REF, fn))           # both recordings are 44.1 kHz (tools/make_fixtures.py)
        x = np.ascontiguousarray(to_i16(f)[:int(secs * RATE)])
        np.savez_compressed(os.path.join(GOLD, name + "_excerpt.npz"), pcm=x)
        manifest[name] = {"source": fn, "rate": RATE, "window_s": [0.0, secs], "samples": int(len(x)),
                          "sha256": hashlib.sha256(x.tobytes()).hexdigest()}
        y, clipped = resample_48k(x)
        twin_pcm = np.load(os.path.join(GOLD, twin + "_excerpt.npz"))["pcm"]
        kw = dict(golden[twin]["kw"])
        entry = {"twin": twin, "kw": kw, "chunk_48k": CHUNK, "chunk_in": CHUNK * RATE // 48000, "resampled_samples": int(len(y)),
                 "resampled_sha256": hashlib.sha256(y.tobytes()).hexdigest(), "resampled_clipped": clipped}
        if twin == "oqpsk_10500":
            got, ref = decode_sus(y, kw), decode_sus(twin_pcm, kw)
            assert len(ref) == golden[twin]["n_su_crc_ok"], (len(ref), golden[twin]["n_su_crc_ok"])
            entry.update(n_su_crc_ok=len(got), su_crc_ok_sha256=hashlib.sha256(json.dumps(got).encode()).hexdigest())
            common = set(got) & set(ref)
            print("%s: %d CRC-valid SUs at 44.1 kHz, %d at 48 kHz, %d in common; same list: %s"
                  % (name, len(got), len(ref), len(common), got == ref))
        else:
            got, ref = decode_rt(y, kw), decode_rt(twin_pcm, kw)
            assert ref == golden[twin]["rt_packets"]
            entry.update(rt_packets=got)
            print("%s: %d R/T packets at 44.1 kHz, %d at 48 kHz; same packets: %s" % (name, len(got), len(ref), got == ref))
        outputs[name] = entry
    with open(os.path.join(GOLD, "native_rate_manifest.json"), "w") as fh:
        json.dump(manifest, fh, indent=1, sort_keys=True)
    with open(os.path.join(GOLD, "native_rate_outputs.json"), "w") as fh:
        json.dump(outputs, fh, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
