"""What decoding an audio recording as parallel segments (jaero_b200.AudioDecoder) gains over the straight chain, on one GPU.

Per recording (--minutes of each continuous mode at 48 kHz, and of 10.5 kbps at 44.1 kHz). The P-channel recordings are
seeded synthetic audio: one minute of frames carrying known ACARS messages (synth.pchannel_bits_from_sus), circular, at
Eb/N0 12 dB, repeated with fresh noise each minute. The 8400 bps recording is the committed 8 s excerpt of a real C-channel
recording (tests/golden/oqpsk_8400_excerpt.npz), repeated:
- AudioDecoder: decode() of the host array with 10 s segments and the default leads, the mode and centre given;
- the straight chain: one DemodBatch channel (the same settings) and its frame layer, with a Resampler in front at 44.1 kHz,
  fed the same recording from device memory in 0.1 s blocks, ticked every whole second, records read every block and the
  CRC-valid units pushed to a Reassembler.
Each path is timed by the wall clock around the whole run (both read results back, so the run ends in a device synchronise).
Both are then run again over the first --profile seconds of the recording under torch.profiler, in runs of their own: the
device-busy time (the union of the kernel and copy intervals) against the wall time of the same run. Printed per recording:
wall seconds, multiple of real time, the busy share, AudioDecoder's batch width and peak PCM buffer, and whether both paths
gave the same ACARS messages and CRC-valid units. The card's name, power limit and clocks are read in the same run.

usage: python tools/audio_bench.py [--minutes 30] [--profile 120] [--only NAME,...] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))     # reasm_synth: ACARS messages as signal units

from receive_bench import card  # noqa: E402
from recording_bench import busy_seconds  # noqa: E402

# (name, mode, bit rate, sample rate)
RECORDINGS = [("10.5k", "oqpsk10500", 10500, 48000), ("8400", "oqpsk8400", 8400, 48000), ("1200", "msk1200", 1200, 48000),
              ("600", "msk600", 600, 48000), ("10.5k@44.1", "oqpsk10500", 10500, 44100)]
EBN0_DB = 12.0


def message_minute(fb, seed):
    """one minute of a P-channel carrier's circular 48 kHz envelope, its frames carrying ACARS messages back to back"""
    import reasm_synth
    from jaero_b200 import synth
    fp = synth.frame_params(fb)
    k = fp["blocks"] * 64 * fp["cols"] // 2 // 96                  # signal units per frame
    n = 60 * fb // fp["frame_bits"] * k                             # a whole number of frames at every P-channel rate
    rng = np.random.default_rng(seed)
    units = []
    while True:
        i = len(units)
        text = "B%d %s" % (i, "".join("ABCDEFGHIJ"[x] for x in rng.integers(0, 10, int(rng.integers(2, 40)))))
        sus = reasm_synth.isu_to_sus(0x400000 + i, 0x90, i & 15, 3,
                                     reasm_synth.acars_userdata("B%05d" % i, "H1", ord("A") + i % 26, text))
        if len(units) + len(sus) > n:
            break
        units += sus
    units += [synth.FILL_SU] * (n - len(units))
    msk = fb != 10500
    bits = synth.pchannel_bits_from_sus(fb, units, loop=True, even_parity=msk)
    return synth.msk_envelope(bits, fb) if msk else synth.oqpsk_envelope(bits, fb)


def recording(jb, mode, fb, rate, minutes, seed):
    """minutes of one carrier at rate, at the mode's CHANNEL_SETTINGS audio centre (8000 Hz, the centre its fixture is decoded
    at, for the 8400 bps excerpt). P-channel: message_minute (a whole number of carrier cycles per minute, so the minutes join
    without a phase step) with fresh noise each minute"""
    from jaero_b200 import synth
    if mode == "oqpsk8400":
        x = np.load(os.path.join(os.path.dirname(HERE), "tests", "golden", "oqpsk_8400_excerpt.npz"))["pcm"]
        n = int(minutes * 60 * 48000)
        return np.tile(x, -(-n // len(x)))[:n], 8000.0
    env = message_minute(fb, seed)
    assert len(env) == 60 * 48000
    fc = jb.CHANNEL_SETTINGS[mode]["audio_hz"]
    out = []
    for k in range(int(minutes)):
        pcm = synth.to_passband_int16(env, fc, ebn0_db=EBN0_DB, fb=float(fb), rng=np.random.default_rng(1000 * seed + k))
        if rate != 48000:
            from scipy.signal import resample_poly
            pcm = np.clip(np.round(resample_poly(pcm.astype(np.float64), rate // 300, 160)), -32768, 32767).astype(np.int16)
        out.append(pcm)
    return np.concatenate(out), fc


def decoder_run(jb, torch, pcm, rate, mode, fc):
    t0 = time.perf_counter()
    with jb.AudioDecoder(rate, modes=mode, centers_hz=fc, emit_sus=True) as dec:
        ev = dec.decode([pcm])
        st = dec.stats()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    g = st["groups"][0]
    return wall, _results(ev), dict(batch_width=g["batch_width"], pcm_bytes_peak=g["pcm_bytes_peak"], chunks=g["chunks"],
                                    late_locks=st["carriers"][0]["late_locks"],
                                    unlocked_segments=st["carriers"][0]["unlocked_segments"])


def _results(ev):
    acars = [(e["record_kind"], e["aesid"], e["reg"], e["label"], e["text"]) for e in ev if e["kind"] == "acars"]
    units = [e["su"] for e in ev if e["kind"] == "su"]
    units += [s for e in ev if e["kind"] == "cframe" for s, o in zip(e["sus"], e["crc_ok"]) if o]
    return acars, units


def chain_run(jb, torch, pcm, rate, mode, fc):
    """the straight chain, from device memory; the upload is not timed"""
    s = jb.CHANNEL_SETTINGS[mode]
    stream = torch.cuda.Stream()
    n_blk = int(round(0.1 * rate))
    n = -(-len(pcm) // n_blk) * n_blk
    x = np.zeros(n, dtype=np.int16)
    x[:len(pcm)] = pcm
    dev = torch.from_numpy(x).cuda()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rs = None
    if rate != 48000:
        rs = jb.Resampler(rate, 1)
        rs.set_stream(stream.cuda_stream)
    b = jb.DemodBatch(s["kind"], 1, fb=s["fb"], freq_center=fc, lockingbw=s["lockingbw"], afc=True)
    b.set_stream(stream.cuda_stream)
    p = mode != "oqpsk8400"
    layer = jb.PChannelBatch(1, s["fb"]) if p else jb.CChannelBatch(1)
    reasm = jb.Reassembler() if p else None
    out = np.empty((1, layer.su_cap if p else 8, 16 if p else jb.CChannelBatch.RECORD), dtype=np.uint8)
    counts = np.zeros(1, dtype=np.int32)
    acars, units = [], []
    for j in range(n // n_blk):
        if rs is None:
            b.write_device(dev.data_ptr() + 2 * j * n_blk, n_blk, n_blk)
        else:
            rs.write_device(dev.data_ptr() + 2 * j * n_blk, n_blk, n_blk)
            ptr, m, stride = rs.output()
            b.write_device(ptr, m, stride)
        layer.process_batch(b)
        if (j + 1) % 10 == 0:
            layer.tick(b)
        if p:
            layer.read_sus_raw(out, counts)
            for r in out[0, :counts[0]]:
                if r[12]:
                    units.append(r[:12].tobytes())
                    reasm.push_su(r[:12].tobytes())
            acars += [(e["kind"], e["aesid"], e["reg"], e["label"], e["text"]) for e in reasm.pop_all()]
        else:
            layer.read_frames_raw(out, counts)
            for r in out[0, :counts[0]]:
                units += [r[16 * k:16 * k + 12].tobytes() for k in range(3) if r[16 * k + 12]]
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    for o in (rs, b, layer, reasm):
        if o is not None:
            o.close()
    return wall, (acars, units), {}


def profiled(torch, fn, *args):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        wall, _, _ = fn(*args)
    busy, n = busy_seconds(prof)
    return dict(profiled_wall_s=wall, device_busy_s=busy, busy_share=busy / wall, device_intervals=n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=int, default=30, help="minutes per recording (default 30)")
    ap.add_argument("--profile", type=float, default=120.0, help="signal seconds per profiled run (0: none)")
    ap.add_argument("--only", default=None, help="comma-separated recording names (%s)" % ", ".join(r[0] for r in RECORDINGS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import jaero_b200 as jb
    if not torch.cuda.is_available():
        sys.exit("audio_bench: no CUDA device")
    lines = []

    def emit(r):
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)

    emit(dict(card=card()))
    want = None if args.only is None else set(args.only.split(","))
    rows = []
    for i, (name, mode, fb, rate) in enumerate(RECORDINGS):
        if want is not None and name not in want:
            continue
        pcm, fc = recording(jb, mode, fb, rate, args.minutes, seed=11 + i)
        seconds = len(pcm) / rate
        dw, dres, dinfo = decoder_run(jb, torch, pcm, rate, mode, fc)
        cw, cres, _ = chain_run(jb, torch, pcm, rate, mode, fc)
        r = dict(recording=name, mode=mode, sample_rate=rate, signal_s=seconds,
                 decoder=dict(wall_s=dw, x_realtime=seconds / dw, **dinfo),
                 chain=dict(wall_s=cw, x_realtime=seconds / cw),
                 speedup=cw / dw, same_acars=dres[0] == cres[0], same_units=dres[1] == cres[1],
                 acars=len(dres[0]), chain_acars=len(cres[0]), units=len(dres[1]), chain_units=len(cres[1]))
        if args.profile > 0:
            head = pcm[:int(args.profile * rate)]
            r["decoder"]["profile"] = dict(signal_s=len(head) / rate, **profiled(torch, decoder_run, jb, torch, head, rate, mode, fc))
            r["chain"]["profile"] = dict(signal_s=len(head) / rate, **profiled(torch, chain_run, jb, torch, head, rate, mode, fc))
        emit(r)
        rows.append(r)
    emit(dict(card_after=card()))
    print("\n| Recording | Path | Wall s | x real time | Device busy (profiled) | Batch width | PCM peak | Same ACARS / units |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        for path in ("decoder", "chain"):
            d = r[path]
            prof = d.get("profile")
            busy = "%.2f s of %.2f (%.0f %%)" % (prof["device_busy_s"], prof["profiled_wall_s"], 100 * prof["busy_share"]) \
                if prof else "-"
            print("| %s, %d min | %s | %.2f | %.1f | %s | %s | %s | %s |" % (
                r["recording"], round(r["signal_s"] / 60), "AudioDecoder" if path == "decoder" else "straight chain", d["wall_s"],
                d["x_realtime"], busy, d.get("batch_width", 1), "%.0f MB" % (d["pcm_bytes_peak"] / 1e6) if path == "decoder" else "-",
                "%s / %s (%d, %d)" % (r["same_acars"], r["same_units"], r["acars"], r["units"]) if path == "decoder" else ""))
    if args.out:
        with open(args.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
