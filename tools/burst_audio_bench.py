"""What decoding a burst recording as parallel segments (jaero_b200.BurstAudioDecoder) gains over the straight chain, on one GPU.

Per recording (--minutes of each burst mode at 48 kHz, and of 10.5 kbps at 44.1 kHz): the committed excerpt of a real burst
recording (tests/golden/burst_*_excerpt.npz; at 600 bps the 1200 bps excerpt time-stretched 2x) tiled between seeded gaps of
noise at the excerpt's quietest level, 0.25 to 3 s long:
- BurstAudioDecoder: decode() of the host array with 10 s segments and the default leads, the mode given;
- the straight chain: one burst demodulator channel with the batch's defaults and its R/T layer, with a Resampler in front at
  44.1 kHz, fed the same recording from device memory in 0.1 s blocks, ticked every whole second, packets read every block
  and pushed to a Reassembler.
Each path is timed by the wall clock around the whole run. Both are then run again over the first --profile seconds under
torch.profiler, in runs of their own: the device-busy time (the union of the kernel and copy intervals) against the wall time
of the same run. Printed per recording: wall seconds, multiple of real time, the busy share, the decoder's batch width and
peak PCM buffer, and whether both paths gave the same packets (with their emission times) and ACARS records; where the packet
lists differ, the first difference. With --out, every result line and both paths' packet lists go to FILE as JSON lines.
The card's name, power limit and clocks are read in the same run.

usage: python tools/burst_audio_bench.py [--minutes 30] [--profile 120] [--only NAME,...] [--out FILE]
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

from receive_bench import card  # noqa: E402
from recording_bench import busy_seconds  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
# (name, mode, excerpt, sample rate)
RECORDINGS = [("10.5k", "burst_oqpsk10500", "burst_oqpsk_10500", 48000), ("1200", "burst_msk1200", "burst_msk_1200_a", 48000),
              ("600", "burst_msk600", "burst_msk_1200_a", 48000),
              ("10.5k@44.1", "burst_oqpsk10500", "burst_oqpsk_10500_44k1", 44100)]
FB = {"burst_msk600": 600, "burst_msk1200": 1200, "burst_oqpsk10500": 10500}


def recording(mode, excerpt, rate, minutes, seed):
    x = np.load(os.path.join(GOLD, excerpt + "_excerpt.npz"))["pcm"]
    if mode == "burst_msk600":
        from scipy.signal import resample_poly
        x = np.clip(np.round(resample_poly(x.astype(np.float64), 2, 1)), -32768, 32767).astype(np.int16)
    n_blk = rate // 10
    sigma = min(np.std(x[a:a + n_blk].astype(np.float64)) for a in range(0, len(x) - n_blk, n_blk))
    rng = np.random.default_rng(seed)
    out, n = [], 0
    while n < minutes * 60 * rate:
        gap = np.clip(np.round(rng.normal(0, sigma, int(rng.integers(rate // 4, 3 * rate)))), -32768, 32767).astype(np.int16)
        out += [gap, x]
        n += len(gap) + len(x)
    return np.concatenate(out)[:int(minutes * 60 * rate)]


def decoder_run(jb, torch, pcm, rate, mode):
    t0 = time.perf_counter()
    with jb.BurstAudioDecoder(rate, modes=mode, emit_packets=True) as dec:
        ev = dec.decode([pcm])
        st = dec.stats()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    g = st["groups"][0]
    packets = [(e["type"], e["nsus"], e["bytes"], e["input_seconds"]) for e in ev if e["kind"] == "rtpacket"]
    acars = [(e["record_kind"], e["aesid"], e["reg"], e["label"], e["text"]) for e in ev if e["kind"] == "acars"]
    return wall, (packets, acars), dict(batch_width=g["batch_width"], pcm_bytes_peak=g["pcm_bytes_peak"], chunks=g["chunks"],
                                        boundary_matches=st["carriers"][0]["boundary_matches"])


def chain_run(jb, torch, pcm, rate, mode):
    """the straight chain, from device memory; the upload is not timed"""
    n_blk = rate // 10
    n = -(-len(pcm) // n_blk) * n_blk
    x = np.zeros(n, dtype=np.int16)
    x[:len(pcm)] = pcm
    dev = torch.from_numpy(x).cuda()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rs = jb.Resampler(rate, 1) if rate != 48000 else None
    b = (jb.BurstOqpskBatch if mode == "burst_oqpsk10500" else jb.BurstMskBatch)(1, fb=float(FB[mode]))
    rt = jb.RTChannelBatch(1, FB[mode])
    reasm = jb.Reassembler()
    out = np.empty((1, 8, jb.RTChannelBatch.RECORD), dtype=np.uint8)
    counts = np.zeros(1, dtype=np.int32)
    packets, acars = [], []
    for j in range(n // n_blk):
        if rs is None:
            ptr, m = dev.data_ptr() + 2 * j * n_blk, n_blk
        else:
            rs.write_device(dev.data_ptr() + 2 * j * n_blk, n_blk, n_blk)
            ptr, m, _ = rs.output()
            rs.read_pcm()                                         # the burst batch runs on its own stream
        b.write_device(ptr, m, m)
        rt.process_burst(b)
        if (j + 1) % 10 == 0:
            rt.tick()
        rt.read_packets_raw(out, counts)
        for r in out[0, :counts[0]]:
            hdr = r[:16].view(np.int32)
            info = r[16:16 + int(hdr[2])].tobytes()
            packets.append(("R" if hdr[0] == 1 else "T", int(hdr[1]), info, min((j + 1) * n_blk, len(pcm)) / rate))
            if hdr[0] == 1:
                reasm.push_r(info, downlink=True)
            else:
                reasm.push_t_packet(info, int(hdr[1]))
            acars += [(e["kind"], e["aesid"], e["reg"], e["label"], e["text"]) for e in reasm.pop_all()]
        if (j + 1) % 3000 == 0:                                   # progress of a long run: every 5 minutes of signal
            print("chain: %d s of %d s" % ((j + 1) // 10, n // n_blk // 10), file=sys.stderr, flush=True)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    for o in (rs, b, rt, reasm):
        if o is not None:
            o.close()
    return wall, (packets, acars), {}


def first_difference(got, want):
    """None when the packet lists (type, nsus, bytes, emission second) are equal, else the first index where they differ
    and each list's packets from one before it to one after, bytes as hex"""
    if got == want:
        return None
    i = next((k for k in range(min(len(got), len(want))) if got[k] != want[k]), min(len(got), len(want)))
    show = lambda ps: [(k, n, b.hex(), t) for k, n, b, t in ps[max(0, i - 1):i + 2]]
    return dict(index=i, decoder=show(got), chain=show(want))


def profiled(torch, fn, *args):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        wall, _, _ = fn(*args)
    busy, n = busy_seconds(prof)
    return dict(profiled_wall_s=wall, device_busy_s=busy, busy_share=busy / wall, device_intervals=n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, default=30, help="minutes per recording (default 30)")
    ap.add_argument("--profile", type=float, default=120.0, help="signal seconds per profiled run (0: none)")
    ap.add_argument("--only", default=None, help="comma-separated recording names (%s)" % ", ".join(r[0] for r in RECORDINGS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import jaero_b200 as jb
    if not torch.cuda.is_available():
        sys.exit("burst_audio_bench: no CUDA device")
    lines = []

    def emit(r):
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)

    emit(dict(card=card()))
    want = None if args.only is None else set(args.only.split(","))
    rows = []
    for i, (name, mode, excerpt, rate) in enumerate(RECORDINGS):
        if want is not None and name not in want:
            continue
        pcm = recording(mode, excerpt, rate, args.minutes, seed=21 + i)
        seconds = len(pcm) / rate
        dw, dres, dinfo = decoder_run(jb, torch, pcm, rate, mode)
        cw, cres, _ = chain_run(jb, torch, pcm, rate, mode)
        r = dict(recording=name, mode=mode, sample_rate=rate, signal_s=seconds,
                 decoder=dict(wall_s=dw, x_realtime=seconds / dw, **dinfo),
                 chain=dict(wall_s=cw, x_realtime=seconds / cw),
                 speedup=cw / dw, same_packets=dres[0] == cres[0], same_acars=dres[1] == cres[1],
                 first_difference=first_difference(dres[0], cres[0]),
                 packets=len(dres[0]), chain_packets=len(cres[0]), acars=len(dres[1]), chain_acars=len(cres[1]))
        if args.profile > 0:
            head = pcm[:int(args.profile * rate)]
            r["decoder"]["profile"] = dict(signal_s=len(head) / rate, **profiled(torch, decoder_run, jb, torch, head, rate, mode))
            r["chain"]["profile"] = dict(signal_s=len(head) / rate, **profiled(torch, chain_run, jb, torch, head, rate, mode))
        emit(r)
        rows.append(r)
        if args.out:
            for path, res in (("decoder", dres), ("chain", cres)):
                lines.append(json.dumps(dict(recording=name, path=path, packets=[(k, n, b.hex(), t) for k, n, b, t in res[0]])))
    emit(dict(card_after=card()))
    print("\n| Recording | Path | Wall s | x real time | Device busy (profiled) | Batch width | PCM peak | Same packets / ACARS |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        for path in ("decoder", "chain"):
            d = r[path]
            prof = d.get("profile")
            busy = "%.2f s of %.2f (%.0f %%)" % (prof["device_busy_s"], prof["profiled_wall_s"], 100 * prof["busy_share"]) \
                if prof else "-"
            print("| %s, %d min | %s | %.2f | %.1f | %s | %s | %s | %s |" % (
                r["recording"], round(r["signal_s"] / 60), "BurstAudioDecoder" if path == "decoder" else "straight chain",
                d["wall_s"], d["x_realtime"], busy, d.get("batch_width", 1),
                "%.0f MB" % (d["pcm_bytes_peak"] / 1e6) if path == "decoder" else "-",
                "%s / %s (%d, %d)" % (r["same_packets"], r["same_acars"], r["packets"], r["acars"]) if path == "decoder" else ""))
    if args.out:
        with open(args.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
