"""What decoding a recording as parallel segments (jaero_b200.RecordingDecoder) gains over Receiver, on one GPU.

1. widths: per continuous mode, a DemodBatch and its frame layer at 16, 256, 1024 and 4096 channels, fed 0.1 s writes of a
   synthetic 48 kHz signal from the device (process_batch per write, tick once per second, records read every write, as
   RecordingDecoder runs them): seconds of GPU time per second of signal. If a batch's time does not grow with its width,
   the width is free throughput.
2. end to end: Receiver and RecordingDecoder, alternated, on tools/receive_bench.py's circular bands (2.4 MS/s cu8 with 16
   carriers, 9.6 MS/s cs16 with 256), --seconds of signal fed from device memory one block per write_device call from the
   start of the stream (acquisition included), then flush. Per path: x real time from the wall clock (the run ends in a
   device synchronise), the CPU time of the host thread over the same window, the CUDA-event time, signal units decoded, and
   for RecordingDecoder the segments, chunks, batch widths and PCM buffer size.
3. device time (--profile S): each path again over S seconds of signal under torch.profiler (CUDA activity only), in runs of
   their own: the time the device was busy (the union of the kernel and copy intervals) against the wall time of the same
   run. The profiler slows the host, so these runs give the busy share, not the rate.
The card's name, power limit and clocks are read in the same run. One JSON line per measurement.

usage: python tools/recording_bench.py [--seconds 240] [--segment 10] [--widths 16,256,1024,4096] [--width-seconds 5]
                                       [--sizes 0,1] [--skip-widths] [--skip-e2e] [--profile S] [--out FILE]
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

from receive_bench import SIZES, band, card, envelope  # noqa: E402

MODES = [("oqpsk10500", 10500), ("oqpsk8400", 8400), ("msk1200", 1200), ("msk600", 600)]


def width_run(torch, jb, mode, fb, width, seconds):
    from jaero_b200 import synth
    s = jb.CHANNEL_SETTINGS[mode]
    env = envelope(mode, fb, 11)                                 # 2 s, circular
    pcm = synth.to_passband_int16(np.tile(env, 2), s["audio_hz"], ebn0_db=12.0, fb=fb, rng=np.random.default_rng(3))
    period = len(env)
    stream = torch.cuda.Stream()
    x = torch.from_numpy(pcm).cuda().expand(width, -1).contiguous()
    torch.cuda.synchronize()
    b = jb.DemodBatch(s["kind"], width, fb=fb, freq_center=s["audio_hz"], lockingbw=s["lockingbw"])
    b.set_stream(stream.cuda_stream)
    if mode == "oqpsk8400":
        layer = jb.CChannelBatch(width)
        out, counts = np.empty((width, 8, jb.CChannelBatch.RECORD), dtype=np.uint8), np.zeros(width, dtype=np.int32)
        read = lambda: layer.read_frames_raw(out, counts)
    else:
        layer = jb.PChannelBatch(width, fb)
        out, counts = np.empty((width, layer.su_cap, 16), dtype=np.uint8), np.zeros(width, dtype=np.int32)
        read = lambda: layer.read_sus_raw(out, counts)
    m, row = 4800, x.stride(0)

    def run(blocks, k0):
        for k in range(k0, k0 + blocks):
            b.write_device(x.data_ptr() + 2 * ((k * m) % period), m, row)
            layer.process_batch(b)
            if (k + 1) % 10 == 0:
                layer.tick(b)
            read()
        return k0 + blocks

    k = run(20, 0)                                               # 2 s warm-up
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    run(int(seconds * 10), k)
    e1.record(stream)
    e1.synchronize()
    dt = e0.elapsed_time(e1) / 1e3
    b.close(); layer.close()
    return dict(test="width", mode=mode, width=width, signal_s=seconds, s_per_signal_s=dt / seconds, x_realtime=seconds / dt)


def e2e_run(torch, jb, cls, dev, fs, fmt, seconds, bytes_per, period_n, **kw):
    stream = torch.cuda.Stream()
    block_n = int(round(0.1 * fs))
    n_blocks = int(round(seconds / 0.1))
    rx = cls(fs, fmt, stream=stream.cuda_stream, **kw)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    w0, c0 = time.perf_counter(), time.process_time()
    e0.record(stream)
    n_ev = 0
    for k in range(n_blocks):
        n_ev += len(rx.write_device(dev.data_ptr() + ((k * block_n) % period_n) * bytes_per, block_n))
    n_ev += len(rx.flush())
    e1.record(stream)
    e1.synchronize()
    wall, cpu = time.perf_counter() - w0, time.process_time() - c0
    st = rx.stats()
    res = dict(path=cls.__name__, signal_s=seconds, wall_s=wall, x_realtime=seconds / wall, host_cpu_s=cpu,
               event_s=e0.elapsed_time(e1) / 1e3, events=n_ev, planned=len(st["carriers"]),
               sus=sum(c["sus"] for c in st["carriers"]), crc_failures=sum(c["crc_failures"] for c in st["carriers"]),
               cframes=sum(c["cframes"] for c in st["carriers"]))
    if "groups" in st:
        res.update(groups=st["groups"], late_locks=sum(c["late_locks"] for c in st["carriers"]),
                   unlocked_segments=sum(c["unlocked_segments"] for c in st["carriers"]),
                   pcm_bytes_peak=sum(g["pcm_bytes_peak"] for g in st["groups"]))
    rx.close()
    return res


def busy_seconds(prof):
    """the union of the device activity intervals (kernels, copies, memsets) the profiler recorded -> (seconds, intervals)"""
    from torch.autograd import DeviceType
    iv = sorted((e.time_range.start, e.time_range.end) for e in prof.events() if e.device_type == DeviceType.CUDA)
    total, end = 0.0, None
    for a, b in iv:
        if end is None or a > end:
            total += b - a
            end = b
        elif b > end:
            total += b - end
            end = b
    return total / 1e6, len(iv)


def profiled_run(torch, jb, cls, dev, fs, fmt, seconds, bytes_per, period_n, **kw):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        r = e2e_run(torch, jb, cls, dev, fs, fmt, seconds, bytes_per, period_n, **kw)
    busy, n = busy_seconds(prof)
    return dict(path=r["path"], signal_s=seconds, profiled_wall_s=r["wall_s"], device_busy_s=busy, device_intervals=n,
                busy_share=busy / r["wall_s"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=240.0, help="signal seconds per end-to-end run")
    ap.add_argument("--segment", type=int, default=10)
    ap.add_argument("--widths", default="16,256,1024,4096")
    ap.add_argument("--width-seconds", type=float, default=5.0)
    ap.add_argument("--sizes", default="0,1")
    ap.add_argument("--skip-widths", action="store_true")
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--profile", type=float, default=0.0, help="signal seconds per profiled run (0: none)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import jaero_b200 as jb
    if not torch.cuda.is_available():
        sys.exit("recording_bench: no CUDA device")
    info = card()
    lines = []

    def emit(r):
        lines.append(json.dumps(dict(info, **r)))
        print(lines[-1], flush=True)

    if not args.skip_widths:
        for mode, fb in MODES:
            for w in (int(v) for v in args.widths.split(",")):
                emit(width_run(torch, jb, mode, fb, w, args.width_seconds))
    if not args.skip_e2e:
        for i in (int(v) for v in args.sizes.split(",")):
            fs, n, fmt = SIZES[i]
            iq, _, _ = band(fs, n, fmt)
            period_n = iq.size // 2
            bytes_per = 2 if fmt == "cu8" else 4
            dev = torch.from_numpy(iq).cuda()
            size = "%.1f MS/s x %d carriers %s" % (fs / 1e6, n, fmt)
            paths = ((jb.Receiver, {}), (jb.RecordingDecoder, dict(segment_seconds=args.segment)))
            for cls, kw in paths:
                emit(dict(test="e2e", size=size, **e2e_run(torch, jb, cls, dev, fs, fmt, args.seconds, bytes_per, period_n, **kw)))
            for cls, kw in paths if args.profile > 0 else ():
                emit(dict(test="profile", size=size, **profiled_run(torch, jb, cls, dev, fs, fmt, args.profile, bytes_per,
                                                                    period_n, **kw)))
            del dev
    emit(dict(card_after=card()))
    if args.out:
        with open(args.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
