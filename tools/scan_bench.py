"""Throughput of the wideband carrier scanner (jaero_b200.Scanner) on one GPU.

For each input rate x nfft x hop it prints one JSON line with the card name and power limit read in the same run, and:
- scan: input Msamples/s through the scanner alone, the multiple of real time, and the FP64 flop/s achieved against the
  count 5 nfft log2(nfft) flop per frame (a radix-2 complex FFT; the window and |X|^2 are not counted);
- at 9.6 MS/s, nfft 2^16: the scanner beside a 1024-channel down-converter on the same CUDA stream and the same IQ buffer, the
  time that pair takes against the down-converter alone (the scan's share of a scan-while-receiving set-up).
The input is seeded cs16 noise. Time comes from CUDA events around whole writes after warm-up writes; --repeat runs each
size that many times.

usage: python tools/scan_bench.py [--seconds S] [--chunk SECONDS] [--repeat R] [--out FILE]
"""
import argparse
import json
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.ddc_bench import card  # noqa: E402

SIZES = [(fs, 1 << p, h) for fs in (2.4e6, 9.6e6) for p in (14, 16) for h in (2, 4)]
B, DT, FS_OUT, DDC_CHANNELS = 12000.0, 4000.0, 48000.0, 1024


def timed(stream, steps, step, torch):
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        step()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / 1e3


def bench_size(fs, nfft, hop_div, seconds, chunk_s, torch, jaero_b200, with_ddc):
    D = int(round(fs / FS_OUT))
    chunk = int(round(fs * chunk_s))
    chunk -= chunk % D
    steps = max(1, int(round(seconds / chunk_s)))
    rng = np.random.default_rng(1)
    iq = torch.from_numpy(rng.integers(-3000, 3000, size=2 * chunk, dtype=np.int16)).cuda()
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    hop = nfft // hop_div
    s = jaero_b200.Scanner(fs, nfft, hop)
    s.set_stream(stream.cuda_stream)
    t_scan = timed(stream, steps, lambda: s.write_device(iq.data_ptr(), chunk, "cs16"), torch)
    frames = steps * chunk / hop
    signal_s = steps * chunk / fs
    r = dict(input_rate=fs, nfft=nfft, hop=hop, signal_seconds=signal_s, writes=steps, samples_per_write=chunk,
             scan_seconds=t_scan, scan_input_msps=steps * chunk / t_scan / 1e6, scan_x_realtime=signal_s / t_scan,
             scan_fp64_gflops=frames * 5 * nfft * math.log2(nfft) / t_scan / 1e9)
    if with_ddc:
        off = np.random.default_rng(2).uniform(-(fs / 2 - B / 2), fs / 2 - B / 2, size=DDC_CHANNELS)
        d = jaero_b200.Ddc(fs, D, off, 8000.0, B, DT, gain=4.0)
        d.set_stream(stream.cuda_stream)
        t_ddc = timed(stream, steps, lambda: d.write_device(iq.data_ptr(), chunk, "cs16"), torch)

        def both():
            d.write_device(iq.data_ptr(), chunk, "cs16")
            s.write_device(iq.data_ptr(), chunk, "cs16")
        t_both = timed(stream, steps, both, torch)
        d.close()
        r.update(ddc_channels=DDC_CHANNELS, ddc_seconds=t_ddc, ddc_plus_scan_seconds=t_both, scan_share_of_ddc=(t_both - t_ddc) / t_ddc)
    s.close()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=10.0, help="seconds of signal per size")
    ap.add_argument("--chunk", type=float, default=0.1, help="seconds of signal per write")
    ap.add_argument("--repeat", type=int, default=2, help="runs of each size")
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    a = ap.parse_args()
    import torch
    import jaero_b200
    if not torch.cuda.is_available() or jaero_b200.lib().jaero_device_count() < 1:
        sys.exit("scan_bench: no CUDA device")
    info = card()
    res = []
    for run in range(a.repeat):
        for fs, nfft, hop_div in SIZES:
            r = dict(info, run=run, **bench_size(fs, nfft, hop_div, a.seconds, a.chunk, torch, jaero_b200,
                                                with_ddc=(fs == 9.6e6 and nfft == 1 << 16)))
            print(json.dumps(r), flush=True)
            res.append(r)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
