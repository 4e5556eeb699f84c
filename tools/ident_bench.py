"""Throughput of the mode identifier (jaero_b200.Identifier) on one GPU.

Prints one JSON line per size with the card name and power limit read in the same run:
- ident: 48 kHz PCM at 64, 1024 and 4096 channels, nfft 2^14, as a multiple of real time, with the achieved FP64 flop/s and
  bytes/s against the cost model kept here: 3 x 5 N log2 N flop per frame (three complex transforms), and per frame bin the
  bytes the five kernels move through L2 / HBM (reads and writes of the int16 frame, the window, three double2 work matrices
  written and read, the double power row written and read, the running sum read and written).
- probe: probe_carriers' wall time (host clock around a call that ends in a device synchronise) on 4 s of a 9.6 MS/s cs16
  stream with 1024 candidate carriers.
The input is seeded int16 noise, 10 s of it written in 0.1 s writes. Time comes from CUDA events around whole writes, after
three warm-up writes.

usage: python tools/ident_bench.py [--seconds S] [--out FILE] [--sizes 64,1024,4096] [--no-probe]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FS, NFFT, CHUNK_S = 48000, 16384, 0.1
# bytes per frame bin: load reads 2 (int16, each sample in two frames: 2 x 2 / 2) + 8 (window) and writes 16; mask, square and
# power each read 16, mask and square write 16, power writes 8; accumulate reads 8 + 8 and writes 8
BYTES_PER_BIN = 2 + 8 + 16 + 16 + 16 + 16 + 16 + 16 + 8 + 8 + 8 + 8


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def timed(stream, torch, steps, step):
    for k in range(3):
        step(k)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for k in range(steps):
        step(k)
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / 1e3


def bench_size(C, seconds, torch, jaero_b200):
    chunk = int(round(FS * CHUNK_S))
    steps = int(round(seconds / CHUNK_S))
    n = chunk * steps
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randint(-3000, 3000, (C, n), dtype=torch.int16, device="cuda", generator=g)
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    d = jaero_b200.Identifier(FS, C, NFFT)
    d.set_stream(stream.cuda_stream)
    l0 = d.launches
    t = timed(stream, torch, steps, lambda k: d.write_device(x.data_ptr() + 2 * (k % steps) * chunk, chunk, n))
    launches = d.launches - l0
    _, frames = d.read()
    d.close()
    del x
    torch.cuda.empty_cache()
    timed_frames = C * seconds * FS / (NFFT // 2)
    flop = timed_frames * 3 * 5 * NFFT * math.log2(NFFT)
    byts = timed_frames * NFFT * BYTES_PER_BIN
    return dict(rate=FS, channels=C, nfft=NFFT, signal_seconds=seconds, writes=steps, samples_per_write=chunk, seconds=t,
                x_realtime=seconds / t, fp64_gflops=flop / t / 1e9, model_bytes_per_bin=BYTES_PER_BIN, model_gbytes=byts / 1e9,
                achieved_gbytes_per_s=byts / t / 1e9, launches=launches, frames_per_channel=frames)


def bench_probe(torch, jaero_b200, C=1024, rate=9.6e6, seconds=4.0):
    n = int(rate * seconds)
    g = torch.Generator(device="cuda").manual_seed(2)
    iq = torch.randint(-2000, 2000, (2 * n,), dtype=torch.int16, device="cuda", generator=g)
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    span = 0.45 * rate
    cands = [dict(center_hz=-span + 2 * span * k / C, lo_hz=-span + 2 * span * k / C - 3000, hi_hz=-span + 2 * span * k / C + 3000,
                  mode="unknown", power=1e-3, flags=0) for k in range(C)]
    run = lambda s: jaero_b200.probe_carriers(cands, rate, (iq.data_ptr(), n), "cs16", seconds=s, stream=stream.cuda_stream)
    run(0.5)                                                            # warm-up: module load, first allocations
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = run(seconds)
    torch.cuda.synchronize()
    t = time.perf_counter() - t0
    del iq
    torch.cuda.empty_cache()
    return dict(probe_input_rate=rate, probe_channels=C, probe_signal_seconds=seconds, probe_wall_seconds=t,
                probe_unknown=sum(c["mode"] == "unknown" for c in out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=10.0, help="seconds of signal per size")
    ap.add_argument("--sizes", default="64,1024,4096", help="comma-separated channel counts")
    ap.add_argument("--no-probe", action="store_true", help="skip the probe_carriers timing")
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    a = ap.parse_args()
    import torch
    import jaero_b200
    if not torch.cuda.is_available() or jaero_b200.lib().jaero_device_count() < 1:
        sys.exit("ident_bench: no CUDA device")
    info = card()
    res = []
    for C in [int(s) for s in a.sizes.split(",")]:
        r = dict(info, **bench_size(C, a.seconds, torch, jaero_b200))
        print(json.dumps(r), flush=True)
        res.append(r)
    if not a.no_probe:
        r = dict(info, **bench_probe(torch, jaero_b200))
        print(json.dumps(r), flush=True)
        res.append(r)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
