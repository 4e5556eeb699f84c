"""Throughput of the wideband IQ down-converter (jaero_b200.Ddc) on one GPU.

For each size (input rate x channels) it prints one JSON line with the card name and power limit read in the same run, and:
- ddc: input Msamples/s through the DDC alone and the multiple of real time, and the FP64 flop/s achieved against the
  algorithmic count of the planned filters (8 (D2 / L) K1 + 4 ceil(K2 / L) flop per output: complex stage-1 taps on complex
  input, real stage-2 taps of which only every L-th meets a sample that is not a stuffed zero; L = 1 for the integer rates);
- chain: the DDC -> 10.5 kbps OQPSK demodulator -> P-channel frame layer on one CUDA stream, as a multiple of real time.
The input is seeded cs16 noise, so the demodulators run unlocked. Time comes from CUDA events around whole writes.

usage: python tools/ddc_bench.py [--seconds S] [--chunk SECONDS] [--out FILE] [--sizes 0,1,...]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# integer multiples of 48 kHz first (L = 1), then an Airspy's 2.5 and 10 MS/s (L / M = 12 / 625 and 3 / 625)
SIZES = [(2.4e6, 64), (9.6e6, 1024), (2.5e6, 64), (10e6, 1024)]
B, DT, FS_OUT = 12000.0, 4000.0, 48000.0


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def bench_size(fs, C, seconds, chunk_s, torch, jaero_b200):
    L, D = jaero_b200.rate_ratio(fs, FS_OUT)
    plan = jaero_b200.ddc_plan(fs, D, B, DT, interpolation=L)
    flop_per_output = 8 * plan["D2"] * plan["K1"] / L + 4 * -(-plan["K2"] // L)
    chunk = int(round(fs * chunk_s))
    chunk -= chunk % D                                            # whole outputs per write: every write hands the demodulator chunk L/D
    steps = max(1, int(round(seconds / chunk_s)))
    rng = np.random.default_rng(1)
    iq = torch.from_numpy(rng.integers(-3000, 3000, size=2 * chunk, dtype=np.int16)).cuda()
    rng_off = np.random.default_rng(2)
    off = rng_off.uniform(-(fs / 2 - B / 2), fs / 2 - B / 2, size=C)
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()

    def run(with_chain):
        d = jaero_b200.Ddc(fs, D, off, 8000.0, B, DT, gain=4.0, interpolation=L)
        d.set_stream(stream.cuda_stream)
        b = pc = None
        if with_chain:
            b = jaero_b200.DemodBatch("oqpsk", C, fb=10500, freq_center=8000.0, lockingbw=10500)
            pc = jaero_b200.PChannelBatch(C, 10500)
            b.set_stream(stream.cuda_stream)

        def step():
            d.write_device(iq.data_ptr(), chunk, "cs16")
            if with_chain:
                ptr, n, stride = d.output()
                b.write_device(ptr, n, stride)
                pc.process_batch(b)
                pc.discard_sus()
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            step()
        e1.record(stream)
        e1.synchronize()
        ms = e0.elapsed_time(e1)
        launches = d.launches
        d.close()
        if with_chain:
            b.close(); pc.close()
        return ms / 1e3, launches

    t_ddc, launches = run(False)
    t_chain, _ = run(True)
    signal_s = steps * chunk / fs
    outputs = C * steps * chunk * L / D
    return dict(input_rate=fs, channels=C, interpolation=L, decimation=D, stages=[plan["D1"], plan["K1"], plan["D2"], plan["K2"]],
                flop_per_output=flop_per_output, signal_seconds=signal_s, writes=steps, samples_per_write=chunk,
                ddc_seconds=t_ddc, ddc_input_msps=steps * chunk / t_ddc / 1e6, ddc_x_realtime=signal_s / t_ddc,
                ddc_fp64_tflops=outputs * flop_per_output / t_ddc / 1e12, ddc_launches=launches,
                chain_seconds=t_chain, chain_x_realtime=signal_s / t_chain)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=10.0, help="seconds of signal per size")
    ap.add_argument("--chunk", type=float, default=0.1, help="seconds of signal per write")
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    ap.add_argument("--sizes", default=None, help="comma-separated indices into SIZES to run (default: all)")
    a = ap.parse_args()
    import torch
    import jaero_b200
    if not torch.cuda.is_available() or jaero_b200.lib().jaero_device_count() < 1:
        sys.exit("ddc_bench: no CUDA device")
    info = card()
    res = []
    sizes = SIZES if a.sizes is None else [SIZES[int(i)] for i in a.sizes.split(",")]
    for fs, C in sizes:
        r = dict(info, **bench_size(fs, C, a.seconds, a.chunk, torch, jaero_b200))
        print(json.dumps(r), flush=True)
        res.append(r)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
