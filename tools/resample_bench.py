"""Throughput of the PCM rate converter (jaero_b200.Resampler) on one GPU.

Prints one JSON line per size with the card name and power limit read in the same run:
- resample: 44.1 -> 48 kHz at 64, 1024 and 4096 channels, as a multiple of real time, and the FP64 flop/s achieved against the
  algorithmic count of 2 ceil(K / L) flop per output (one multiply-add per tap of a phase; the zero-stuffed samples cost nothing);
- chain (4096 channels): Resampler -> 10.5 kbps OQPSK DemodBatch on one CUDA stream, against the same DemodBatch fed 48 kHz PCM
  from the device directly, and the resampler's share of the chain's time.
The input is seeded int16 noise, 10 s of it written in 0.1 s writes (4410 samples per channel). Time comes from CUDA events
around whole writes, after three warm-up writes.

usage: python tools/resample_bench.py [--seconds S] [--out FILE] [--sizes 64,1024,4096]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FS_IN, FS_OUT, CHUNK_S = 44100, 48000, 0.1


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


def bench_size(C, seconds, chain, torch, jaero_b200):
    chunk = int(round(FS_IN * CHUNK_S))
    steps = int(round(seconds / CHUNK_S))
    n = chunk * steps
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randint(-3000, 3000, (C, n), dtype=torch.int16, device="cuda", generator=g)
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    r = jaero_b200.Resampler(FS_IN, C, output_rate=FS_OUT)
    r.set_stream(stream.cuda_stream)
    L, K = r.plan["L"], r.plan["K"]
    flop_per_output = 2 * -(-K // L)
    t_rs = timed(stream, torch, steps, lambda k: r.write_device(x.data_ptr() + 2 * (k % steps) * chunk, chunk, n))
    launches = r.launches
    outputs = C * steps * chunk * FS_OUT // FS_IN
    res = dict(input_rate=FS_IN, output_rate=FS_OUT, channels=C, L=L, M=r.plan["M"], K=K, flop_per_output=flop_per_output,
               signal_seconds=seconds, writes=steps, samples_per_write=chunk, resample_seconds=t_rs, resample_x_realtime=seconds / t_rs,
               resample_fp64_tflops=outputs * flop_per_output / t_rs / 1e12, resample_launches=launches)
    if chain:
        m = chunk * FS_OUT // FS_IN
        pcm48 = torch.randint(-3000, 3000, (C, m), dtype=torch.int16, device="cuda", generator=g)
        torch.cuda.synchronize()

        def demod():
            b = jaero_b200.DemodBatch("oqpsk", C, fb=10500, freq_center=8000.0, lockingbw=10500)
            b.set_stream(stream.cuda_stream)
            return b
        b = demod()
        t_demod = timed(stream, torch, steps, lambda k: b.write_device(pcm48.data_ptr(), m, m))
        b.close()
        b = demod()

        def step(k):
            r.write_device(x.data_ptr() + 2 * (k % steps) * chunk, chunk, n)
            ptr, mo, stride = r.output()
            b.write_device(ptr, mo, stride)
        t_chain = timed(stream, torch, steps, step)
        b.close()
        res.update(demod_seconds=t_demod, demod_x_realtime=seconds / t_demod, chain_seconds=t_chain, chain_x_realtime=seconds / t_chain,
                   chain_added_over_demod=t_chain / t_demod - 1.0, resample_share_of_chain=t_rs / t_chain)
    r.close()
    del x
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=10.0, help="seconds of signal per size")
    ap.add_argument("--sizes", default="64,1024,4096", help="comma-separated channel counts; the largest also runs the chain")
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    a = ap.parse_args()
    import torch
    import jaero_b200
    if not torch.cuda.is_available() or jaero_b200.lib().jaero_device_count() < 1:
        sys.exit("resample_bench: no CUDA device")
    info = card()
    sizes = [int(s) for s in a.sizes.split(",")]
    res = []
    for C in sizes:
        r = dict(info, **bench_size(C, a.seconds, C == max(sizes), torch, jaero_b200))
        print(json.dumps(r), flush=True)
        res.append(r)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
