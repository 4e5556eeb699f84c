"""Overhead of jaero_b200.Receiver over the same stages wired by hand, on one GPU.

For each size (input rate x carriers) a periodic wideband IQ signal is built (mixed continuous modes: 10.5 kbps and 8400 bps
OQPSK, 1200 and 600 bps MSK P-channel frames, every carrier at Eb/N0 15 dB; 2 s long and circular, so it can be fed for as long
as the run lasts) and copied to the device once. Then, on one CUDA stream and in alternating rounds:
- receiver: a Receiver acquires on the first seconds (not timed), runs warm-up blocks, and then the timed blocks go through
  write_device, one block per call;
- by hand: the Ddc / DemodBatch / PChannelBatch / CChannelBatch groups channel_plan gives for the receiver's carriers, and one
  Reassembler per P-channel carrier, fed the same blocks in the same order (write the DDC, demodulate, run the frame layer,
  tick once per second of signal, read the signal units or frames, push the CRC-valid ones, pop the messages).
Time comes from CUDA events on the stream around the timed blocks; both paths read their results back every block, so the
window ends in a device synchronise. Each size prints one JSON line: the card, its power limit and SM clock read in the same
run, the carriers planned, the median seconds per signal second of both paths, the receiver's overhead in percent and the
multiple of real time.

usage: python tools/receive_bench.py [--seconds S] [--warmup S] [--rounds R] [--block SECONDS] [--sizes 0,1] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SIZES = [(2.4e6, 16, "cu8"), (9.6e6, 256, "cs16")]
PERIOD = 2.0                                                     # seconds; a whole number of frames of every P-channel rate
MODES = [("oqpsk10500", 10500), ("msk1200", 1200), ("oqpsk8400", 8400), ("msk600", 600)]
EBN0_DB = 15.0


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    name, power, clock, max_clock = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return dict(gpu=name, power_limit=power, sm_clock=clock, max_sm_clock=max_clock)


def envelope(mode, fb, seed):
    """PERIOD seconds of one mode's circular 48 kHz envelope"""
    from jaero_b200 import synth
    if mode == "oqpsk8400":                                      # no frame structure needed: random bits
        bits = np.random.default_rng(seed).integers(0, 2, int(PERIOD * fb)).astype(np.uint8)
        return synth.oqpsk_envelope(bits, fb)
    n_frames = int(round(PERIOD * fb / synth.frame_params(fb)["frame_bits"]))
    if mode == "oqpsk10500":
        return synth.oqpsk_envelope(synth.pchannel_bits(fb, n_frames, seed=seed, loop=True), fb)
    return synth.msk_envelope(synth.pchannel_bits(fb, n_frames, seed=seed, loop=True, even_parity=True), fb)


def band(fs, n_carriers, fmt, seed=1):
    """PERIOD seconds of circular IQ at fs with n_carriers carriers of mixed modes, spread evenly over 90 % of the band, built in
    the frequency domain (every offset a multiple of 1 / PERIOD Hz) -> (interleaved IQ, offsets, modes)"""
    N = int(round(fs * PERIOD))
    rng = np.random.default_rng(seed)
    W = (rng.standard_normal(N) + 1j * rng.standard_normal(N)) * np.sqrt(N / 2.0)     # unit-variance complex noise
    envs = {}
    spacing = 0.9 * fs / n_carriers
    offs, modes = [], []
    for i in range(n_carriers):
        mode, fb = MODES[i % len(MODES)]
        k = i % 3
        if (mode, k) not in envs:
            e = envelope(mode, fb, 100 + 7 * i)
            envs[(mode, k)] = np.fft.fft(e / np.sqrt(np.mean(np.abs(e) ** 2)))
        E = envs[(mode, k)]
        ne = len(E)
        f = round((-0.45 * fs + (i + 0.5) * spacing) * PERIOD) / PERIOD
        if abs(f) < 20e3:
            f += 40e3
        amp = np.sqrt(10 ** (EBN0_DB / 10.0) * fb / fs) * N / ne
        kf = np.fft.fftfreq(ne, 1.0 / 48000.0)
        W[np.round((kf + f) * PERIOD).astype(np.int64) % N] += amp * E
        offs.append(f); modes.append(mode)
    x = np.fft.ifft(W)
    x *= 0.25 / np.sqrt(np.mean(np.abs(x) ** 2))
    iq = np.empty(2 * N)
    iq[0::2], iq[1::2] = x.real, x.imag
    if fmt == "cu8":
        return np.clip(np.round(iq * 128.0 + 127.5), 0, 255).astype(np.uint8), offs, modes
    return np.clip(np.round(iq * 32768.0), -32768, 32767).astype(np.int16), offs, modes


class ByHand:
    """The stages of channel_plan(carriers), wired as INTEGRATION.md 3a describes, with the reads a user needs"""

    def __init__(self, jb, carriers, fs, fmt, stream):
        L, M = jb.rate_ratio(fs)
        plans, _ = jb.channel_plan(carriers, fs, M, L)
        self.fs, self.fmt, self.n_in, self.ticks = int(fs), fmt, 0, 0
        self.groups = []
        for mode in sorted(plans, key=lambda m: plans[m]["carriers"][0]["center_hz"]):
            p = plans[mode]
            d, b = jb.Ddc(**p["ddc"]), jb.DemodBatch(**p["demod"])
            d.set_stream(stream); b.set_stream(stream)
            if mode == "oqpsk8400":
                layer, rs = jb.CChannelBatch(b.n), None
            else:
                layer, rs = jb.PChannelBatch(b.n, p["demod"]["fb"]), [jb.Reassembler() for _ in range(b.n)]
            self.groups.append((d, b, layer, rs))
        self.messages = 0

    def block(self, ptr, n):
        for d, b, layer, _ in self.groups:
            d.write_device(ptr, n, self.fmt)
            b.write_device(*d.output())
            layer.process_batch(b)
        self.n_in += n
        due = self.n_in // self.fs - self.ticks
        for _ in range(due):
            for _, b, layer, _ in self.groups:
                layer.tick(b)
        self.ticks += due
        for _, _, layer, rs in self.groups:
            if rs is None:
                layer.read_frames()
                continue
            out, counts = layer.read_sus_raw()
            for ch in np.flatnonzero(counts):
                recs = out[ch, :counts[ch]]
                for r in recs[recs[:, 12] != 0]:
                    rs[ch].push_su(r[:12].tobytes())
                self.messages += len(rs[ch].pop_all())

    def close(self):
        for d, b, layer, rs in self.groups:
            d.close(); b.close(); layer.close()
            for r in rs or []:
                r.close()


def timed(torch, stream, feed, dev, bytes_per, block_n, period_n, start, n_blocks):
    """seconds for n_blocks blocks fed from the circular device signal, from sample `start` on"""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    a = start
    for _ in range(n_blocks):
        feed(dev.data_ptr() + (a % period_n) * bytes_per, block_n)
        a += block_n
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / 1e3


def bench_size(fs, n_carriers, fmt, args, torch, jb):
    iq, offs, modes = band(fs, n_carriers, fmt)
    period_n = iq.size // 2
    bytes_per = 2 if fmt == "cu8" else 4
    block_n = int(round(args.block * fs))
    assert period_n % block_n == 0, "the signal period must hold whole blocks"
    stream = torch.cuda.Stream()
    dev = torch.from_numpy(np.concatenate([iq, iq[:2 * block_n]])).cuda()   # a block may wrap past the period's end
    torch.cuda.synchronize()
    acquire = 4.0
    rx = jb.Receiver(fs, fmt, acquire_seconds=acquire, block_seconds=args.block, stream=stream.cuda_stream)
    a = 0
    while not rx.acquired:                                       # acquisition, not timed
        rx.write_device(dev.data_ptr() + (a % period_n) * bytes_per, block_n); a += block_n
    carriers = [dict(c) for c in rx.carriers()]
    hand = ByHand(jb, carriers, fs, fmt, stream.cuda_stream)
    warm, steps = int(round(args.warmup / args.block)), int(round(args.seconds / args.block))
    h_at = 0
    hand_feed = hand.block
    # both paths start from sample 0 of the period: the by-hand groups first decode what the receiver decoded while acquiring
    for _ in range(int(round(acquire / args.block))):
        hand.block(dev.data_ptr() + (h_at % period_n) * bytes_per, block_n); h_at += block_n
    timed(torch, stream, rx.write_device, dev, bytes_per, block_n, period_n, a, warm); a += warm * block_n
    timed(torch, stream, hand_feed, dev, bytes_per, block_n, period_n, h_at, warm); h_at += warm * block_n
    t_rx, t_hand = [], []
    for _ in range(args.rounds):
        t_rx.append(timed(torch, stream, rx.write_device, dev, bytes_per, block_n, period_n, a, steps)); a += steps * block_n
        t_hand.append(timed(torch, stream, hand_feed, dev, bytes_per, block_n, period_n, h_at, steps)); h_at += steps * block_n
    signal_s = steps * block_n / fs
    rx_s, hand_s = float(np.median(t_rx)) / signal_s, float(np.median(t_hand)) / signal_s
    by_mode = {}
    for c in carriers:
        by_mode[c["mode"]] = by_mode.get(c["mode"], 0) + 1
    st = rx.stats()
    res = dict(size="%.1f MS/s x %d carriers %s" % (fs / 1e6, n_carriers, fmt), planned=len(carriers), planned_by_mode=by_mode,
               unplanned=len(rx.unplanned()), block_s=args.block, timed_signal_s=signal_s, rounds=args.rounds,
               receiver_s_per_signal_s=rx_s, by_hand_s_per_signal_s=hand_s, overhead_pct=100.0 * (rx_s / hand_s - 1.0),
               receiver_x_realtime=1.0 / rx_s, by_hand_x_realtime=1.0 / hand_s,
               receiver_rounds_s=t_rx, by_hand_rounds_s=t_hand,
               receiver_messages=sum(c["messages"] for c in st["carriers"]), by_hand_messages=hand.messages)
    rx.close(); hand.close()
    del dev
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=10.0, help="signal seconds per timed round")
    ap.add_argument("--warmup", type=float, default=2.0, help="signal seconds of warm-up blocks per path")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--block", type=float, default=0.1)
    ap.add_argument("--sizes", default=",".join(str(i) for i in range(len(SIZES))))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import jaero_b200 as jb
    if not torch.cuda.is_available():
        sys.exit("receive_bench: no CUDA device")
    info = card()
    lines = []
    for i in (int(s) for s in args.sizes.split(",")):
        fs, n, fmt = SIZES[i]
        r = dict(info, **bench_size(fs, n, fmt, args, torch, jb))
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
