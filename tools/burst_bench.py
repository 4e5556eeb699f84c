"""BASELINE cfg 4: the 1200 bps burst recording replicated over N channels through the burst demodulator + R/T packet layer.
With --oqpsk, the 10.5 kbps burst OQPSK excerpt instead, through the burst OQPSK demodulator + R/T packet layer.

    python tools/burst_bench.py [channels] [--oqpsk]"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import jaero_b200  # noqa: E402

if __name__ == "__main__":
    args = [x for x in sys.argv[1:] if x != "--oqpsk"]
    oqpsk = "--oqpsk" in sys.argv[1:]
    C = int(args[0]) if args else 2048
    if oqpsk:
        name, fb, label = "burst_oqpsk_10500_excerpt.npz", 10500, "burst OQPSK 10500"
        make = lambda: jaero_b200.BurstOqpskBatch(C, fb=10500.0, freq_center=8000.0, lockingbw=10500.0, signalthreshold=0.6)
    else:
        name, fb, label = "burst_msk_1200_a_excerpt.npz", 1200, "burst MSK 1200"
        make = lambda: jaero_b200.BurstMskBatch(C, fb=1200.0, freq_center=1000.0, lockingbw=1800.0, signalthreshold=0.6)
    pcm = np.load(os.path.join(ROOT, "tests", "golden", name))["pcm"]
    pcm2 = np.ascontiguousarray(np.tile(pcm[None, :], (C, 1)))
    b = make()
    rt = jaero_b200.RTChannelBatch(C, fb)
    chunk = 48000
    b.write(pcm2[:, :chunk]); rt.process_burst(b); b.sync()          # warm-up (allocations, module load)
    b.close(); rt.close()
    b = make()
    rt = jaero_b200.RTChannelBatch(C, fb)
    t0 = time.perf_counter()
    npk = 0
    for a in range(0, pcm2.shape[1], chunk):
        b.write(pcm2[:, a:a + chunk])
        rt.process_burst(b)
        npk += sum(len(p) for p in rt.read_packets())
    b.sync()
    dt = time.perf_counter() - t0
    st = b.status()
    print("%s: %d channels x %d samples in %.2f s = %.1f Msamples/s (host buffers, wall clock); bursts acquired %d, T packets %d, launches %d" % (
        label, C, pcm2.shape[1], dt, C * pcm2.shape[1] / dt / 1e6, int(sum(s["n_sig_true"] for s in st)), npk, b.launches + rt.launches))
