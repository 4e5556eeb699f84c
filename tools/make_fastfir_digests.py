"""SHA-256 digests of what the two streaming FFT convolutions feed, the 8400 bps pre-filter (K6, nfft 4096, 2049 taps) and the
burst demodulators' Hilbert filter (nfft 8192, 2048 taps), and of the burst demodulators' whole output, seen through the C ABI
as every soft bit and the full status of every channel (all doubles bit for bit, all ints).

    python tools/make_fastfir_digests.py        # writes tests/golden/fastfir_digests.json (needs a GPU)

8400 bps OQPSK runs the committed oqpsk_8400 excerpt on three channels (the recording, 2/3 of it, and the recording reversed),
under write patterns that cut the 2048-sample K6 blocks at every edge. K6's mix-up frequency is set at the end of every write
(mixer_fir_pre.SetFreq(mixer2_freq_sum/i)), so the 8400 bps output depends on how the stream is cut and every pattern has its
own digest. The burst modes run the tests/burst_edge_streams.py streams whose accepted fill completes at a multiple of the
6145-sample Hilbert block and one sample after it, with 4800-sample and with odd-sized writes. The burst_* cases pin the burst
demodulators themselves: one channel per tests/burst_edge_streams.py stream of the mode (9 for MSK, 10 for burst OQPSK, so the
last 32-channel group of the demodulator tail has idle lanes) under both write patterns, plus burst MSK 1200 with AFC off and
burst OQPSK with the squelch on.
tests/test_gpu_fastfir_digest.py recomputes the digests and compares them."""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "fastfir_digests.json")

K6_L = 2048
# 8400 bps write patterns: name -> write lengths (the last one repeats, cut short at the end of the excerpt)
PATTERNS_8400 = {
    "w2047": [2047],
    "w2048": [2048],
    "w2049": [2049],
    "single_edges": [K6_L - 4] + [1] * 8 + [K6_L - 8] + [1] * 8 + [4800],    # one-sample writes across the 1st and 2nd block edge
    "w4800": [4800],
    "w80000": [80000],              # many blocks per write; a longer write would overflow the 16864-value soft-bit ring
}
BURST_MODES = ["msk1200", "msk600", "oqpsk"]
BURST_STREAMS = ["hil_edge", "hil_edge1"]
BURST_PATTERNS = ["P1", "P2"]
# burst_<mode>_<set>_<pattern>: "all" is every stream of the mode; "afc0" is that with AFC off, "sql" with the squelch on
BURST_SETS = [(m, "all", p) for m in BURST_MODES for p in BURST_PATTERNS] + [("msk1200", "afc0", "P1"), ("oqpsk", "sql", "P1")]


def _writes(pattern, n):
    out, a, k = [], 0, 0
    while a < n:
        w = min(pattern[min(k, len(pattern) - 1)], n - a)
        out.append(w); a += w; k += 1
    return out


def _status_digest(status):
    """every field of every channel's status, doubles as their exact hex form"""
    def enc(v):
        if isinstance(v, float):
            return v.hex()
        if isinstance(v, int):
            return str(v)
        return "[" + ",".join(enc(float(x)) for x in v) + "]"           # ctypes double arrays (scatter)
    text = "\n".join(";".join("%s=%s" % (k, enc(v)) for k, v in st.items()) for st in status)
    return hashlib.sha256(text.encode()).hexdigest()


def _run(batch, pcm2, writes):
    acc = [[] for _ in range(pcm2.shape[0])]
    a = 0
    for w in writes:
        batch.write(pcm2[:, a:a + w]); a += w
        for c, s in enumerate(batch.read_softbits()):
            acc[c].append(s)
    soft = hashlib.sha256(b"".join(np.concatenate(x).astype("<i2").tobytes() + b"|" for x in acc)).hexdigest()
    st = _status_digest(batch.status())
    batch.close()
    return dict(soft=soft, status=st)


def cases():
    return (["8400_" + p for p in PATTERNS_8400] + ["%s_%s" % (m, p) for m in BURST_MODES for p in BURST_PATTERNS]
            + ["burst_%s_%s_%s" % s for s in BURST_SETS])


def run_case(name):
    """-> dict(soft=digest of every channel's soft bits, status=digest of every channel's status)"""
    import jaero_b200
    from conftest import load_excerpt
    if name.startswith("8400_"):
        pcm = load_excerpt("oqpsk_8400")
        pcm2 = np.stack([pcm, (pcm.astype(np.int32) * 2 // 3).astype(np.int16), pcm[::-1].copy()])
        b = jaero_b200.DemodBatch("oqpsk", 3, fb=8400, freq_center=8000.0, lockingbw=10500, fft_power=14,
                                  signalthreshold=0.65, afc=True)
        return _run(b, pcm2, _writes(PATTERNS_8400[name[5:]], pcm2.shape[1]))
    import burst_edge_streams as S
    if name.startswith("burst_"):
        mode, streams, pattern = name[6:].split("_")
    else:
        (mode, pattern), streams = name.rsplit("_", 1), "edges"
    v = S.variants(mode)
    pcm2 = np.stack([v[k] for k in (BURST_STREAMS if streams == "edges" else v)])
    m = S.MODES[mode]
    C = pcm2.shape[0]
    if m["kind"] == "burst_oqpsk":
        b = jaero_b200.BurstOqpskBatch(C, sql=streams == "sql", **m["kw"])
    else:
        b = jaero_b200.BurstMskBatch(C, **m["kw"])
        if streams == "afc0":
            jaero_b200._check(jaero_b200.lib().jaero_burst_set_afc(b.h, 0))
    return _run(b, pcm2, S.cycle_writes(getattr(S, pattern), pcm2.shape[1]))


if __name__ == "__main__":
    out = {name: run_case(name) for name in cases()}
    with open(OUT, "w") as fh:
        json.dump(out, fh, indent=1, sort_keys=True)
        fh.write("\n")
    print("wrote %s (%d cases)" % (OUT, len(out)))
