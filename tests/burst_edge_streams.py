"""Deterministic test streams and write patterns for the burst demodulators' edge tests (tests/test_burst_edges_cpu.py and
tests/test_gpu_burst_edges.py).

Every stream is built from the committed excerpts only: circular shifts and splices place trident-buffer fills where the
device path cuts its work (internal chunks of CHUNK samples, Hilbert blocks of HIL_L samples), frequency-offset replicas
(synth.offset_replicas, as in cfg 4) give channels whose fills coincide, and for burst OQPSK a gated carrier packs fills as
densely as the burst detector allows. Fill positions come from the restated oracle's fill log (take_aux(2)); a placement
that does not land exactly where planned raises, so the streams are the same on every machine."""
import numpy as np

from conftest import load_excerpt
from jaero_b200 import synth
from oracle import restated

CHUNK = 16384          # internal chunk of jaero_burst_write_device (BURST_CHUNK, burst.cuh)
HIL_L = 6145           # Hilbert overlap-save block: nfft 8192 - 2048 taps + 1
EV_ROUND = 128         # trident events per launch
SOFT_CAP = {"msk1200": 4096, "msk600": 4096, "oqpsk": 21064}

MODES = {
    "msk1200": dict(kind="burst_msk", kw=dict(fb=1200.0, freq_center=1000.0, lockingbw=1800.0, signalthreshold=0.6), tri_sz=8000, span=300.0),
    "msk600": dict(kind="burst_msk", kw=dict(fb=600.0, freq_center=500.0, lockingbw=900.0, signalthreshold=0.6), tri_sz=17920, span=150.0),
    "oqpsk": dict(kind="burst_oqpsk", kw=dict(fb=10500.0, freq_center=8000.0, lockingbw=10500.0, signalthreshold=0.6), tri_sz=2633, span=300.0),
}

P1 = [4800]
P2 = [1, 2, 3, 7, 8, 9, 63, 64, 65, 4093, 6144, 6145, 6146, 16383, 16384, 16385, 1]
P4 = [65536, 40000, 49152, 61440, 45055]
N_LAYOUT_B = 300


def stretched_600(name):
    """a 1200 bps burst recording time-stretched 2x: the same bursts at 600 bps, 500 Hz carrier"""
    from scipy.signal import resample_poly
    y = resample_poly(load_excerpt(name).astype(np.float64), 2, 1)
    return np.clip(np.round(y), -32768, 32767).astype(np.int16)


def base_stream(mode):
    return stretched_600("burst_msk_1200_a") if mode == "msk600" else load_excerpt("burst_oqpsk_10500" if mode == "oqpsk" else "burst_msk_1200_a")


def oracle_fills(mode, x, writes=None, sql=False):
    """(fill sample indices, accepted flags, soft bits) of the restated oracle over stream x"""
    m = MODES[mode]
    d = restated.OracleDemod(m["kind"], sql=sql, **m["kw"])
    a = 0
    for n in (writes if writes is not None else [65536] * -(-len(x) // 65536)):
        d.write(x[a:a + n]); a += n
    f = d.take_aux(2).astype(np.int64)
    acc = d.take_aux(1).reshape(-1, 5)[:, 4] > 0
    soft = d.take_soft()
    d.close()
    assert len(f) == len(acc)
    return f, acc, soft


def cycle_writes(pattern, n):
    """write lengths repeating `pattern` until n samples are written (the last one cut short)"""
    out, a, k = [], 0, 0
    while a < n:
        w = min(pattern[k % len(pattern)], n - a)
        out.append(w); a += w; k += 1
    return out


def writes_at(points, n, cap=48000):
    """write lengths whose boundaries fall on `points`, no write longer than cap"""
    cuts = sorted({int(p) for p in points if 0 < p < n})
    edges = [0]
    for c in cuts + [n]:
        while c - edges[-1] > cap:
            edges.append(edges[-1] + cap)
        edges.append(c)
    return list(np.diff(edges))


def chunk_spans(writes):
    """[start, end) of every internal chunk the device path runs for these writes"""
    spans, a = [], 0
    for w in writes:
        for c in range(0, w, CHUNK):
            spans.append((a + c, a + min(w, c + CHUNK)))
        a += w
    return spans


def _place(mode, x, src, target):
    """circularly shift x so that the fill oracle_fills(x) puts at src completes at target instead"""
    d = target - src
    for _ in range(4):
        y = np.roll(x, d)
        f = oracle_fills(mode, y)[0]
        near = f[np.argmin(np.abs(f - target))]
        if near == target:
            return y
        d += target - near
    raise AssertionError("could not place a %s fill at %d" % (mode, target))


def gated_carrier(n, period, duty, f0=8000.0, amp=8000.0, seed=7):
    """burst OQPSK capacity probe: a carrier switched on for duty * period of every period samples, in light noise"""
    k = np.arange(n)
    rng = np.random.default_rng(seed)
    x = amp * np.cos(2 * np.pi * f0 * k / 48000.0) * ((k % period) < duty * period) + rng.normal(0, 200.0, n)
    return np.clip(np.round(x), -32768, 32767).astype(np.int16)


# fills tri_sz + 1 = 2634 samples apart at the closest: 7 of them complete inside one internal chunk, the most the trident
# buffer bound allows (consecutive fills complete at least tri_sz + 1 samples apart)
DENSE = dict(period=2636, duty=0.5)
SPLICE_PAIR = {"msk1200": 1, "msk600": 0, "oqpsk": 1}      # accepted bursts k, k + 1 of the recording


def splice(mode, x, A):
    """(stream, planned fill) with the quiet after accepted burst k cut short, so that burst k + 1 follows it sooner. The
    cut starts 1 s (the AGC window) after burst k's fill and leaves 4 trident buffers of quiet before burst k + 1's fill."""
    k = SPLICE_PAIR[mode]
    gap = int(A[k + 1] - A[k])
    cut = min(gap - 48000 - 4 * MODES[mode]["tri_sz"], gap // 2)
    s0 = int(A[k]) + 48000
    return np.concatenate([x[:s0], x[s0 + cut:], x[:cut]]), int(A[k + 1]) - cut, int(A[k])


_cache = {}


def variants(mode):
    """{name: stream} for one mode; all streams have the base recording's length. Names:
    base, off0, off1        the recording and two frequency-offset replicas (fills at the same samples)
    chunk_last, chunk_first an accepted fill completing on the last / first sample of a P4 internal chunk
    hil_edge, hil_edge1     an accepted fill completing at a multiple of HIL_L / one sample after it
    inside                  the stream starts inside a burst's preamble
    splice                  two recorded bursts moved closer together
    dense                   (burst OQPSK) fills as close together as the detector places them"""
    if mode in _cache:
        return _cache[mode]
    m = MODES[mode]
    x = base_stream(mode)
    n = len(x)
    f, acc, _ = oracle_fills(mode, x)
    A = f[acc]
    v = {"base": x}
    offs = synth.replica_offsets(0, 2, span_hz=m["span"])
    v["off0"], v["off1"] = synth.offset_replicas(x, offs)
    starts = np.array([s for s, _ in chunk_spans(cycle_writes(P4, n))])
    b = int(starts[np.argmin(np.abs(starts - A[0]))])
    v["chunk_last"] = _place(mode, x, A[0], b - 1)
    v["chunk_first"] = _place(mode, x, A[0], b)
    h = int(round(A[-1] / HIL_L)) * HIL_L
    v["hil_edge"] = _place(mode, x, A[-1], h)
    v["hil_edge1"] = _place(mode, x, A[-1], h + 1)
    v["inside"] = np.roll(x, -(int(A[0]) - m["tri_sz"] // 2))
    v["splice"] = splice(mode, x, A)[0]
    if mode == "oqpsk":
        v["dense"] = gated_carrier(n, **DENSE)
    for k in v:
        v[k] = np.ascontiguousarray(v[k], dtype=np.int16)
        assert len(v[k]) == n
    _cache[mode] = v
    return v


def layout_b(mode):
    """variant index of each of N_LAYOUT_B channels: the three streams whose fills coincide (base, off0, off1) take half the
    channels, the others share the rest, in a scrambled order"""
    names = list(variants(mode))
    counts = [50, 50, 50] + [0] * (len(names) - 3)
    rest = N_LAYOUT_B - 150
    for i in range(rest):
        counts[3 + i % (len(names) - 3)] += 1
    idx = np.random.default_rng(0xB300).permutation(np.repeat(np.arange(len(names)), counts))
    return names, idx
