"""SHA-256 digests of what the three frame layers (P-channel, C-channel, R/T) return through the C ABI: every record read (P
signal units with their CRC flag, index and frame number; C-channel signal units and voice bytes; R/T packet headers and
payloads), the per-read counts, the layer's stats and, where a demodulator batch is attached, the DCD the layer wrote back
into the demodulator's status.

    python tools/make_frame_digests.py        # writes tests/golden/frame_digests.json (needs a GPU)

P-channel (10500, 1200, 600 bps) and C-channel (8400 bps) run three channels: the committed excerpt, the excerpt at 2/3
amplitude and seeded noise that never syncs. Each runs two ways:
  - batch: write_batch (the stream cut at every estimator trigger, SignalStatus(false) events handed over as LostSignal at
    their soft-bit positions) with tick() and one lost_signal(channel=1) at fixed writes;
  - host: process_softbits on the demodulator's soft bits, cut per channel at 1, 31, 32, 33 values and at the frame block
    length -1, 0, +1, so the cuts cross the edges between the P-channel kernel's 32-bit fast path and its bit-serial path;
    tick() and one lost_signal(channel=0) at fixed calls.
R/T runs the three burst excerpts on three channels (the excerpt, rolled, at 3/5 amplitude) through process_burst with
vector mode off and on, and process() on the burst demodulator's soft bits (with their -1 start-of-burst markers) under the
same cuts, with tick() at fixed calls.
tests/test_gpu_frame_digest.py recomputes the digests and compares them."""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "frame_digests.json")

P_RATES = {"10500": ("oqpsk_10500", 78 * 64), "1200": ("msk_1200", 9 * 64), "600": ("msk_600", 6 * 64)}
C_BLOCK = 4096                      # C-channel frame bits
RT_EXCERPTS = ["burst_msk_1200_a", "burst_msk_1200_b", "burst_oqpsk_10500"]
CHUNK = 4800


def _cuts(block):
    return [1, 31, 32, 33, block - 1, block, block + 1]


class _Digest:
    """named SHA-256 streams; every update is length-prefixed so that moving bytes between reads changes the digest"""
    def __init__(self, *names):
        self.h = {n: hashlib.sha256() for n in names}

    def add(self, name, arr):
        b = np.ascontiguousarray(arr).tobytes()
        self.h[name].update(len(b).to_bytes(8, "little") + b)

    def result(self):
        return {n: h.hexdigest() for n, h in self.h.items()}


def _golden_kw(name):
    with open(os.path.join(ROOT, "tests", "golden", "expected_outputs.json")) as fh:
        return json.load(fh)[name]["kw"]


def _three_channels(pcm, seed):
    noise = np.random.default_rng(seed).integers(-2000, 2000, size=len(pcm)).astype(np.int16)
    return np.stack([pcm, (pcm.astype(np.int32) * 2 // 3).astype(np.int16), noise])


def _demod_soft(jb, kind, kw, pcm2):
    b = jb.DemodBatch(kind, pcm2.shape[0], **kw)
    acc = [[] for _ in range(pcm2.shape[0])]
    for a in range(0, pcm2.shape[1], CHUNK):
        b.write(pcm2[:, a:a + CHUNK])
        for c, s in enumerate(b.read_softbits()):
            acc[c].append(s)
    b.close()
    return [np.concatenate(x) for x in acc]


def _host_feed(layer_process, soft, block, on_call):
    """feed each channel's soft bits in pieces of _cuts(block), channel c starting c places into the cycle"""
    cuts = _cuts(block)
    pos = [0] * len(soft)
    k = 0
    while any(p < len(s) for p, s in zip(pos, soft)):
        pieces = []
        for c, s in enumerate(soft):
            n = cuts[(k + 2 * c) % len(cuts)]
            pieces.append(s[pos[c]:pos[c] + n]); pos[c] += len(pieces[-1])
        layer_process(pieces)
        on_call(k)
        k += 1


def _read_p(d, pc):
    out, counts = pc.read_sus_raw()
    d.add("counts", counts)
    for c in range(pc.n):
        d.add("records", out[c, :counts[c]])


def _read_c(d, cc):
    fr = cc.read_frames()
    d.add("counts", np.array([len(f[3]) for f in fr], dtype=np.int32))
    for su, ok, voice, frame in fr:
        d.add("records", su); d.add("records", ok); d.add("records", voice); d.add("records", frame)


def _read_rt(d, rt):
    pk = rt.read_packets()
    d.add("counts", np.array([len(p) for p in pk], dtype=np.int32))
    for p in pk:
        for q in p:
            d.add("records", np.array([q["type"], q["nsus"], q["start_bit"], len(q["bytes"])], dtype=np.int32))
            d.add("records", q["bytes"])


def _run_continuous(layer, rate, path):
    import jaero_b200 as jb
    from conftest import load_excerpt
    if layer == "p":
        excerpt, block = P_RATES[rate]
    else:
        excerpt, block = "oqpsk_8400", C_BLOCK
    kw = dict(_golden_kw(excerpt))
    kind = "oqpsk" if excerpt.startswith("oqpsk") else "msk"
    pcm2 = _three_channels(load_excerpt(excerpt), seed=int(kw["fb"]))
    make = (lambda: jb.PChannelBatch(3, kw["fb"])) if layer == "p" else (lambda: jb.CChannelBatch(3))
    read = _read_p if layer == "p" else _read_c
    d = _Digest("records", "counts", "stats", *(["dcd"] if path == "batch" else []))
    fl = make()
    if path == "batch":
        b = jb.DemodBatch(kind, 3, **kw)
        for k, a in enumerate(range(0, pcm2.shape[1], CHUNK)):
            fl.write_batch(b, pcm2[:, a:a + CHUNK])
            if k % 10 == 9:
                fl.tick(b)
            if k == 23:
                fl.lost_signal(b, channel=1)
            if k % 3 == 2:
                read(d, fl)
            d.add("dcd", np.array([s["dcd"] for s in b.status()], dtype=np.int32))
        b.close()
    else:
        soft = _demod_soft(jb, kind, kw, pcm2)
        process = fl.process_softbits if layer == "p" else fl.process

        def on_call(k):
            if k % 17 == 16:
                fl.tick()
            if k == 20:
                fl.lost_signal(channel=0)
            if k % 5 == 4:
                read(d, fl)
        _host_feed(process, soft, block, on_call)
    read(d, fl)
    dcd, tot, ok = fl.stats()
    d.add("stats", dcd); d.add("stats", tot); d.add("stats", ok)
    fl.close()
    assert tot[2] == 0 and tot[0] > 0                                 # the noise channel never completes a frame; the excerpt does
    return d.result()


def _run_rt(excerpt, path):
    import jaero_b200 as jb
    from conftest import load_excerpt
    with open(os.path.join(ROOT, "tests", "golden", "expected_outputs.json")) as fh:
        case = json.load(fh)[excerpt]
    pcm = load_excerpt(excerpt)
    pcm2 = np.stack([pcm, np.roll(pcm, 7001), (pcm.astype(np.int32) * 3 // 5).astype(np.int16)])
    oq = case["kind"] == "burst_oqpsk"
    b = (jb.BurstOqpskBatch if oq else jb.BurstMskBatch)(3, **case["kw"])
    rt = jb.RTChannelBatch(3, case["kw"]["fb"])
    d = _Digest("records", "counts", "stats")
    chunk = case["chunk"]
    if path in ("burst", "burst_vec"):
        rt.set_vector_mode(path == "burst_vec")
        for k, a in enumerate(range(0, pcm2.shape[1], chunk)):
            b.write(pcm2[:, a:a + chunk])
            rt.process_burst(b)
            if k % 10 == 9:
                rt.tick()
            if k % 3 == 2:
                _read_rt(d, rt)
    else:
        acc = [[] for _ in range(3)]
        for a in range(0, pcm2.shape[1], chunk):
            b.write(pcm2[:, a:a + chunk])
            for c, s in enumerate(b.read_softbits()):
                acc[c].append(s)
        soft = [np.concatenate(x) for x in acc]
        assert all((s < 0).any() for s in soft)                       # the start-of-burst markers are in the stream

        def on_call(k):
            if k % 17 == 16:
                rt.tick()
            if k % 5 == 4:
                _read_rt(d, rt)
        _host_feed(rt.process, soft, 64 * 5, on_call)
    b.close()
    _read_rt(d, rt)
    for s in rt.stats():
        d.add("stats", s)
    rt.close()
    return d.result()


def cases():
    return (["p%s_%s" % (r, p) for r in P_RATES for p in ("batch", "host")] + ["c8400_batch", "c8400_host"]
            + ["rt_%s_%s" % (e, p) for e in RT_EXCERPTS for p in ("burst", "burst_vec", "host")])


def run_case(name):
    """-> dict of digests: records, counts, stats (and dcd, the demodulator's DCD, for the batch paths)"""
    if name.startswith("rt_"):
        excerpt, path = name[3:].rsplit("_", 1) if not name.endswith("burst_vec") else (name[3:-10], "burst_vec")
        return _run_rt(excerpt, path)
    head, path = name.split("_")
    return _run_continuous(head[0], head[1:], path)


if __name__ == "__main__":
    out = {name: run_case(name) for name in cases()}
    with open(OUT, "w") as fh:
        json.dump(out, fh, indent=1, sort_keys=True)
        fh.write("\n")
    print("wrote %s (%d cases)" % (OUT, len(out)))
