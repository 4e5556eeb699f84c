"""GPU checks of the PCM rate converter (jaero_b200.Resampler, include/jaero_b200.h jaero_resample_*): every output sample and
clipped count against the float64 polyphase reference (tests/resample_reference.py) for nine rate pairs at 1, 33 and 300
channels, independence of how the stream is cut into writes, host and device writes with a channel stride, and the reference's
own 44.1 kHz recordings through Resampler -> DemodBatch -> PChannelBatch and Resampler -> BurstOqpskBatch -> RTChannelBatch
against tests/golden/native_rate_outputs.json."""
import hashlib
import json
import os

import numpy as np
import pytest

import resample_reference as rr
from test_gpu_ddc import _assert_matches

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PAIRS = [(44100, 48000), (32000, 48000), (22050, 48000), (11025, 48000), (8000, 48000), (96000, 48000), (192000, 48000),
         (44100, 24000), (48000, 12000)]


def _plan(a, b):
    import jaero_b200
    return jaero_b200.resample_plan(a, b, 0.45 * min(a, b))


def _input(C, n, fs, seed):
    """random int16 on most channels; every third channel a full-scale tone, driven past full scale so that it clips at the
    input and overshoots after filtering"""
    rng = np.random.default_rng(seed)
    x = rng.integers(-32768, 32768, size=(C, n)).astype(np.int16)
    t = np.arange(n)
    for c in range(0, C, 3):
        f = rng.uniform(50.0, 0.4 * min(fs, 12000))
        x[c] = np.clip(np.round(1.3 * 32767 * np.sin(2 * np.pi * f / fs * t + c)), -32768, 32767).astype(np.int16)
    return x


@pytest.mark.parametrize("a,b", PAIRS)
@pytest.mark.parametrize("C", [1, 33, 300])
def test_resampler_equals_reference(a, b, C):
    import jaero_b200
    p = _plan(a, b)
    L, M = p["L"], p["M"]
    n_out = min(200_000, max(8000, 3_000_000 // C))
    n = n_out * M // L + 7
    x = _input(C, n, a, seed=a + b + C)
    r = jaero_b200.Resampler(a, C, output_rate=b)
    assert (r.plan["L"], r.plan["M"], r.plan["K"]) == (L, M, p["K"])
    cut = n * 3 // 7
    r.write(x[:, :cut]); first = r.read_pcm()
    r.write(x[:, cut:]); second = r.read_pcm()
    inputs, clipped = r.stats()
    r.close()
    got = np.concatenate([first, second], axis=1)
    _, val, clip_ref = rr.resample_reference(x, p["h"], L, M)
    assert inputs == n and first.shape[1] == rr.n_outputs(cut, L, M) and got.shape == (C, rr.n_outputs(n, L, M))
    _assert_matches(got, val)
    np.testing.assert_array_equal(clipped, clip_ref)
    assert clip_ref[0] > 0                                       # channel 0 is a tone that clips


@pytest.mark.parametrize("a,b", [(44100, 48000), (11025, 48000), (96000, 48000)])
def test_output_does_not_depend_on_how_the_stream_is_cut(a, b):
    import torch
    import jaero_b200
    p = _plan(a, b)
    L, M = p["L"], p["M"]
    C, n = 40, 60_011
    x = _input(C, n, a, seed=5)
    r = jaero_b200.Resampler(a, C, output_rate=b)
    r.write(x)
    whole = r.read_pcm()
    r.close()
    assert whole.shape == (C, rr.n_outputs(n, L, M))
    rng = np.random.default_rng(9)
    pieces = [1, 0, 1, 1, L, M - 1, M, M + 1, 0, 7, 101, 997, 2, 3, 4410, 13_001]
    cuts = []
    while sum(cuts) < n:
        cuts.append(min(int(pieces[len(cuts)] if len(cuts) < len(pieces) else rng.choice(pieces)), n - sum(cuts)))
    dev = torch.from_numpy(x).cuda()
    torch.cuda.synchronize()
    for path in ("host", "device"):
        r = jaero_b200.Resampler(a, C, output_rate=b)
        parts, s0 = [], 0
        for c in cuts:
            if path == "host":
                r.write(x[:, s0:s0 + c])
            else:
                r.write_device(dev.data_ptr() + 2 * s0, c, n)
            part = r.read_pcm()
            assert part.shape == (C, rr.n_outputs(s0 + c, L, M) - rr.n_outputs(s0, L, M))
            parts.append(part)
            s0 += c
        launches = r.launches
        r.close()
        assert launches <= 3 * sum(1 for c in cuts if c)          # an empty write queues nothing
        got = np.concatenate(parts, axis=1)
        assert got.tobytes() == whole.tobytes(), path


def test_host_and_device_writes_honour_the_channel_stride():
    import torch
    import jaero_b200
    C, n, pitch = 37, 30_001, 30_001 + 4099
    big = _input(C, pitch, 44100, seed=17)
    x = big[:, :n]                                               # a strided view: row pitch 34100 samples
    p = _plan(44100, 48000)
    _, val, _ = rr.resample_reference(np.ascontiguousarray(x), p["h"], p["L"], p["M"])
    outs = []
    r = jaero_b200.Resampler(44100, C)
    r.write(x); outs.append(r.read_pcm()); r.close()
    dev = torch.from_numpy(big).cuda()
    torch.cuda.synchronize()
    r = jaero_b200.Resampler(44100, C)
    r.write_device(dev.data_ptr(), n, pitch); outs.append(r.read_pcm())
    ptr, m, stride = r.output()
    assert m == rr.n_outputs(n, p["L"], p["M"]) and stride % 8 == 0 and ptr % 16 == 0
    with pytest.raises(jaero_b200.JaeroError, match="stride"):
        r.write_device(dev.data_ptr(), n, n - 1)
    r.close()
    assert outs[0].tobytes() == outs[1].tobytes()
    _assert_matches(outs[0], val)


def _excerpt(name):
    return np.load(os.path.join(GOLD, name + "_excerpt.npz"))["pcm"]


def test_44k1_continuous_recording_through_resampler_demod_and_pchannel():
    """the reference's 10.5k_sample.ogg at its own 44.1 kHz: Resampler -> DemodBatch -> PChannelBatch on one CUDA stream, no host
    copy of the PCM, decodes the CRC-valid signal units the oracle decodes from the reference resampler's output"""
    import torch
    import jaero_b200
    want = json.load(open(os.path.join(GOLD, "native_rate_outputs.json")))["oqpsk_10500_44k1"]
    x = _excerpt("oqpsk_10500_44k1")
    kw = dict(want["kw"])
    step = want["chunk_in"]
    stream = torch.cuda.Stream()
    dev = torch.from_numpy(x).cuda()
    torch.cuda.synchronize()
    r = jaero_b200.Resampler(44100, 1)
    b = jaero_b200.DemodBatch("oqpsk", 1, **kw)
    pc = jaero_b200.PChannelBatch(1, kw["fb"])
    r.set_stream(stream.cuda_stream); b.set_stream(stream.cuda_stream)
    sus, produced = [], 0
    for k, a in enumerate(range(0, len(x), step)):
        r.write_device(dev.data_ptr() + 2 * a, min(step, len(x) - a), len(x))
        ptr, m, stride = r.output()
        b.write_device(ptr, m, stride)
        pc.process_batch(b)
        if (produced + m) % 48000 < m:
            pc.tick(b)
        produced += m
        if k % 10 == 9:
            sus.append(pc.read_sus()[0])
    sus.append(pc.read_sus()[0])
    _, clipped = r.stats()
    r.close(); b.close(); pc.close()
    assert produced == want["resampled_samples"] and clipped[0] == want["resampled_clipped"]
    got = [bytes(s).hex() for r in sus for s, o in zip(r[0], r[1]) if o]
    assert len(got) == want["n_su_crc_ok"]
    assert hashlib.sha256(json.dumps(got).encode()).hexdigest() == want["su_crc_ok_sha256"]


def test_44k1_burst_recording_through_resampler_burst_demod_and_rt_channel():
    """the reference's 10.5k_burst_sample.mp3 at its own 44.1 kHz: Resampler -> BurstOqpskBatch -> RTChannelBatch.process_burst
    decodes the R/T packets the oracle decodes from the reference resampler's output"""
    import torch
    import jaero_b200
    want = json.load(open(os.path.join(GOLD, "native_rate_outputs.json")))["burst_oqpsk_10500_44k1"]
    x = _excerpt("burst_oqpsk_10500_44k1")
    kw = dict(want["kw"])
    step = want["chunk_in"]
    dev = torch.from_numpy(x).cuda()
    torch.cuda.synchronize()
    r = jaero_b200.Resampler(44100, 1)
    b = jaero_b200.BurstOqpskBatch(1, **kw)
    rt = jaero_b200.RTChannelBatch(1, kw["fb"])
    got, produced = [], 0
    for k, a in enumerate(range(0, len(x), step)):
        r.write_device(dev.data_ptr() + 2 * a, min(step, len(x) - a), len(x))
        ptr, m, stride = r.output()
        r.read_pcm()                                             # the burst batch runs on its own stream: the PCM must be complete
        b.write_device(ptr, m, stride)
        rt.process_burst(b)
        b.sync()                                                 # and read before the next write replaces it
        if k % 10 == 9:
            rt.tick()
        produced += m
        got += rt.read_packets()[0]
    r.close(); b.close(); rt.close()
    assert produced == want["resampled_samples"]
    packets = [dict(type=q["type"], nsus=q["nsus"], n_bytes=int(len(q["bytes"])), sha256=hashlib.sha256(q["bytes"].tobytes()).hexdigest())
               for q in got]
    assert packets == want["rt_packets"]
