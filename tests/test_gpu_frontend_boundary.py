"""GPU checks of the front-end stages' argument checks (down-converter, rate converter, carrier scanner, mode identifier): every
rejected write, device write, read and retune returns JAERO_E_ARG with its exact text, the first check that applies is the one
that fires, a rejected call leaves the stage exactly as it was (its next good write matches a twin that never saw the bad call,
launch counts included), and empty writes describe an empty output (down-converter, rate converter) or change nothing
(scanner, identifier)."""
import ctypes

import numpy as np
import pytest

from conftest import has_cuda

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

E_ARG = -1
HUGE = (1 << 34) + 1


def _jb():
    import jaero_b200
    return jaero_b200


def _rejects(call, text):
    L = _jb().lib()
    rc = call()
    assert (rc, L.jaero_last_error().decode()) == (E_ARG, text)


def _iq(fmt, n, seed):
    rng = np.random.default_rng(seed)
    if fmt == "cu8":
        return rng.integers(0, 256, size=2 * n).astype(np.uint8)
    return rng.integers(-6000, 6000, size=2 * n).astype(np.int16)


def _pcm(C, n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    x = rng.normal(0, 2000, size=(C, n)) + 9000 * np.cos(2 * np.pi * 0.07 * t + np.arange(C)[:, None])
    return np.clip(np.round(x), -32768, 32767).astype(np.int16)


def _vp(x):
    return ctypes.c_void_p(x)


def _check_iq_write_rejections(jb, L, stage, h, dev, host):
    """the argument checks shared by jaero_ddc_* and jaero_scan_* IQ writes, in the order they fire"""
    w, wd = getattr(L, "jaero_%s_write" % stage), getattr(L, "jaero_%s_write_device" % stage)
    p = dev.data_ptr()
    hp = host.ctypes.data_as(ctypes.c_void_p)
    pre = "jaero_%s_write_device: " % stage
    _rejects(lambda: wd(h, _vp(p), 16, 7), pre + "unknown IQ format")
    _rejects(lambda: wd(h, _vp(p + 1), 16, 7), pre + "unknown IQ format")
    _rejects(lambda: wd(h, _vp(p + 1), 0, jb.IQ_CU8), pre + "IQ pointer not aligned to one sample")
    _rejects(lambda: wd(h, _vp(p + 2), 16, jb.IQ_CS16), pre + "IQ pointer not aligned to one sample")
    _rejects(lambda: wd(h, _vp(p + 1), HUGE, jb.IQ_CS16), pre + "IQ pointer not aligned to one sample")
    _rejects(lambda: wd(h, _vp(p), HUGE, jb.IQ_CS16), pre + "too many samples in one write")
    _rejects(lambda: wd(h, _vp(p + 2), HUGE, jb.IQ_CU8), pre + "too many samples in one write")
    pre = "jaero_%s_write: " % stage
    _rejects(lambda: w(h, hp, 16, 2), pre + "unknown IQ format")
    _rejects(lambda: w(h, hp, HUGE, 2), pre + "unknown IQ format")
    _rejects(lambda: w(h, hp, HUGE, jb.IQ_CU8), pre + "too many samples in one write")
    _rejects(lambda: w(h, hp, HUGE, jb.IQ_CS16), pre + "too many samples in one write")


def _check_pcm_write_rejections(L, stage, h, dev, host):
    """the argument checks shared by jaero_resample_* and jaero_ident_* PCM writes, in the order they fire"""
    w, wd = getattr(L, "jaero_%s_write" % stage), getattr(L, "jaero_%s_write_device" % stage)
    p = dev.data_ptr()
    hp = host.ctypes.data_as(ctypes.c_void_p)
    pre = "jaero_%s_write_device: " % stage
    _rejects(lambda: wd(h, _vp(p + 1), 16, 16), pre + "PCM pointer not aligned to one sample")
    _rejects(lambda: wd(h, _vp(p + 1), 0, 0), pre + "PCM pointer not aligned to one sample")
    _rejects(lambda: wd(h, _vp(p + 1), HUGE, 4), pre + "PCM pointer not aligned to one sample")
    _rejects(lambda: wd(h, _vp(p), 16, 15), pre + "channel stride is smaller than n_samples")
    _rejects(lambda: wd(h, _vp(p), HUGE, 4), pre + "channel stride is smaller than n_samples")
    _rejects(lambda: wd(h, _vp(p), HUGE, HUGE), pre + "too many samples in one write")
    pre = "jaero_%s_write: " % stage
    _rejects(lambda: w(h, hp, 16, 15), pre + "channel stride is smaller than n_samples")
    _rejects(lambda: w(h, hp, HUGE, 4), pre + "channel stride is smaller than n_samples")
    _rejects(lambda: w(h, hp, HUGE, HUGE), pre + "too many samples in one write")


def _pcm_state(s):
    _, n, stride = s.output()
    inputs, clipped = s.stats()
    return n, stride, s.read_pcm().tobytes(), inputs, clipped.tobytes(), s.launches


@pytest.mark.parametrize("interpolation,decimation,fs", [(1, 50, 2.4e6), (12, 625, 2.5e6)])
@pytest.mark.parametrize("fmt", ["cu8", "cs16"])
def test_ddc_rejections_leave_the_output_and_the_next_write_unchanged(interpolation, decimation, fs, fmt):
    import torch
    jb = _jb()
    L = jb.lib()
    off, aud = [100e3, -210e3, 333e3], [8000.0, 9000.0, 7000.0]
    a, b = (jb.Ddc(fs, decimation, off, aud, 12000.0, 4000.0, gain=4.0, interpolation=interpolation) for _ in range(2))
    iq = _iq(fmt, 120_003, seed=7)
    cut = 2 * 50_001
    for d in (a, b):
        d.write(iq[:cut], fmt)
    before = _pcm_state(a)
    assert before[0] > 0
    dev = torch.from_numpy(iq[:64].copy()).cuda()
    torch.cuda.synchronize()
    _check_iq_write_rejections(jb, L, "ddc", a.h, dev, iq)
    n = before[0]
    out = np.zeros((3, n), dtype=np.int16)
    got = ctypes.c_size_t(99)
    _rejects(lambda: L.jaero_ddc_read_pcm(a.h, out.ctypes.data_as(ctypes.c_void_p), n - 1, ctypes.byref(got)),
             "jaero_ddc_read_pcm: cap_per_channel is smaller than the last write's output")
    assert got.value == 99
    for ch in (-2, 3, 1000):
        _rejects(lambda: L.jaero_ddc_set_offset(a.h, ch, 0.0), "jaero_ddc_set_offset: bad argument")
        _rejects(lambda: L.jaero_ddc_set_audio_freq(a.h, ch, 8000.0), "jaero_ddc_set_audio_freq: bad argument")
    for hz in (fs / 2, -fs, float("nan"), float("inf")):
        _rejects(lambda: L.jaero_ddc_set_offset(a.h, 1, hz), "jaero_ddc_set_offset: |offset| must not exceed input_rate/2 - bandwidth/2")
    for hz in (6000.0, 0.0, 20000.0, float("nan")):
        _rejects(lambda: L.jaero_ddc_set_audio_freq(a.h, -1, hz), "jaero_ddc_set_audio_freq: the audio passband must lie inside (0, output_rate/2)")
    _rejects(lambda: L.jaero_ddc_set_offset(a.h, 7, float("nan")), "jaero_ddc_set_offset: bad argument")
    assert _pcm_state(a) == before
    # a stream switch away and back queues nothing
    st = torch.cuda.Stream()
    a.set_stream(st.cuda_stream); a.set_stream(0)
    for d in (a, b):
        d.write(iq[cut:], fmt)
    after = _pcm_state(a)
    assert after == _pcm_state(b)
    assert after[0] > 0
    a.close(); b.close()


def test_ddc_and_resampler_empty_writes_describe_an_empty_output():
    import torch
    jb = _jb()
    iq = _iq("cs16", 40_000, seed=3)
    pcm = _pcm(2, 9_000, seed=4)
    dev_iq = torch.from_numpy(iq).cuda()
    dev_pcm = torch.from_numpy(pcm).cuda()
    torch.cuda.synchronize()
    for kind in ("ddc", "resample"):
        if kind == "ddc":
            a, b = (jb.Ddc(2.4e6, 50, [100e3, -50e3], 8000.0, 12000.0, 4000.0) for _ in range(2))
            first = lambda s: s.write(iq[:40_000], "cs16")
            rest = lambda s: s.write(iq[40_000:], "cs16")
            empties = [lambda s: s.write(iq[:0], "cs16"), lambda s: s.write_device(dev_iq.data_ptr(), 0, "cs16"),
                       lambda s: s.write_device(dev_iq.data_ptr(), 0, "cu8")]
        else:
            a, b = (jb.Resampler(44100, 2) for _ in range(2))
            first = lambda s: s.write(pcm[:, :5_000])
            rest = lambda s: s.write(pcm[:, 5_000:])
            empties = [lambda s: s.write(pcm[:, :0]), lambda s: s.write_device(dev_pcm.data_ptr(), 0, 0),
                       lambda s: s.write_device(dev_pcm.data_ptr(), 0, 9_000)]
        for s in (a, b):
            first(s)
        inputs, clipped = a.stats()
        launches = a.launches
        for e in empties:
            e(a)
            _, n, stride = a.output()
            assert (n, stride) == (0, 8), kind
            assert a.read_pcm().shape == (2, 0)
            assert a.stats()[0] == inputs and a.stats()[1].tobytes() == clipped.tobytes()
            assert a.launches == launches
        for s in (a, b):
            rest(s)
        assert _pcm_state(a) == _pcm_state(b), kind
        a.close(); b.close()


def test_resampler_rejections_leave_the_output_and_the_next_write_unchanged():
    import torch
    jb = _jb()
    L = jb.lib()
    C = 3
    pcm = _pcm(C, 30_011, seed=11)
    a, b = jb.Resampler(44100, C), jb.Resampler(44100, C)
    for s in (a, b):
        s.write(pcm[:, :12_345])
    before = _pcm_state(a)
    dev = torch.from_numpy(pcm[:, :64].copy()).cuda()
    torch.cuda.synchronize()
    _check_pcm_write_rejections(L, "resample", a.h, dev, pcm)
    n = before[0]
    out = np.zeros((C, n), dtype=np.int16)
    got = ctypes.c_size_t(99)
    _rejects(lambda: L.jaero_resample_read_pcm(a.h, out.ctypes.data_as(ctypes.c_void_p), n - 1, ctypes.byref(got)),
             "jaero_resample_read_pcm: cap_per_channel is smaller than the last write's output")
    assert got.value == 99
    assert _pcm_state(a) == before
    st = torch.cuda.Stream()
    a.set_stream(st.cuda_stream); a.set_stream(0)
    for s in (a, b):
        s.write(pcm[:, 12_345:])
    assert _pcm_state(a) == _pcm_state(b)
    a.close(); b.close()


def _scan_state(s):
    mean, mx, frames = s.read()
    return mean.tobytes(), mx.tobytes(), frames, s.launches


@pytest.mark.parametrize("fmt", ["cu8", "cs16"])
def test_scanner_rejections_and_empty_writes_change_nothing(fmt):
    import torch
    jb = _jb()
    L = jb.lib()
    nfft = 4096
    a, b = jb.Scanner(2.4e6, nfft), jb.Scanner(2.4e6, nfft)
    iq = _iq(fmt, 40_000, seed=21)
    cut = 2 * 13_333                                                  # leaves a carry of part of a frame
    for s in (a, b):
        s.write(iq[:cut], fmt)
    before = _scan_state(a)
    assert before[2] > 0
    dev = torch.from_numpy(iq[:64].copy()).cuda()
    torch.cuda.synchronize()
    _check_iq_write_rejections(jb, L, "scan", a.h, dev, iq)
    _rejects(lambda: L.jaero_scan_write_device(a.h, _vp(dev.data_ptr()), 0, 7), "jaero_scan_write_device: unknown IQ format")
    a.write(iq[:0], fmt)
    a.write_device(dev.data_ptr(), 0, fmt)
    assert _scan_state(a) == before
    st = torch.cuda.Stream()
    a.set_stream(st.cuda_stream); a.set_stream(0)
    for s in (a, b):
        s.write(iq[cut:], fmt)
    assert _scan_state(a) == _scan_state(b)
    a.close(); b.close()


def _ident_state(s):
    sq, frames = s.read()
    return sq.tobytes(), frames, s.launches


def test_identifier_rejections_empty_and_short_writes():
    import torch
    jb = _jb()
    L = jb.lib()
    C, nfft = 2, 1024
    pcm = _pcm(C, 9_000, seed=31)
    a, b = jb.Identifier(48000, C, nfft=nfft), jb.Identifier(48000, C, nfft=nfft)
    for s in (a, b):
        s.write(pcm[:, :3_000])
    before = _ident_state(a)
    assert before[1] > 0
    dev = torch.from_numpy(pcm[:, :64].copy()).cuda()
    torch.cuda.synchronize()
    _check_pcm_write_rejections(L, "ident", a.h, dev, pcm)
    a.write(pcm[:, :0])
    a.write_device(dev.data_ptr(), 0, 0)
    assert _ident_state(a) == before
    # 3000 samples leave frames 0..3 and a carry from sample 2048; until sample 3072 no frame completes, so these writes only
    # join the carry: nothing is launched and the average stays
    a.write(pcm[:, 3_000:3_030])
    a.write(pcm[:, 3_030:3_060])
    assert _ident_state(a) == before
    b.write(pcm[:, 3_000:3_060])
    assert _ident_state(b) == before
    st = torch.cuda.Stream()
    a.set_stream(st.cuda_stream); a.set_stream(0)
    for s in (a, b):
        s.write(pcm[:, 3_060:])
    assert _ident_state(a) == _ident_state(b)
    assert _ident_state(a)[1] > before[1]
    a.close(); b.close()
