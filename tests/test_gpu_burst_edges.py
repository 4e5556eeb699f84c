"""Burst demodulators (MSK 1200, MSK 600, burst OQPSK 10500) at every write size, internal-chunk edge and channel layout the
device path distinguishes (pytest -m gpu, on an H100).

jaero_burst_write_device cuts a write into internal chunks of 16384 samples, runs the Hilbert FFT-FIR in stream-aligned
blocks of 6145, records at most 8 trident-buffer fills per channel and chunk, and runs the trident FFTs 128 events per
launch. The streams of tests/burst_edge_streams.py put fills on the first and last samples of chunks, writes and Hilbert
blocks; 4800-sample writes are checked against the restated oracle, and every other way of cutting the same stream, the
300-channel layout and the pitched device entry point must then give the same soft bits and state bit for bit: nothing in
the burst path depends on how the stream is cut or where a channel sits."""
import multiprocessing as mp
import os

import numpy as np
import pytest

import burst_edge_streams as S
from conftest import has_cuda
from oracle import restated

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]
STATE_TOL = 1e-6
MODES = list(S.MODES)


def _batch(mode, n_channels, sql=False):
    import jaero_b200 as jb
    m = S.MODES[mode]
    if m["kind"] == "burst_oqpsk":
        return jb.BurstOqpskBatch(n_channels, sql=sql, **m["kw"])
    return jb.BurstMskBatch(n_channels, **m["kw"])


def _run(mode, pcm2, writes, sql=False, device=None):
    """soft bits (drained after every write) and status of every channel. device: a CUDA int16 tensor [channels][pitch] holding
    the stream (fed through write_device) instead of the host array pcm2."""
    C = pcm2.shape[0] if device is None else device.shape[0]
    b = _batch(mode, C, sql)
    acc = [[] for _ in range(C)]
    a = 0
    for w in writes:
        if device is None:
            b.write(pcm2[:, a:a + w])
        else:
            b.write_device(device.data_ptr() + 2 * a, w, device.shape[1])
        a += w
        for c, s in enumerate(b.read_softbits()):
            acc[c].append(s)
    st = b.status()
    b.close()
    return [np.concatenate(x) for x in acc], st


def _oracle_jobs(mode, streams, writes, sql=False):
    m = S.MODES[mode]
    kw = dict(m["kw"], sql=True) if sql else m["kw"]
    with mp.get_context("spawn").Pool(min(len(streams), os.cpu_count() or 1)) as pool:
        return pool.map(restated.run_demod_job, [(m["kind"], kw, x, writes) for x in streams])


def _assert_oracle(sg, stg, ref, what):
    """the burst-parity criteria: markers and hard decisions identical, soft values within 1 LSB, loop state within 1e-6"""
    so, os_, eb = ref
    assert len(so) == len(sg), what
    assert np.array_equal(np.nonzero(so < 0)[0], np.nonzero(sg < 0)[0]), what
    assert np.array_equal(so >= 128, sg >= 128), what
    assert np.abs(so.astype(int) - sg.astype(int)).max(initial=0) <= 1, what
    for k in ("mixer2_freq", "vol_gain", "rotator_freq", "mse"):
        assert abs(stg[k] - os_[k]) <= STATE_TOL * max(abs(os_[k]), 1e-9), (what, k, stg[k], os_[k])
    for k in ("n_sig_true", "n_sig_false", "cntr", "startstop"):
        assert stg[k] == os_[k], (what, k)
    assert stg["n_ebno_emits"] == len(eb), what


def _assert_same(soft, st, soft_ref, st_ref, what):
    for c in range(len(soft)):
        assert np.array_equal(soft[c], soft_ref[c]), (what, c)
        assert st[c] == st_ref[c], (what, c)


_P1 = {}


def _p1(mode):
    """layout (a), one channel per stream variant, 4800-sample writes: (names, streams, soft, status, oracle results)"""
    if mode not in _P1:
        v = S.variants(mode)
        names = list(v)
        pcm2 = np.stack([v[k] for k in names])
        soft, st = _run(mode, pcm2, S.cycle_writes(S.P1, pcm2.shape[1]))
        _P1[mode] = (names, pcm2, soft, st, _oracle_jobs(mode, list(pcm2), 4800))
    return _P1[mode]


@pytest.mark.parametrize("mode", MODES)
def test_p1_matches_oracle(mode):
    names, pcm2, soft, st, ref = _p1(mode)
    for c, k in enumerate(names):
        _assert_oracle(soft[c], st[c], ref[c], (mode, k))
    assert all((s < 0).any() for s in soft)                        # every stream acquires at least one burst


def _fills(mode):
    return np.concatenate([S.oracle_fills(mode, x)[0] for x in S.variants(mode).values()])


@pytest.mark.parametrize("pattern", ["P2", "P3_first", "P3_last", "P4"])
@pytest.mark.parametrize("mode", MODES)
def test_write_patterns_bitwise(mode, pattern):
    """P2: a cycle of 1..16385-sample writes; P3: boundaries on every fill, so that each one completes on the first (P3_first)
    or the last (P3_last) sample of a write; P4: 40000..65536-sample writes of several internal chunks each"""
    names, pcm2, soft1, st1, _ = _p1(mode)
    n = pcm2.shape[1]
    if pattern == "P2":
        writes = S.cycle_writes(S.P2, n)
    elif pattern == "P4":
        writes = S.cycle_writes(S.P4, n)
    else:
        f = _fills(mode)
        writes = S.writes_at(f if pattern == "P3_first" else f + 1, n)
        starts = set(np.cumsum([0] + writes[:-1]).tolist())
        assert all((int(t) if pattern == "P3_first" else int(t) + 1) in starts for t in f if t + 1 < n)
    assert sum(writes) == n and max(writes) <= 65536
    soft, st = _run(mode, pcm2, writes)
    _assert_same(soft, st, soft1, st1, (mode, pattern))


@pytest.mark.parametrize("mode", MODES)
def test_300_channels(mode):
    """300 channels in a scrambled variant order: several front-kernel CTAs with a ragged tail, and more than 128 trident events
    in one internal chunk. Every channel equals its variant's single-CTA result bit for bit (which the oracle checks), with
    4800-sample writes and with P4 writes."""
    import torch
    names, pcm2, soft1, st1, ref = _p1(mode)
    _, idx = S.layout_b(mode)
    dev = torch.from_numpy(pcm2).cuda()[torch.from_numpy(idx).cuda()].contiguous()
    torch.cuda.synchronize()
    n = pcm2.shape[1]
    for pattern in (S.P1, S.P4):
        soft, st = _run(mode, None, S.cycle_writes(pattern, n), device=dev)
        for c, v in enumerate(idx):
            assert np.array_equal(soft[c], soft1[v]), (mode, pattern[0], c, names[v])
            assert st[c] == st1[v], (mode, pattern[0], c, names[v])
    for v in range(len(names)):
        c = int(np.nonzero(idx == v)[0][-1])
        _assert_oracle(soft[c], st[c], ref[v], (mode, names[v], c))
    del dev


@pytest.mark.parametrize("mode", MODES)
def test_write_device_with_row_pitch(mode):
    """write_device from a CUDA tensor whose rows are 40 samples longer than the stream, one 4800-sample window at a time"""
    import torch
    names, pcm2, soft1, st1, _ = _p1(mode)
    n = pcm2.shape[1]
    dev = torch.zeros((pcm2.shape[0], n + 40), dtype=torch.int16, device="cuda")
    dev[:, :n] = torch.from_numpy(pcm2).cuda()
    dev[:, n:] = 12345
    torch.cuda.synchronize()
    soft, st = _run(mode, None, S.cycle_writes(S.P1, n), device=dev)
    _assert_same(soft, st, soft1, st1, (mode, "write_device"))


@pytest.mark.parametrize("pattern", ["P2", "P4"])
def test_oqpsk_squelch_matches_oracle(pattern):
    """burst OQPSK with sql on: a soft-bit vector passes if mse or the mse latched at the start of the WRITE is below the
    threshold. The first write is longer than one internal chunk, so latching per internal chunk would differ."""
    names, pcm2, _, _, ref1 = _p1("oqpsk")
    n = pcm2.shape[1]
    writes = [20000] + S.cycle_writes(S.P2, n - 20000) if pattern == "P2" else S.cycle_writes(S.P4, n)
    assert writes[0] > S.CHUNK
    soft, st = _run("oqpsk", pcm2, writes, sql=True)
    ref = _oracle_jobs("oqpsk", list(pcm2), writes, sql=True)
    for c, k in enumerate(names):
        _assert_oracle(soft[c], st[c], ref[c], ("sql", pattern, k))
    assert sum(len(r[0]) for r in ref) < sum(len(r[0]) for r in ref1)        # the squelch withheld something
