"""The continuous demodulators' run-time controls and write paths on the GPU (pytest -m gpu, on an H100), against the
restated oracle (tests/test_demod_controls_cpu.py pins that oracle to the reference's own slots).

- jaero_batch_set_center_freq / set_afc / set_sql / set_cpu_reduce under the schedules of tests/control_schedules.py on
  every kernel variant (10.5k pipelined, 8400 with the pre-filter, 8000 single-warp, MSK 600, MSK 1200) at 1, 33 and 300
  channels, batch-wide and on single channels (also with the 10.5k seating permuted and on a batch created with CPU-reduce);
- writes that end on, one before and one after an estimator trigger sample, on a pre-filter block edge, and of one sample;
- device writes from unaligned pointers and odd strides, host writes whose row stride exceeds the write;
- PeakVolume of every write, from page-locked host memory (sliced asynchronous copies), short writes and device memory.

Parity is the rule of tests/test_gpu_parity.py: hard decisions identical, soft values within 1 LSB, loop state within 1e-6."""
import ctypes
import functools
import multiprocessing as mp
import os

import numpy as np
import pytest

import control_schedules as cs
from conftest import has_cuda, load_excerpt
from oracle import restated

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]
STATE_TOL = 1e-6
FS = 48000


# kernel variant -> (kind, settings, seconds to lock, stream loader)
VARIANTS = {
    "oqpsk_10500": cs.RECORDINGS["oqpsk_10500"][:3] + (lambda: load_excerpt("oqpsk_10500"),),
    "oqpsk_8400": cs.RECORDINGS["oqpsk_8400"][:3] + (lambda: load_excerpt("oqpsk_8400"),),
    "oqpsk_8000": cs.SYNTHETIC["oqpsk_8000"] + (lambda: cs.synthetic_stream("oqpsk_8000"),),
    "msk_600": cs.RECORDINGS["msk_600"][:3] + (lambda: load_excerpt("msk_600"),),
    "msk_1200": cs.RECORDINGS["msk_1200"][:3] + (lambda: load_excerpt("msk_1200"),),
}


@functools.lru_cache(maxsize=None)
def _streams(variant):
    """three different streams of one signal: the recording, scaled by 2/3, and delayed by 777 samples"""
    pcm = VARIANTS[variant][3]()
    return np.stack([pcm, (pcm.astype(np.int32) * 2 // 3).astype(np.int16), np.roll(pcm, 777)])


def _gpu_kw(kw):
    g = {k: v for k, v in kw.items() if k != "cpureduce"}
    if kw.get("cpureduce"):
        g["cpu_reduce"] = True
    return g


def _oracle(jobs):
    """restated.run_demod_job over a process pool: jobs [(kind, kw, pcm, chunk, events)] -> [(soft, state, cfe)]"""
    with mp.get_context("spawn").Pool(min(len(jobs), os.cpu_count() or 1)) as pool:
        return pool.map(restated.run_demod_job, jobs)


def _assert_parity(soft_g, st_g, ref, what=""):
    soft_o, st_o = ref[0], ref[1]
    assert len(soft_g) == len(soft_o), (what, len(soft_g), len(soft_o))
    assert np.array_equal(soft_g >= 128, soft_o >= 128), what
    assert np.abs(soft_g.astype(int) - soft_o.astype(int)).max(initial=0) <= 1, what
    for k, v in st_o.items():
        if k in st_g and k not in ("n_sig_true", "n_sig_false"):
            assert abs(st_g[k] - v) <= STATE_TOL * max(abs(v), 1e-9) + 1e-12, (what, k, st_g[k], v)
    assert st_g["n_sig_true"] == st_o["n_sig_true"] and st_g["n_sig_false"] == st_o["n_sig_false"], what


def _run_gpu(kind, kw, pcm2, chunk, events=(), channel_events=None, freq_center=None, before_write=None):
    """one DemodBatch over pcm2 [C, n], written as restated.write_plan cuts it; events apply to every channel,
    channel_events {channel: events} to one channel each (set_center_freq / set_dcd with channel=k)"""
    import jaero_b200 as jb
    C = pcm2.shape[0]
    kwg = _gpu_kw(kw)
    if freq_center is not None:
        kwg["freq_center"] = freq_center
    b = jb.DemodBatch(kind, C, **kwg)
    per = {}
    for a, calls in events:
        per.setdefault(a, []).extend((c, -1) for c in calls)
    for ch, evs in (channel_events or {}).items():
        for a, calls in evs:
            per.setdefault(a, []).extend((c, ch) for c in calls)
    acc = [[] for _ in range(C)]
    for k, (a, n, _) in enumerate(restated.write_plan(pcm2.shape[1], chunk, [(a, []) for a in per])):
        for (name, *args), ch in per.get(a, []):
            if ch >= 0:
                getattr(b, name)(*args, channel=ch)
            else:
                getattr(b, name)(*args)
        if before_write:
            before_write(b, k)
        b.write(pcm2[:, a:a + n])
        for c, s in enumerate(b.read_softbits()):
            acc[c].append(s)
    st = b.status()
    b.close()
    return [np.concatenate(x) for x in acc], st


@functools.lru_cache(maxsize=None)
def _schedule_refs(variant):
    kind, kw, t_lock, _ = VARIANTS[variant]
    x = _streams(variant)
    ev = cs.events(cs.schedule(kind, kw, x.shape[1], t_lock))
    return ev, _oracle([(kind, kw, x[s], 4800, ev) for s in range(3)])


@pytest.mark.parametrize("C", [1, 33, 300])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_control_schedule_on_every_kernel(variant, C):
    """Every centre-change branch, AFC / squelch / CPU-reduce toggle and DCD call of the schedule, made batch-wide between
    writes, on every kernel variant: each channel equals the oracle run of its stream under the same calls."""
    kind, kw, _, _ = VARIANTS[variant]
    ev, refs = _schedule_refs(variant)
    x = _streams(variant)
    idx = np.arange(C) % 3
    soft, st = _run_gpu(kind, kw, np.ascontiguousarray(x[idx]), 4800, ev)
    for c in range(C):
        _assert_parity(soft[c], st[c], refs[idx[c]], (variant, c))
    assert len(soft[0]) > 5000


def _single_channel_events(kind, kw, n, t_lock):
    """events for single channels: a change inside the window, a jump far off the carrier and back, and the low clamp, each
    in the middle of an epoch or at its edge"""
    T = cs.trigger_every(kw)
    fc0, lbw = float(kw["freq_center"]), float(kw["lockingbw"])
    k = int(t_lock * FS) // T + 3
    return {
        3: [(k * T + T // 2, [("set_center_freq", fc0 + 17.0)])],
        17: [((k + 4) * T - 2, [("set_center_freq", fc0 + 1.25 * lbw)]), ((k + 12) * T - 1, [("set_center_freq", fc0)])],
        32: [((k + 2) * T + 1, [("set_center_freq", 1.0)]), ((k + 20) * T, [("set_center_freq", fc0 - 20.0)])],
        # created at -100 Hz (a centre of 0 Hz, far off the carrier): brought onto the carrier in the middle of the first epoch,
        # before the estimator has seen a ring of real samples (see test_zero_hz_centre_estimate_is_the_oracle_s_or_its_mirror)
        6: [(T // 2, [("set_center_freq", fc0)])],
    }


@pytest.mark.parametrize("variant,mode", [("oqpsk_10500", "plain"), ("oqpsk_10500", "regrouped"), ("oqpsk_10500", "cpu_reduce_created"),
                                          ("oqpsk_8400", "plain"), ("oqpsk_8000", "plain"), ("msk_600", "plain"), ("msk_1200", "plain")])
def test_single_channel_centre_changes(variant, mode):
    """set_center_freq(hz, channel=k) re-centres channel k alone (and empties only its estimator ring): the other channels
    equal their oracle runs without the change. Channels are also created at their own centres, some beyond the create-time
    clamp. At 10.5k the seating is permuted before the changes, so that seat and channel differ; and a batch created with
    CPU-reduce (which has no seating table) is switched to the full-rate estimator half way."""
    kind, kw, t_lock, _ = VARIANTS[variant]
    kw = dict(kw)
    x = _streams(variant)[:, :FS * 8]
    n, C = x.shape[1], 33
    idx = np.arange(C) % 3
    fc0 = float(kw["freq_center"])
    fcs = np.full(C, fc0)
    fcs[5], fcs[6], fcs[7], fcs[8] = 30000.0, -100.0, fc0 + 23.0, fc0 - 31.0          # beyond both create-time clamps, and off the carrier
    common = []
    if mode == "cpu_reduce_created":
        kw["cpureduce"] = True
        common = [(FS * 4 + 1234, [("set_cpu_reduce", 0)])]
    if kind == "msk":
        common = [(int(t_lock * FS), [("set_dcd", 1)])] + common
    chan = _single_channel_events(kind, kw, n, t_lock)
    # every channel's oracle is fed the writes the batch gets (cut at every channel's events): the 8400 bps pre-filter and its
    # mixer follow the write boundaries (oqpskdemodulator.cpp:343-381,608), so its output depends on where writes end
    writes = [m for _, m, _ in restated.write_plan(n, 4800, common + [e for evs in chan.values() for e in evs])]
    jobs, key = [], {}
    for c in range(C):
        k = (idx[c], fcs[c], c if c in chan else -1)
        if k not in key:
            key[k] = len(jobs)
            evs = sorted(common + chan.get(c, []), key=lambda e: e[0])
            jobs.append((kind, dict(kw, freq_center=float(fcs[c])), x[idx[c]], writes, evs))
    refs = _oracle(jobs)
    perm = np.random.default_rng(5).permutation(C)

    def regroup(b, k):
        if mode == "regrouped" and k == 3:
            b.regroup(perm)
    soft, st = _run_gpu(kind, kw, np.ascontiguousarray(x[idx]), 4800, common, chan, freq_center=fcs, before_write=regroup)
    for c in range(C):
        _assert_parity(soft[c], st[c], refs[key[(idx[c], fcs[c], c if c in chan else -1)]], (variant, mode, c))


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_zero_hz_centre_estimate_is_the_oracle_s_or_its_mirror(variant):
    """A channel created at a negative centre runs at 0 Hz, as in the reference (WaveTable::SetFreq clamps, DSP.cpp:146):
    status and output equal those of a channel created at 0 Hz, and the loops start from the oracle's state. mixer_center
    then stands still at table entry 0, so the estimator's ring holds real samples, whose spectrum is mirror-symmetric
    about nfft/2: which of two mirror bins wins the fold search is decided by the rounding of each implementation's FFTs
    (DESIGN.md §2). The first estimate is the oracle's, or the same offset with the other sign; nothing else."""
    import jaero_b200 as jb
    kind, kw, _, _ = VARIANTS[variant]
    x = _streams(variant)[:1]
    T = cs.trigger_every(kw)
    b = jb.DemodBatch(kind, 2, **dict(_gpu_kw(kw), freq_center=np.array([-100.0, 0.0])))
    o = restated.OracleDemod(kind, **dict(kw, freq_center=-100.0))
    same = lambda a, c: all(a[k] == c[k] for k in a if k != "scatter")
    st0 = b.status()
    assert st0[0]["center_freq"] == st0[0]["mixer2_freq"] == 0.0 and same(st0[0], st0[1])
    for key in ("mixer2_freq", "center_freq", "st_freq", "mse"):
        assert st0[0][key] == o.state()[key], key
    # the first two epochs (each write ends on a trigger sample): the first estimate is not emitted (emptyingcountdown,
    # coarsefreqestimate.cpp:134), so mixer2 still stands at 0 Hz on both sides when the second is made
    for e in range(2):
        b.write(np.ascontiguousarray(np.repeat(x[:, e * T:(e + 1) * T], 2, axis=0)))
        o.write(x[0, e * T:(e + 1) * T])
        st, so = b.status(), o.state()
        assert same(st[0], st[1]), e
        assert st[0]["cfe_est"] in (so["cfe_est"], -so["cfe_est"]), (e, st[0]["cfe_est"], so["cfe_est"])
    b.close()


def trigger_samples(n, kw, cpu_reduce=False):
    """indices of the samples on which the coarse estimator triggers (oqpskdemodulator.cpp:410-429)"""
    N = 1 << kw["fft_power"]
    out, ptr, cc = [], 0, 0
    for i in range(n):
        if cc >= FS or not cpu_reduce:
            ptr = (ptr + 1) % N
            if ptr % (N if cpu_reduce else N // 4) == 0:
                out.append(i); cc = 0
        cc += 1
    return out


def edge_writes(n, kw, cpu_reduce=False, block=2048):
    """write sizes whose ends fall one sample before, on and one after every trigger sample (the last two as single-sample
    writes), and on the pre-filter's block edges between triggers"""
    ends = set()
    for t in trigger_samples(n, kw, cpu_reduce):
        ends.update((t, t + 1, t + 2))
        ends.add(t + 1 + block - (t + 1) % block)
        ends.add(t + 1 + 3 * block // 2 + 7)
    ends = sorted(e for e in ends if 0 < e < n) + [n]
    return list(np.diff([0] + ends))


@pytest.mark.parametrize("sql", [False, True])
@pytest.mark.parametrize("cpu_reduce", [False, True])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_writes_ending_at_estimator_and_prefilter_edges(variant, cpu_reduce, sql):
    """Writes that end on a trigger sample, one before and one after it (every bbnfft/4 samples, or at the end of every
    CPU-reduce ring run), on a 2048-sample pre-filter block edge and of a single sample, with squelch off and on: every
    channel equals the oracle fed the same writes."""
    kind, kw, _, _ = VARIANTS[variant]
    kw = dict(kw, sql=sql, cpureduce=cpu_reduce)
    x = _streams(variant)[:, :FS * 6]
    writes = edge_writes(x.shape[1], kw, cpu_reduce)
    assert min(writes) == 1 and sum(writes) == x.shape[1]
    refs = _oracle([(kind, kw, x[s], writes, ()) for s in range(3)])
    soft, st = _run_gpu(kind, kw, x, writes)
    for c in range(3):
        _assert_parity(soft[c], st[c], refs[c], (variant, c))


@pytest.mark.parametrize("variant", ["oqpsk_10500", "oqpsk_8400", "msk_600"])
def test_unaligned_and_strided_writes(variant):
    """write_device from pointers 1..7 samples off a 16-byte boundary and with row strides that are not a multiple of 8
    (re-pitched on the device), and jaero_batch_write with a host row stride of n + 37: the same stream as aligned writes,
    and the oracle's."""
    import torch
    import jaero_b200 as jb
    kind, kw, _, _ = VARIANTS[variant]
    x = _streams(variant)[:, :FS * 4]
    C, n = x.shape
    writes = [4800, 1, 4093, 9000, 7, 20000, 3, 8192, 12345] * 40
    writes = list(np.diff([0] + sorted(set(np.minimum(np.cumsum(writes), n)))))
    assert sum(writes) == n
    ref = _oracle([(kind, kw, x[s], writes, ()) for s in range(C)])
    aligned, sta = _run_gpu(kind, kw, x, writes)
    for c in range(C):
        _assert_parity(aligned[c], sta[c], ref[c], (variant, "aligned", c))

    def run(feed):
        b = jb.DemodBatch(kind, C, **_gpu_kw(kw))
        acc = [[] for _ in range(C)]
        a = 0
        for k, w in enumerate(writes):
            feed(b, k, a, w)
            a += w
            for c, s in enumerate(b.read_softbits()):
                acc[c].append(s)
        st = b.status(); b.close()
        return [np.concatenate(v) for v in acc], st

    dev = {}
    for off, pitch in ((3, n + 13), (5, n + 8 * 7), (0, n + 37)):          # off: first sample's position in its row
        t = torch.zeros((C, pitch + off), dtype=torch.int16)
        t[:, off:off + n] = torch.from_numpy(x)
        dev[(off, pitch)] = t.to("cuda")
    keys = list(dev)

    def feed_device(b, k, a, w):
        off, pitch = keys[k % len(keys)]
        t = dev[(off, pitch)]
        b.write_device(t.data_ptr() + 2 * int(off + a), int(w), t.shape[1])   # pointer offset (off + a) % 8, stride pitch + off
    got, stg = run(feed_device)
    host = np.zeros((C, n + 37), dtype=np.int16)
    host[:, :n] = x

    def feed_host(b, k, a, w):
        r = jb.lib().jaero_batch_write(b.h, ctypes.c_void_p(host.ctypes.data + 2 * int(a)), int(w), host.shape[1])
        assert r == 0
    goth, sth = run(feed_host)
    for c in range(C):
        assert np.array_equal(got[c], aligned[c]) and np.array_equal(goth[c], aligned[c]), c
        for key in ("mixer2_freq", "mixer2_wtptr", "st_wtptr", "mse", "agc", "center_wtptr"):
            assert stg[c][key] == sta[c][key] == sth[c][key], (c, key)


@pytest.mark.parametrize("variant", ["oqpsk_10500", "msk_1200"])
def test_peak_volume_of_every_write(variant):
    """PeakVolume (max |sample| / 32768 of the input since the last read-out) after every write, silent and loud writes in
    turn with the loudest sample in the last copy slice: writes of 8192 samples and more from page-locked memory (copied in
    slices on a second stream, overlapping the demodulation), short writes, and device writes."""
    import torch
    import jaero_b200 as jb
    kind, kw, _, _ = VARIANTS[variant]
    C = 128
    sizes = [96000, 8192, 4000, 50000, 8200, 1000]
    total = 2 * sum(sizes)
    rng = np.random.default_rng(11)
    pinned = torch.zeros((C, total), dtype=torch.int16).pin_memory()
    host = pinned.numpy()
    b = jb.DemodBatch(kind, C, **_gpu_kw(kw))
    a = 0
    for rep in range(2):
        for k, w in enumerate(sizes):
            loud = (k + rep) % 2 == 1
            seg = host[:, a:a + w]
            if loud:
                seg[:] = rng.integers(-3000, 3000, size=seg.shape, dtype=np.int16)
                hot = w - 1 - rng.integers(0, max(1, w // 16), size=C)               # in the last of the eight copy slices
                seg[np.arange(C), hot] = rng.integers(20000, 32767, size=C).astype(np.int16) * np.where(np.arange(C) % 2, 1, -1).astype(np.int16)
            else:
                seg[:] = rng.integers(-5, 5, size=seg.shape, dtype=np.int16)
            expect = np.abs(seg.astype(np.int32)).max(axis=1) / 32768.0
            if rep == 1 and k % 3 == 2:
                d = torch.from_numpy(np.ascontiguousarray(seg)).to("cuda")
                b.write_device(d.data_ptr(), w, d.stride(0))
            else:
                r = jb.lib().jaero_batch_write(b.h, ctypes.c_void_p(seg.ctypes.data), w, host.shape[1])
                assert r == 0
            got = np.array([s["peak_volume"] for s in b.status()])
            assert np.array_equal(got, expect), (rep, k, w, loud, np.nonzero(got != expect)[0][:8])
            a += w
    b.close()
