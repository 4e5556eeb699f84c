"""GPU tests of the coarse frequency estimator kernels (pytest -m gpu) against the long-double restatement of
CoarseFreqEstimate::ProcessBasebandData in tests/cfe_reference.py, one epoch at a time through jaero_batch_probe_cfe: the
four-pass kernels at every FFT size and the cluster kernel at 2^14, channel groups, cluster reuse across channels, the general
fold-search path, odd channel counts; then whole recordings against the CPU oracle's per-epoch estimates.

Each epoch checks the spectrum max(|X|,1) recovered from the smoothed y against the long-double value, the fold search on the
kernel's own y against the restated loop (exactly), the estimate against the reference (near-ties counted and skipped), and the
emit gate."""
import functools
import os

import numpy as np
import pytest

import cfe_reference as R
from conftest import has_cuda, load_excerpt
from oracle import restated

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

FOUR_PASS, CLUSTER = 1, 2


def default_flags(C):
    """bigchange() before epoch 0 on every third channel (the all-zero channel among them) and mid-sequence on others"""
    c = np.arange(C)
    return {0: c % 3 == 0, 3: c % 3 == 1}


def run_epochs(kind, fb, lockingbw, power, C, runs, epochs=8, flags=None, max_group=0, seed=0):
    """runs: list of (impl, max_clusters); one batch per run, all fed the same rings. Returns the checkers."""
    import jaero_b200
    g = R.geometry(power, lockingbw, fb)
    N = g["nfft"]
    batches = [jaero_b200.DemodBatch(kind, C, fb=fb, lockingbw=lockingbw, fft_power=power) for _ in runs]
    geo = batches[0].cfe_geometry()
    assert (geo["nfft"], geo["lo"], geo["hi"], geo["expectedpeakbin"]) == (N, g["lo"], g["hi"], g["expectedpeakbin"])
    bb_len = geo["bb_len"]
    kinds = [R.KINDS[c % len(R.KINDS)] for c in range(C)]
    rng = np.random.default_rng(seed + power * 131 + int(fb))
    offsets = rng.uniform(-0.4, 0.4, C) * lockingbw / 2
    ref = R.CfeReference(g, C)
    checkers = [R.Checker(g, C) for _ in runs]
    ties = [c for c in range(C) if kinds[c] in R.TIE_KINDS]
    orc = {c: restated.OracleCfe(power, lockingbw, fb) for c in ties}
    flags = default_flags(C) if flags is None else flags
    oldests = [0, 1, None, bb_len - 1]
    try:
        for e in range(epochs):
            oldest = oldests[e % len(oldests)]
            oldest = int(rng.integers(0, bb_len)) if oldest is None else oldest
            ring = np.stack([R.make_ring(k, bb_len, fb, lockingbw, offsets[c], rng) for c, k in enumerate(kinds)])
            data = R.linearise(ring, oldest, N)
            bc = np.asarray(flags.get(e, np.zeros(C, dtype=bool)), dtype=bool)
            ref.bigchange(bc)
            tie_raw = np.full(C, np.nan)
            for c in ties:
                if bc[c]:
                    orc[c].bigchange()
                tie_raw[c] = orc[c].process(data[c])[1]
            out = ref.process(data)
            for (impl, mc), b, chk in zip(runs, batches, checkers):
                what = "%s fb %g 2^%d C=%d impl %d clusters %d epoch %d oldest %d" % (kind, fb, power, C, impl, mc, e, oldest)
                y, raw, emitted = b.probe_cfe(ring, oldest, bc.astype(np.int32), impl=impl, max_clusters=mc, max_group=max_group)
                chk.epoch(out, y, raw, bc, kinds, tie_raw=tie_raw, what=what)
                gate = np.where(out["gate_open"], raw, 0.0)
                assert np.array_equal(emitted, gate), "%s: emitted %r, gate says %r" % (what, emitted, gate)
                if e == 0:
                    assert (emitted == 0).all(), what
    finally:
        for b in batches:
            b.close()
        for o in orc.values():
            o.close()
    for (impl, mc), chk in zip(runs, checkers):
        print("CFE-STATS %s fb=%g 2^%d C=%d impl=%d clusters=%d group=%d: compared %d, near-tie skips %d, worst spectrum error %.3g of the bound"
              % (kind, fb, power, C, impl, mc, max_group, chk.compared, chk.skips, chk.worst))
        assert chk.skips <= max(1, 0.02 * chk.compared), (chk.skips, chk.compared, chk.skipped_kinds)
        assert chk.compared >= epochs * C * 0.9
    return checkers


CONFIGS = [("oqpsk", 10500.0, 10500.0, p) for p in (10, 11, 12, 13, 14)] + [("oqpsk", 8400.0, 10500.0, p) for p in (10, 11, 12, 13, 14)] + \
          [("msk", 600.0, 900.0, 13), ("msk", 1200.0, 1800.0, 13)]


@pytest.mark.parametrize("kind,fb,lockingbw,power", CONFIGS)
def test_estimator_matches_long_double_reference(kind, fb, lockingbw, power):
    """every FFT size and both spectrum shapes (boxcar mask, raised-cosine window at 8400) through the four-pass kernels; nfft 16384
    through the cluster kernel too"""
    runs = [(FOUR_PASS, 0)] + ([(CLUSTER, 0)] if power == 14 else [])
    run_epochs(kind, fb, lockingbw, power, 7, runs)


def test_channel_groups_offset_every_per_channel_array():
    """groups of 16 at 70 channels: four full groups and a ragged one; bigchange() on both sides of every group boundary"""
    C = 70
    flags = {0: np.isin(np.arange(C), [0, 15, 32, 47, 64, 69]), 3: np.isin(np.arange(C), [16, 31, 48, 63, 1])}
    run_epochs("oqpsk", 10500.0, 10500.0, 13, C, [(FOUR_PASS, 0)], flags=flags, max_group=16)


def test_cluster_kernel_reuses_its_clusters_across_channels():
    """few clusters for many channels: each cluster runs several channels in turn through the same shared memory"""
    run_epochs("oqpsk", 10500.0, 10500.0, 14, 20, [(CLUSTER, 1), (CLUSTER, 2), (CLUSTER, 7)])
    import jaero_b200
    b = jaero_b200.DemodBatch("oqpsk", 1, fb=10500.0)
    cap = b.cfe_geometry()["clusters"]
    b.close()
    assert cap > 0, "the cluster estimator cannot run on this device"
    run_epochs("oqpsk", 8400.0, 10500.0, 14, 3 * cap + 5, [(CLUSTER, 0)], epochs=6)


@pytest.mark.parametrize("power", [13, 14])
def test_fold_search_general_path(power):
    """lockingbw + fb/2 > Fs/2: the fold leaves the spectrum and the search kernel takes its range-checked path"""
    g = R.geometry(power, 20000.0, 10500.0)
    assert g["lo"] - g["expectedpeakbin"] - 1 < 0 or g["hi"] + g["expectedpeakbin"] + 1 >= g["nfft"]
    run_epochs("oqpsk", 10500.0, 20000.0, power, 7, [(FOUR_PASS, 0)] + ([(CLUSTER, 0)] if power == 14 else []))


@pytest.mark.parametrize("C", [1, 5])
def test_odd_channel_counts(C):
    run_epochs("oqpsk", 10500.0, 10500.0, 14, C, [(FOUR_PASS, 0), (CLUSTER, 0)])


# ---------------------------------------------------------------------------------------------------- whole recordings

def _variants(pcm):
    return np.stack([pcm, (pcm.astype(np.int32) * 2 // 3).astype(np.int16), pcm[::-1].copy()])


@functools.lru_cache(maxsize=None)
def _oracle_estimates(name):
    import json
    from conftest import ROOT
    with open(os.path.join(ROOT, "tests", "golden", "expected_outputs.json")) as fh:
        case = json.load(fh)[name]
    kw = dict(case["kw"])
    quarter = (1 << kw["fft_power"]) // 4
    pcm = _variants(load_excerpt(case["excerpt"]))
    pcm = np.ascontiguousarray(pcm[:, :pcm.shape[1] - pcm.shape[1] % quarter])    # whole trigger intervals only
    raw, emitted = [], []
    for c in range(3):
        o = restated.OracleDemod(case["kind"], **kw)
        for a in range(0, pcm.shape[1], quarter):
            o.write(pcm[c, a:a + quarter])
        emitted.append(o.take_cfe_log())
        raw.append(o.take_cfe_log(raw=True))
        o.close()
    return case["kind"], kw, pcm, raw, emitted


def _gpu_estimates(name):
    import jaero_b200
    kind, kw, pcm, _, _ = _oracle_estimates(name)
    quarter = (1 << kw["fft_power"]) // 4
    b = jaero_b200.DemodBatch(kind, 3, **kw)
    geo = b.cfe_geometry()
    ests = []
    try:
        for a in range(0, pcm.shape[1], quarter):
            b.write(pcm[:, a:a + quarter])                        # exactly one estimator epoch per call
            ests.append([s["cfe_est"] for s in b.status()])
    finally:
        b.close()
    return geo, np.asarray(ests).T


@pytest.mark.parametrize("name", ["oqpsk_10500", "oqpsk_8400", "msk_1200"])
def test_recording_estimates_per_epoch(name):
    """3 channels of a recording, one trigger interval per write: the estimate of every epoch equals the oracle's (the cluster
    kernel at nfft 2^14, the four-pass kernels below it)"""
    _, _, pcm, raw, emitted = _oracle_estimates(name)
    geo, got = _gpu_estimates(name)
    if geo["nfft"] == 16384:
        assert geo["clusters"] > 0
    for c in range(3):
        assert len(raw[c]) == got.shape[1] and len(raw[c]) > 50
        bad = np.nonzero(got[c] != raw[c])[0]
        assert len(bad) == 0, "%s channel %d: epochs %s differ, gpu %s, oracle %s" % (name, c, bad[:8], got[c][bad[:4]], raw[c][bad[:4]])
        nz = emitted[c] != 0                                      # what the oracle emitted past the gate is that epoch's estimate
        assert np.array_equal(emitted[c][nz], raw[c][nz])
