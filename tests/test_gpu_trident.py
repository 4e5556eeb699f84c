"""GPU tests: the burst demodulators' trident FFTs and peak searches (burst.cu: trident_fft_kernel, trident_peaks_kernel,
trident_peaks_oqpsk_kernel, argmax_first) on caller segments through jaero_burst_probe_trident, against the long-double
reference of tests/trident_reference.py, for burst MSK 1200, burst MSK 600 and burst OQPSK.

300 events per mode (three rounds of 128) over 48 channels and all eight slots, each with its own segment: synthetic preamble
tones, noise, zeros, DC, single samples either side of the base/top split, and (1200 bps MSK, OQPSK) the oracle's fills of the
burst recordings. Each spectrum must lie within the FFT bound; the restated search on the kernel's own spectra must give the
kernel's bins exactly and its values within a few ulp; the bins must agree with the long-double search apart from counted
near-ties. Hand-built spectra through spectra_in pin the searches' tie-breaks and range edges exactly."""
import json
import os

import numpy as np
import pytest

import trident_reference as T
from conftest import ROOT, has_cuda

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

MODES = {"msk1200": ("msk", 1200.0), "msk600": ("msk", 600.0), "oqpsk": ("oqpsk", 10500.0)}
RECORDINGS = {"msk1200": ("burst_msk_1200_a", "burst_msk_1200_b"), "msk600": (), "oqpsk": ("burst_oqpsk_10500",)}
C = 48
N_EVENTS = 300
KINDS = ("tone", "noise", "zeros", "dc", "imp_base_last", "imp_top_first")
# a single sample has a spectrum of one magnitude in every bin: every peak decision on it is a near-tie by construction, so
# these segments pin the section split through the spectrum bound, and their decisions are compared only where not near-tied
FLAT = ("imp_base_last", "imp_top_first")


def make_batch(mode, n_channels=C):
    import jaero_b200
    kind, fb = MODES[mode]
    return jaero_b200.BurstOqpskBatch(n_channels) if kind == "oqpsk" else jaero_b200.BurstMskBatch(n_channels, fb=fb)


def synthetic(kind_name, mode, g, rng):
    kind, fb = MODES[mode]
    sz, nb = g["tri_sz"], g["base_len"]
    t = np.arange(sz) / 48000.0
    if kind_name == "tone":
        f0 = rng.uniform(1500.0, 3000.0) if kind == "msk" else rng.uniform(3000.0, 9000.0)
        side = fb / 2.0 if kind == "msk" else fb / 4.0
        ph = rng.uniform(0, 2 * np.pi, 3)
        s = np.cos(2 * np.pi * f0 * t + ph[0])
        s[nb:] = 0.7 * (np.cos(2 * np.pi * (f0 - side) * t[nb:] + ph[1]) + np.cos(2 * np.pi * (f0 + side) * t[nb:] + ph[2]))
        return s * rng.uniform(0.5, 2.0) + 0.05 * rng.standard_normal(sz)
    if kind_name == "noise":
        return rng.standard_normal(sz)
    if kind_name == "zeros":
        return np.zeros(sz)
    if kind_name == "dc":                                 # one level in the base, another in the top section
        s = np.full(sz, rng.uniform(0.1, 1.0))
        s[nb:] = rng.uniform(1.5, 3.0)
        return s
    s = np.zeros(sz)
    s[nb - 1 if kind_name == "imp_base_last" else nb] = rng.uniform(0.5, 2.0)
    return s


def recording_fills(name):
    from oracle import restated
    from conftest import load_excerpt
    with open(os.path.join(ROOT, "tests", "golden", "expected_outputs.json")) as fh:
        case = json.load(fh)[name]
    d = restated.OracleDemod(case["kind"], **case["kw"])
    pcm = load_excerpt(case["excerpt"])
    segs, logs = [], []
    for a in range(0, len(pcm), case["chunk"]):
        d.write(pcm[a:a + case["chunk"]])
        segs.append(d.take_aux(3, cap=1 << 22))
        logs.append(d.take_aux(1, cap=1 << 16))
    d.close()
    return np.concatenate(segs), np.concatenate(logs).reshape(-1, 5)


def layout(rng):
    """300 distinct (channel, slot) pairs in random order, including (C-1, 7)"""
    pairs = [(c, s) for c in range(C) for s in range(8)]
    idx = rng.permutation(len(pairs))[:N_EVENTS]
    chosen = [pairs[i] for i in idx]
    if (C - 1, 7) not in chosen:
        chosen[int(rng.integers(0, N_EVENTS))] = (C - 1, 7)
    ch = np.array([p[0] for p in chosen], dtype=np.int32)
    sl = np.array([p[1] for p in chosen], dtype=np.int32)
    assert len(set(np.unique(ch))) >= 40 and set(sl) == set(range(8))
    return ch, sl


def events(mode):
    """(channels, slots, segments [300, tri_sz], labels, oracle trident log rows (None for synthetic))"""
    kind, fb = MODES[mode]
    g = T.geometry(kind, fb)
    rng = np.random.default_rng({"msk1200": 1, "msk600": 2, "oqpsk": 3}[mode])
    ch, sl = layout(rng)
    segs, labels, logs = [], [], []
    for name in RECORDINGS[mode]:
        s, lg = recording_fills(name)
        s = s.reshape(-1, g["tri_sz"])
        for k in range(len(s)):
            segs.append(s[k]); labels.append("rec:%s:%d" % (name, k)); logs.append(lg[k])
    while len(segs) < N_EVENTS:
        k = KINDS[len(segs) % len(KINDS)]
        segs.append(synthetic(k, mode, g, rng)); labels.append(k); logs.append(None)
    order = rng.permutation(N_EVENTS)                     # recordings spread over the rounds
    return ch, sl, np.stack(segs)[order], [labels[i] for i in order], [logs[i] for i in order]


def _ulp_close(a, b, ulps=4):
    return abs(a - b) <= ulps * np.spacing(max(abs(a), abs(b))) or a == b


@pytest.mark.parametrize("mode", sorted(MODES))
def test_trident_against_long_double(mode):
    kind, fb = MODES[mode]
    g = T.geometry(kind, fb)
    b = make_batch(mode)
    assert b.trident_geometry() == g
    ch, sl, segs, labels, logs = events(mode)
    res, spec = b.probe_trident(ch, sl, segs, want_spectra=True)
    b.close()
    chk = T.Checker()
    ulp_ties = ld_ties = 0
    for e0 in range(0, N_EVENTS, 50):
        ref = T.spectra(segs[e0:e0 + 50], g)
        chk.spectra(spec[e0:e0 + 50], ref, what=mode)
        for j in range(ref.shape[0]):
            e = e0 + j
            r, got, lab = res[e], spec[e], labels[e]
            # the restated search on the kernel's own spectra
            mine = T.search(kind, fb, got)
            mag = np.hypot(got.real, got.imag)
            if T.near_tie(kind, fb, mag, T.ulp_tol(got)):
                assert lab.startswith("rec") or lab in FLAT, "%s event %d (%s): near-tie on a synthetic segment" % (mode, e, lab)
                ulp_ties += lab not in FLAT
            else:
                assert int(r[0]) == mine[0] and int(r[2]) == mine[2], (mode, e, lab, r, mine)
                if kind == "msk":
                    assert int(r[3]) == mine[3], (mode, e, lab, r, mine)
                else:
                    tol = 8 * sum(np.spacing(float(mag[w][k])) for w in range(2) for k in (mine[2] - T.oqpsk_bps(), mine[2], mine[2] + T.oqpsk_bps()))
                    assert abs(r[3] - float(mine[3])) <= tol + 4 * np.spacing(abs(r[3])), (mode, e, lab, r, mine)
                assert _ulp_close(r[1], float(mine[1])), (mode, e, lab, r, mine)
                mb = int(r[0])
                assert _ulp_close(r[4], float(np.arctan2(got[0, mb].imag, got[0, mb].real))), (mode, e, lab, r)
            # against the long-double search
            ldm = np.abs(ref[j]).astype(np.float64)
            tol = np.stack([np.full(T.N, 2 * T.SPECTRUM_REL * float(np.sqrt(np.sum(ldm[w] ** 2)))) for w in range(2)]) + T.ulp_tol(got)
            ld = T.search(kind, fb, ref[j])
            if T.near_tie(kind, fb, ldm, tol):
                ld_ties += lab not in FLAT
            else:
                assert int(r[0]) == ld[0] and int(r[2]) == ld[2], (mode, e, lab, r, ld)
                if kind == "msk":
                    assert int(r[3]) == ld[3], (mode, e, lab, r, ld)
            # the recordings: the oracle's trident log
            if logs[e] is not None and not T.near_tie(kind, fb, ldm, tol):
                o = logs[e]
                assert int(r[0]) == int(o[0]) and int(r[2]) == int(o[2]), (mode, e, lab, r, o)
                if kind == "msk":
                    assert int(r[3]) == int(o[3]), (mode, e, lab, r, o)
                assert abs(r[1] - o[1]) <= tol[0][0] + 4 * np.spacing(o[1]), (mode, e, lab, r, o)
        del ref
    print("TRIDENT-STATS %s: %d events, worst spectrum error / bound = %.3g, near-ties outside the single-sample segments: "
          "%d (own spectra), %d (long double)" % (mode, N_EVENTS, chk.worst, ulp_ties, ld_ties))
    assert ld_ties * 100 <= N_EVENTS, "%d near-ties against the long-double spectra" % ld_ties


# ---------------------------------------------------------------------------------------------------- hand-built spectra
def _spec(base=None, top=None):
    s = np.zeros((2, T.N), dtype=np.complex128)
    for w, d in ((0, base), (1, top)):
        for k, v in (d or {}).items():
            s[w, k] = v
    return s


def msk_cases(fb):
    h = T.peak_spacing(fb) // 2
    m = 1000
    return {
        # exact ties: adjacent bins (threads 1000 and 1001), 1024 apart (one thread's stride), and 1023 / 1024 (thread 1023 and 0)
        "tie_adjacent": (_spec({m: 3.0, m + 1: 3.0}), (m, None, None)),
        "tie_stride": (_spec({m: 3.0, m + 1024: 3.0}), (m, None, None)),
        "tie_wrap": (_spec({1023: 3.0, 1024: 3.0, 5000: 1.0}), (1023, None, None)),
        "above_half": (_spec({m: 3.0, 20000: 30.0}, {20000: 9.0, 600: 1.0}), (m, 600, None)),
        "bins_50_51": (_spec({m: 3.0}, {50: 9.0, 51: 1.0}), (m, 51, None)),
        "bin_50_only": (_spec({m: 3.0}, {50: 9.0}), (m, 0, None)),
        "exclusion_edges": (_spec({m: 3.0}, {m - h: 9.0, m - h - 1: 2.0, m + h: 9.0, m + h + 1: 2.0}), (m, m - h - 1, m + h + 1)),
        "top_ties": (_spec({m: 3.0}, {200: 2.0, 201: 2.0, 3000: 2.0, 3000 + 1024: 2.0}), (m, 200, 3000)),
        "zero_top": (_spec({m: 3.0}), (m, 0, 0)),
        "zero_base": (_spec(None, {60: 1.0, 4000: 2.0}), (0, 0, 4000)),
        "all_zero": (_spec(), (0, 0, 0)),
        "complex_tie": (_spec({777: 3 - 4j, 777 + 2048: 3 - 4j, 99: 3 - 4j}), (99, None, None)),
    }


def oqpsk_cases():
    bps = T.oqpsk_bps()
    first, lst = bps, T.HALF - bps

    def peak(k0, a=5.0):                     # testval(k0) = 2a, the largest
        return {k0 - bps: a, k0 + bps: a}
    return {
        "at_firstbin": (_spec({300: 1.0}, peak(first)), (300, first)),
        "at_lstbin_minus_1": (_spec({300: 1.0}, peak(lst - 1)), (300, lst - 1)),
        "past_lstbin": (_spec({300: 1.0, lst: 50.0}), (lst, first)),
        "constant_diff": (_spec(None, {k: 1.0 for k in range(T.HALF)}), (0, first)),
        "all_zero": (_spec(), (0, first)),
        "tie_adjacent": (_spec({300: 1.0}, {**peak(5000), **peak(5001)}), (300, 5000)),
        "tie_stride": (_spec({300: 1.0}, {**peak(5000), **peak(5000 + 1024)}), (300, 5000)),
        "base_ties": (_spec({1500: 2.0, 1501: 2.0, 1500 + 1024: 2.0}), (1500, None)),
        "above_half": (_spec({700: 2.0, 17000: 20.0}, {17000: 20.0}), (700, None)),
    }


@pytest.mark.parametrize("mode", sorted(MODES))
def test_trident_peaks_on_hand_built_spectra(mode):
    kind, fb = MODES[mode]
    cases = msk_cases(fb) if kind == "msk" else oqpsk_cases()
    names = sorted(cases)
    spec = np.stack([cases[k][0] for k in names])
    n = len(names)
    b = make_batch(mode, n_channels=3)
    ch = np.arange(n, dtype=np.int32) % 3
    sl = (7 - np.arange(n, dtype=np.int32) // 3).astype(np.int32)       # slots counted down, so a slot is not its event number
    res, _ = b.probe_trident(ch, sl, spectra_in=spec)
    b.close()
    for e, name in enumerate(names):
        r = res[e]
        want = T.search(kind, fb, spec[e])
        exp = cases[name][1]
        got_bins = (int(r[0]), int(r[2]), int(r[3])) if kind == "msk" else (int(r[0]), int(r[2]))
        want_bins = (want[0], want[2], want[3]) if kind == "msk" else (want[0], want[2])
        assert got_bins == want_bins, "%s %s: kernel %r, restated search %r" % (mode, name, got_bins, want_bins)
        for g_, x_ in zip(want_bins, exp):
            if x_ is not None:
                assert g_ == x_, "%s %s: restated search %r, case expects %r" % (mode, name, want_bins, exp)
        assert _ulp_close(r[1], float(want[1])), (mode, name, r, want)
        if kind == "oqpsk":
            assert _ulp_close(r[3], float(want[3])), (mode, name, r, want)


def test_trident_probe_rejects_bad_events():
    import jaero_b200
    b = make_batch("msk1200", n_channels=4)
    g = b.trident_geometry()
    seg = np.zeros((2, g["tri_sz"]))
    with pytest.raises(jaero_b200.JaeroError, match="channel out of range"):
        b.probe_trident([0, 4], [0, 1], seg)
    with pytest.raises(jaero_b200.JaeroError, match="channel out of range"):
        b.probe_trident([-1, 0], [0, 1], seg)
    with pytest.raises(jaero_b200.JaeroError, match="slot outside"):
        b.probe_trident([0, 1], [0, 8], seg)
    with pytest.raises(jaero_b200.JaeroError, match="slot outside"):
        b.probe_trident([0, 1], [-1, 0], seg)
    with pytest.raises(jaero_b200.JaeroError, match="appears twice"):
        b.probe_trident([2, 2], [5, 5], seg)
    res, _ = b.probe_trident([3, 3], [7, 0], seg)
    assert not res[:, :4].any()
    b.close()
