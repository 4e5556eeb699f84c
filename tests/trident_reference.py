"""Plain long-double restatement of the burst demodulators' trident test (the two zero-padded FFTs of a fill and the peak searches
of BurstMskDemodulator::writeData, JAERO/burstmskdemodulator.cpp:474-520, and BurstOqpskDemodulator::writeData,
burstoqpskdemodulator.cpp:416-462), for the tests that compare the CUDA kernels (jaero_b200/csrc/burst.cu) with it.

The transforms run in scipy.fft on np.clongdouble (80-bit extended precision on x86-64). The searches are the reference's loops
with strict '>' (the first maximum wins), written as first-argmax over the same ranges; they run on any spectrum, the
long-double one or one a kernel produced.

Error bound (standard FP64 FFT analysis with margin): ||X - X_ref||_2 / ||X_ref||_2 <= 4 * 15 * 2^-52 per 32768-point transform
(log2 32768 = 15). An all-zero section must give exact zeros."""
import numpy as np
import scipy.fft

N = 32768
HALF = N // 2
SPECTRUM_REL = 4 * 15 * 2.0 ** -52
HZPERBIN = 48000.0 / N


def _qround(d):
    return int(np.floor(d + 0.5))


def geometry(kind, fb):
    """tri_sz, base_len, top_len of the reference's trident buffer (burstmskdemodulator.cpp:205-311, 447-448;
    burstoqpskdemodulator.cpp:202-277, 404)"""
    if kind == "oqpsk":
        sps = 2 * 48000.0 / 10500.0
        nseg = _qround(128.0 * sps)
        return dict(tri_sz=_qround(288.0 * sps), base_len=nseg, top_len=nseg, nfft=N)
    sps = 48000.0 / fb
    base, tri = (126, 200) if fb >= 1200 else (150, 224)
    return dict(tri_sz=_qround(tri * sps), base_len=_qround(base * sps), top_len=_qround(74 * sps), nfft=N)


def sections(seg, g):
    """the base and the top section of one fill, zero-padded to N: base = seg[0:base_len], top = seg[base_len:base_len+top_len],
    both cut at tri_sz"""
    nb, nt, sz = g["base_len"], g["top_len"], g["tri_sz"]
    out = np.zeros((2, N), dtype=np.float64)
    b = seg[:min(nb, sz)]
    t = seg[nb:min(nb + nt, sz)]
    out[0, :len(b)] = b
    out[1, :len(t)] = t
    return out


def spectra(segs, g):
    """[n, 2, N] long-double spectra (base, top) of segments [n, tri_sz]"""
    x = np.stack([sections(s, g) for s in np.asarray(segs, dtype=np.float64)])
    return scipy.fft.fft(x.astype(np.clongdouble), axis=-1)


def peak_spacing(fb):
    """qRound((0.5 fb) / hzperbin): the MSK side peaks' spacing in bins"""
    return int(np.floor(0.5 * fb / HZPERBIN + 0.5))


def oqpsk_bps():
    return int(np.floor(0.25 * 10500.0 / HZPERBIN + 0.5))


def _first_max(v, lo, hi, init=None):
    """the reference loop `for k in [lo, hi): if v[k] > best: best, pos = v[k], k` from (init, None) or, init None, from
    (v[lo], lo) -> (pos or None, best)"""
    seg = v[lo:hi]
    if len(seg) == 0:
        return (None, init) if init is not None else (lo, v[lo])
    k = int(np.argmax(seg))
    if init is not None and not seg[k] > init:
        return None, init
    return lo + k, seg[k]


def search_msk(mag_base, mag_top, fb):
    """:478-520 on magnitude rows [N] (only bins < N/2 are read) -> (minvalbin, minval, maxtoppos, maxtopposhigh)"""
    psb = peak_spacing(fb)
    mb, mt = mag_base[:HALF], mag_top[:HALF]
    k, v = _first_max(mb, 0, HALF, init=0.0)
    minvalbin, minval = (0, 0.0) if k is None else (k, v)
    lo_hi = minvalbin - psb // 2                    # candidates k > 50 and k < lo_hi, or k > 50 and k > hi_lo
    hi_lo = minvalbin + psb // 2
    k1, _ = _first_max(mt, 51, max(51, lo_hi), init=0.0)
    k2, _ = _first_max(mt, max(51, hi_lo + 1), HALF, init=0.0)
    return minvalbin, minval, (0 if k1 is None else k1), (0 if k2 is None else k2)


def oqpsk_testvals(mag_base, mag_top):
    """testval[k] = diff[k-bps] + diff[k+bps] - diff[k] for k in [firstbin, lstbin) (index k), diff = |top| - |base|"""
    bps = oqpsk_bps()
    diff = mag_top[:HALF] - mag_base[:HALF]
    t = np.full(HALF, np.nan, dtype=diff.dtype)
    k = np.arange(bps, HALF - bps)
    t[k] = diff[k - bps] + diff[k + bps] - diff[k]
    return t


def search_oqpsk(mag_base, mag_top):
    """:416-462 -> (minvalbin, minval, maxvalbin, maxval)"""
    bps = oqpsk_bps()
    first, lst = bps, HALF - bps
    t = oqpsk_testvals(mag_base, mag_top)
    maxvalbin, maxval = _first_max(t, first, lst)
    mb = mag_base[:HALF]
    k, v = _first_max(mb, 0, HALF, init=mb[0])
    minvalbin, minval = (0, mb[0]) if k is None else (k, v)
    return minvalbin, minval, maxvalbin, maxval


def search(kind, fb, spec):
    """the peak search of `kind` ('msk' or 'oqpsk') on one event's spectra [2, N] (any complex dtype; magnitudes by hypot in the
    spectrum's precision) -> (minvalbin, minval, bin2, value/bin3) as jaero_burst_probe_trident's result[0:4]"""
    spec = np.asarray(spec)
    if spec.dtype == np.clongdouble:
        mag = np.abs(spec)
    else:
        mag = np.hypot(spec.real, spec.imag)
    return search_msk(mag[0], mag[1], fb) if kind == "msk" else search_oqpsk(mag[0], mag[1])


def _close_to(v, best, tol, lo, hi, before):
    """candidates in [lo, hi) other than the winner `before` whose value + tol passes best - tol, or reaches it from a lower bin
    (the first maximum wins). With zero tolerances exact ties are decided the same way everywhere and do not count."""
    if hi <= lo:
        return False
    s = v[lo:hi]
    ts = tol[lo:hi]
    idx = np.arange(lo, hi)
    floor = best - tol_at(tol, before)
    close = (s + ts > floor) | ((s + ts >= floor) & (idx < (before if before is not None else lo)))
    if before is not None:
        close &= idx != before
    return bool(close.any())


def tol_at(tol, k):
    return 0.0 if k is None else float(tol[k])


def near_tie(kind, fb, mag, tol):
    """True where an implementation whose magnitudes lie within tol [2, N] of mag [2, N] (float64) could take another decision:
    another candidate comes within the tolerances of a winner, or a winner within its tolerance of the loop's starting value"""
    mb, mt = mag[0][:HALF], mag[1][:HALF]
    tb, tt = tol[0][:HALF], tol[1][:HALF]
    if kind == "msk":
        psb = peak_spacing(fb)
        mvb, mv, k1, k2 = search_msk(mag[0], mag[1], fb)
        if mv - tb[mvb] <= 0 and (mb + tb > 0).any():
            return True
        if mv > 0 and _close_to(mb, mv, tb, 0, HALF, mvb):
            return True
        for k, lo, hi in ((k1, 51, max(51, mvb - psb // 2)), (k2, max(51, mvb + psb // 2 + 1), HALF)):
            if k == 0 or k is None:
                if hi > lo and (mt[lo:hi] + tt[lo:hi] > 0).any():
                    return True
            elif mt[k] - tt[k] <= 0 or _close_to(mt, mt[k], tt, lo, hi, k):
                return True
        # a winner moving by its tolerance could move the exclusion window by a bin: only when minvalbin itself is a near-tie
        return False
    bps = oqpsk_bps()
    t = oqpsk_testvals(mb, mt)
    td = tt + tb
    tt_ = np.zeros(HALF)
    k = np.arange(bps, HALF - bps)
    tt_[k] = td[k - bps] + td[k + bps] + td[k] + _ulps(t[k], 4)
    mvb, _, kx, _ = search_oqpsk(mag[0], mag[1])
    if _close_to(t, t[kx], tt_, bps, HALF - bps, kx):
        return True
    if _close_to(mb, mb[mvb], tb, 0, HALF, mvb):
        return True
    return False


def ulp_tol(spec64, ulps=4):
    """per-bin magnitude tolerance of `ulps` ulp of hypot, for searches on the same double spectrum with another hypot"""
    return _ulps(np.hypot(spec64.real, spec64.imag), ulps)


def _ulps(v, ulps):
    """ulps ulp of each value, and 0 for exact zeros (a zero stays exact in every implementation)"""
    v = np.abs(np.asarray(v, dtype=np.float64))
    return np.where(v != 0, ulps * np.spacing(v), 0.0)


class Checker:
    """Counts compared events and near-ties, and the largest spectrum error as a fraction of the bound"""

    def __init__(self):
        self.compared = self.ties = 0
        self.worst = 0.0

    def spectra(self, got, ref, what=""):
        """got [n, 2, N] complex128, ref [n, 2, N] clongdouble: each transform within SPECTRUM_REL; all-zero inputs exactly 0"""
        for e in range(got.shape[0]):
            for w in range(2):
                r = ref[e, w]
                nr = float(np.sqrt(np.sum(np.abs(r) ** 2)))
                if nr == 0.0:
                    assert not got[e, w].any(), "%s: event %d section %d: zero input, nonzero spectrum" % (what, e, w)
                    continue
                err = float(np.sqrt(np.sum(np.abs(got[e, w].astype(np.clongdouble) - r) ** 2)))
                ratio = err / (SPECTRUM_REL * nr)
                self.worst = max(self.worst, ratio)
                assert ratio <= 1.0, "%s: event %d section %d: relative error %.3g, bound %.3g" % (what, e, w, err / nr, SPECTRUM_REL)
