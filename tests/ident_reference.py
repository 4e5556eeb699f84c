"""Plain restatement of the mode identifier's two contracts (include/jaero_b200.h, jaero_ident_*): the squared-signal spectrum in
long double, and the line-pair classifier in float64.

The transforms run in scipy.fft on np.clongdouble (80-bit extended precision on x86-64), so the reference spectrum is about
three decimal digits more accurate than any double-precision implementation it is compared with. The classifier is restated
with numpy on the same float64 spectrum the library's classifier reads, with its tie rules (the first bin, the first partner
offset, the first mode)."""
import math

import numpy as np
import scipy.fft

import scan_reference

FBS = (600.0, 1200.0, 8400.0, 10500.0)
MODES = ("msk600", "msk1200", "oqpsk8400", "oqpsk10500")
DEFAULTS = dict(threshold_db=5.0, floor_window_hz=400.0, floor_quantile=0.5)
LD_PI = np.arccos(np.longdouble(-1))

# The committed excerpts: (fixture, Fs, bit rate, carrier(s) in Hz any of which the identified one may be). The carriers are
# what this reference finds on the whole excerpt; where a recording holds two carriers of the rate, both are listed.
EXCERPTS = (
    ("oqpsk_10500", 48000, 10500, (5757.3,)),
    ("oqpsk_10500_44k1", 44100, 10500, (5757.3,)),
    ("oqpsk_8400", 48000, 8400, (2536.4, 7536.0)),
    ("msk_600", 48000, 600, (1020.4, 3515.0)),
    ("msk_1200", 48000, 1200, (2037.0,)),
    ("burst_msk_1200_a", 48000, 1200, (1831.0,)),
    ("burst_msk_1200_b", 48000, 1200, (2085.3,)),
    ("burst_oqpsk_10500", 48000, 10500, (11173.4,)),
)
# the margin (dB) of the right rate over the best wrong one that each excerpt keeps, about 1 dB below what it shows
MARGINS = dict(oqpsk_10500=14.0, oqpsk_10500_44k1=22.0, oqpsk_8400=5.0, msk_600=8.0, msk_1200=14.0, burst_msk_1200_a=4.5,
               burst_msk_1200_b=1.5, burst_oqpsk_10500=12.0)


def c_round(x):
    """C round(): halves away from zero"""
    return math.copysign(math.floor(abs(x) + 0.5), x)


def hann(nfft):
    n = np.arange(nfft, dtype=np.longdouble)
    return np.longdouble(0.5) - np.longdouble(0.5) * np.cos(2 * LD_PI * n / nfft)


def frame_count(n, nfft):
    return (n - nfft) // (nfft // 2) + 1 if n >= nfft else 0


def spectrum(pcm, nfft, chunk=16):
    """pcm [C, n] int16 -> (sq_mean [C, nfft] float64 of the long-double result, frames); frames added in frame order"""
    pcm = np.atleast_2d(np.asarray(pcm))
    C, n = pcm.shape
    N, hop = nfft, nfft // 2
    F = frame_count(n, N)
    w = hann(N)
    norm = np.sum(w * w) ** 2
    out = np.zeros((C, N))
    for c in range(C):
        x = pcm[c].astype(np.longdouble) / 32768
        acc = np.zeros(N, dtype=np.longdouble)
        for f0 in range(0, F, chunk):
            fs = np.arange(f0, min(F, f0 + chunk))
            fr = x[fs[:, None] * hop + np.arange(N)[None, :]] * w
            X = scipy.fft.fft(fr.astype(np.clongdouble), axis=-1)
            A = np.zeros_like(X)
            A[:, 1:N // 2] = 2 * X[:, 1:N // 2]
            a = scipy.fft.ifft(A, axis=-1)
            Y = scipy.fft.fft(a * a, axis=-1)
            P = (Y.real * Y.real + Y.imag * Y.imag) / norm
            for row in P:
                acc += row
        if F:
            acc /= F
        out[c] = np.fft.fftshift(acc).astype(np.float64)
    return out, F


def _refine(y, k):
    n = len(y)
    y0, y1, y2 = y[(k - 1) % n], y[k % n], y[(k + 1) % n]
    if not (y0 > 0 and y1 > 0 and y2 > 0):
        return 0.0
    l0, l1, l2 = math.log(y0), math.log(y1), math.log(y2)
    den = l0 - 2 * l1 + l2
    if den == 0:
        return 0.0
    return min(0.5, max(-0.5, (l0 - l2) / (2 * den)))


def classify(sq_mean, Fs, threshold_db=5.0, floor_window_hz=400.0, floor_quantile=0.5, fl=None):
    """jaero_ident_classify restated: dict(mode, carrier_hz, fb_hz, line_hz, score_db, margin_db, bins=(i, j unwrapped))"""
    y = np.asarray(sq_mean, dtype=np.float64)
    n = len(y)
    bin_hz = Fs / n
    if fl is None:
        fl = scan_reference.floor(y, Fs, floor_window_hz, floor_quantile)
    Q = np.zeros(n)
    pos = fl > 0
    Q[pos] = y[pos] / fl[pos]
    score, pairs = [], []
    idx = np.arange(n)
    for fb in FBS:
        D = int(c_round(fb * n / Fs))
        part = np.stack([Q[(idx + D + e) % n] for e in (-1, 0, 1)])
        e = np.argmax(part, axis=0)                                  # the first e with the largest Q
        s = np.minimum(Q, part[e, idx])
        i = int(np.argmax(s))                                        # the first i with the largest score
        score.append(float(s[i]))
        pairs.append((i, i + D + int(e[i]) - 1))
    score_db = [10 * math.log10(s) if s > 0 else -math.inf for s in score]
    best = int(np.argmax(score))
    margin = score_db[best] - max(score_db[m] for m in range(4) if m != best)
    i, j = pairs[best]
    di, dj = _refine(y, i), _refine(y, j)
    lo, hi = i + di, j + dj
    mid = (0.5 * (lo + hi) - n // 2) * bin_hz
    return dict(mode=MODES[best] if score_db[best] >= threshold_db else "unknown", best=MODES[best],
                carrier_hz=math.fmod(math.fmod(mid, Fs) + Fs, Fs) / 2, fb_hz=(hi - lo) * bin_hz,
                line_hz=[(lo - n // 2) * bin_hz, (j % n + dj - n // 2) * bin_hz], score_db=dict(zip(MODES, score_db)),
                margin_db=margin, bins=(i, j))
