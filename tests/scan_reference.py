"""float64 numpy restatement of the carrier scanner's contract (include/jaero_b200.h, jaero_scan_* and
jaero_scan_find_carriers): frames, periodic Hann window, np.fft.fft, the in-order sum and max, the sliding floor (np.partition
on the exact window definition), the detector and its measurements. Independent of the library: the tests compare the two."""
import numpy as np

MODE_NOMINAL = {"msk600": 0.594482 * 600, "msk1200": 0.594482 * 1200, "oqpsk8400": 4200.0, "oqpsk10500": 5250.0}
DEFAULTS = dict(threshold_db=3.0, floor_window_hz=100e3, floor_quantile=0.25, min_width_hz=200.0, dc_guard_hz=0.0)


def iq_to_complex(iq, fmt):
    iq = np.asarray(iq)
    if fmt == "cu8":
        v = (iq.astype(np.float64) - 127.5) / 128.0
    else:
        v = iq.astype(np.float64) / 32768.0
    return v[0::2] + 1j * v[1::2]


def hann(nfft):
    return 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(nfft) / nfft)


def frame_powers(x, nfft, hop):
    """[F, nfft] normalised |X_f|^2 in fftshift order, F = the frames complete in x"""
    F = (len(x) - nfft) // hop + 1 if len(x) >= nfft else 0
    w = hann(nfft)
    wss = np.sum(w * w)
    out = np.empty((F, nfft))
    for f0 in range(0, F, 256):
        f1 = min(F, f0 + 256)
        idx = (np.arange(f0, f1)[:, None] * hop) + np.arange(nfft)[None, :]
        X = np.fft.fft(x[idx] * w[None, :], axis=1)
        out[f0:f1] = np.fft.fftshift(np.abs(X) ** 2, axes=1) / wss
    return out


def scan(x, nfft, hop):
    """(mean, max_hold, frames) of the complex stream x, the sum taken frame after frame"""
    P = frame_powers(x, nfft, hop)
    F = P.shape[0]
    if F == 0:
        return np.zeros(nfft), np.zeros(nfft), 0
    s = np.zeros(nfft)
    for f in range(F):
        s += P[f]
    return s / F, P.max(axis=0), F


def freqs(nfft, rate):
    return (np.arange(nfft) - nfft // 2) * (rate / nfft)


def window_len(nfft, rate, floor_window_hz):
    x = min(floor_window_hz / (rate / nfft), float(nfft))
    return int(min(max(2 * int(np.floor(x / 2)) + 1, 3), nfft))


def floor(psd, rate, floor_window_hz=100e3, floor_quantile=0.25):
    n = len(psd)
    W = window_len(n, rate, floor_window_hz)
    k = int(np.floor((W - 1) * floor_quantile))
    out = np.empty(n)
    for i in range(n):
        s = min(max(i - (W - 1) // 2, 0), n - W)
        out[i] = np.partition(psd[s:s + W], k)[k]
    return out


def mode_hint(width):
    if not width > 0:
        return "unknown"
    best = min(MODE_NOMINAL, key=lambda m: abs(np.log(width / MODE_NOMINAL[m])))
    r = width / MODE_NOMINAL[best]
    return best if 0.8 <= r <= 1.25 else "unknown"


def find_carriers(psd, rate, fl=None, **params):
    p = dict(DEFAULTS, **params)
    psd = np.asarray(psd, dtype=np.float64)
    n = len(psd)
    bin_hz = rate / n
    fl = floor(psd, rate, p["floor_window_hz"], p["floor_quantile"]) if fl is None else fl
    e = psd - fl
    occ = psd >= fl * 10 ** (p["threshold_db"] / 10.0)
    hz = lambda i: (i - n // 2) * bin_hz
    out, i = [], 0
    while i < n:
        if not occ[i]:
            i += 1
            continue
        i1 = i
        while i1 + 1 < n and occ[i1 + 1]:
            i1 += 1
        if (i1 - i + 1) * bin_hz >= p["min_width_hz"]:
            r = np.arange(i, i1 + 1)
            pk = i + int(np.argmax(psd[i:i1 + 1]))
            se = float(np.sum(e[r]))
            er = e[i:i1 + 1]
            top = 0.0
            for v in er[er >= 0.5 * np.max(er)]:                    # in bin order, as the library adds them
                top += v
            h = 0.5 * (top / np.count_nonzero(er >= 0.5 * np.max(er)))
            j = pk + 1
            while j < n and e[j] >= h:
                j += 1
            xr = n - 1 if j == n else (j - 1) + (e[j - 1] - h) / (e[j - 1] - e[j])
            j = pk - 1
            while j >= 0 and e[j] >= h:
                j -= 1
            xl = 0 if j < 0 else (j + 1) - (e[j + 1] - h) / (e[j + 1] - e[j])
            c = dict(peak_hz=hz(pk), center_hz=float(np.sum(hz(r) * e[r])) / se if se > 0 else hz(pk), lo_hz=hz(i), hi_hz=hz(i1),
                     width_hz=(xr - xl) * bin_hz, power=se / n, snr_db=10 * np.log10(se / np.sum(fl[r])),
                     peak_db=10 * np.log10(np.max(psd[r] / fl[r])), floor=fl[pk], lo=i, hi=i1)
            c["mode"] = mode_hint(c["width_hz"])
            c["flags"] = (1 if abs(c["center_hz"]) < p["dc_guard_hz"] else 0) | (2 if (i == 0 or i1 == n - 1) else 0)
            # the largest term of each sum, the scale the comparison with the library is made on
            c["_scale"] = dict(center_hz=(float(np.max(np.abs(hz(r) * e[r]))) + abs(c["center_hz"]) * float(np.max(np.abs(e[r])))) / se
                               if se > 0 else bin_hz,
                               power=float(np.max(np.abs(e[r]))) / n, snr_db=1.0, peak_db=1.0,
                               width_hz=bin_hz, peak_hz=bin_hz, lo_hz=bin_hz, hi_hz=bin_hz, floor=abs(fl[pk]))
            out.append(c)
        i = i1 + 1
    return out
