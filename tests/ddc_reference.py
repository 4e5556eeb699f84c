"""float64 numpy reference of the wideband IQ down-converter (include/jaero_b200.h, jaero_ddc_*).

Two forms of the same chain:
- `ddc_direct`: the contract as written, mix every input sample, then filter and decimate each stage (np.convolve).
- `ddc_reference`: the mix folded into complex stage-1 taps, h1[k] exp(+2 pi i (k T mod 2^32) / 2^32), and one rotation per
  stage-1 output; it evaluates only the samples the decimation keeps and takes a retune schedule.
The two agree to rounding (tests/test_ddc_cpu.py); the GPU output is checked against `ddc_reference`.
"""
import numpy as np

TWO32 = 4294967296


def iq_to_complex(iq, fmt):
    """interleaved cu8 / cs16 -> complex128 per the contract: (v - 127.5) / 128, v / 32768"""
    v = np.asarray(iq).reshape(-1, 2).astype(np.float64)
    v = (v - 127.5) / 128.0 if fmt == "cu8" else v / 32768.0
    return v[:, 0] + 1j * v[:, 1]


def tuning_word(f, fs):
    """round(f / fs * 2^32) mod 2^32, halves away from zero (C llround)"""
    r = float(f) / float(fs) * TWO32
    q = np.floor(abs(r) + 0.5)
    return int(np.copysign(q, r)) % TWO32


def phasor(idx, word):
    """exp(+2 pi i ((idx * word) mod 2^32) / 2^32) for integer sample indices idx >= 0"""
    p = ((np.asarray(idx, dtype=np.uint64) % np.uint64(TWO32)) * np.uint64(word)) % np.uint64(TWO32)
    return np.exp(2j * np.pi * p.astype(np.float64) / TWO32)


def _segments(schedule, lo, hi, step):
    """for a schedule [(first input index, value), ...] (first entry at 0): (value, indices i in [lo, hi) whose input i * step
    falls in the value's span)"""
    out = []
    for s, (start, val) in enumerate(schedule):
        end = schedule[s + 1][0] if s + 1 < len(schedule) else None
        a = max(lo, -(-start // step))
        b = hi if end is None else min(hi, -(-end // step))
        if b > a:
            out.append((val, a, b))
    return out


def ddc_reference(x, h1, D1, h2, D2, T, S, gain=1.0, n_channels=None):
    """x: complex input from sample 0. T, S: per-channel tuning words (sequences), or retune schedules
    [(first input index, words[n_channels]), ...]. Returns (pcm int16 [C, M], value before rounding [C, M], clipped [C],
    v [C, M] complex stage-2 output)."""
    x = np.asarray(x, dtype=np.complex128)
    h1 = np.asarray(h1, dtype=np.float64); h2 = np.asarray(h2, dtype=np.float64)
    N, K1, K2, D = len(x), len(h1), len(h2), D1 * D2
    Tsch = T if (len(T) and isinstance(T[0], tuple)) else [(0, list(T))]
    Ssch = S if (len(S) and isinstance(S[0], tuple)) else [(0, list(S))]
    C = len(Tsch[0][1])
    J = (N - 1) // D1 + 1
    M = (N - 1) // D + 1
    xp = np.concatenate([np.zeros(K1 - 1, dtype=np.complex128), x, np.zeros(D1, dtype=np.complex128)])
    k = np.arange(K1)
    u = np.zeros((C, J), dtype=np.complex128)
    for words, a, b in _segments(Tsch, 0, J, D1):
        words = np.asarray(words, dtype=np.uint64)
        # folded taps, flipped so that row j of the window matrix is xp[j D1 .. j D1 + K1 - 1] = x[j D1 - K1 + 1 .. j D1]
        h1c = np.stack([h1 * phasor(k, w) for w in words])[:, ::-1]
        for j0 in range(a, b, 4096):
            j1 = min(b, j0 + 4096)
            win = np.lib.stride_tricks.as_strided(xp[j0 * D1:], shape=(j1 - j0, K1), strides=(D1 * 16, 16))
            acc = h1c @ win.T
            jj = np.arange(j0, j1) * D1
            u[:, j0:j1] = acc * np.conj(np.stack([phasor(jj, w) for w in words]))
    up = np.concatenate([np.zeros((C, K2 - 1), dtype=np.complex128), u], axis=1)
    idx = np.arange(M) * D2 + K2 - 1
    v = np.zeros((C, M), dtype=np.complex128)
    for kk in range(K2):
        v += h2[kk] * up[:, idx - kk]
    val = np.zeros((C, M))
    for words, a, b in _segments(Ssch, 0, M, D):
        m = np.arange(a, b)
        val[:, a:b] = gain * 32768.0 * np.real(v[:, a:b] * np.stack([phasor(m, w) for w in words]))
    r = np.rint(val)
    clipped = ((r > 32767) | (r < -32768)).sum(axis=1)
    return np.clip(r, -32768, 32767).astype(np.int16), val, clipped, v


def ddc_direct(x, h1, D1, h2, D2, T, S, gain=1.0):
    """The contract formula term by term for fixed tuning words: (value before rounding [C, M], v [C, M])."""
    x = np.asarray(x, dtype=np.complex128)
    N, D = len(x), D1 * D2
    n = np.arange(N)
    vals, vs = [], []
    for t, s in zip(T, S):
        z = x * np.conj(phasor(n, t))
        u = np.convolve(z, h1)[:N][::D1]
        v = np.convolve(u, h2)[:len(u)][::D2]
        m = np.arange(len(v))
        vals.append(gain * 32768.0 * np.real(v * phasor(m, s)))
        vs.append(v)
    assert len(vs[0]) == (N - 1) // D + 1
    return np.array(vals), np.array(vs)


def composite_response(h1, D1, h2, fs, freqs):
    """H(f) = H1(f) H2(f) of the two-stage chain for a complex tone at offset f (H2 runs at fs / D1)"""
    f = np.asarray(freqs, dtype=np.float64)[:, None]
    H1 = np.exp(-2j * np.pi * f * np.arange(len(h1)) / fs) @ np.asarray(h1)
    H2 = np.exp(-2j * np.pi * f * D1 * np.arange(len(h2)) / fs) @ np.asarray(h2)
    return H1 * H2
