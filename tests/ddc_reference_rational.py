"""float64 numpy reference of the rational-rate down-converter (include/jaero_b200.h, jaero_ddc_plan_rational /
jaero_ddc_create_rational): output rate Fs_in L / M, stage 1 as in ddc_reference.py, stage 2 a polyphase resampler.

Two forms of the same chain, as for the integer down-converter:
- `ddc_direct_rational`: the contract as written, mix, filter and decimate by D1, zero-stuff by L, filter with h2 and keep every
  M2-th sample (np.convolve).
- `ddc_reference_rational`: stage 1 from `ddc_reference`, then the polyphase sum over the stage-1 rows; it takes retune schedules.
The two agree to rounding (tests/test_ddc_rational_cpu.py); the GPU output is checked against `ddc_reference_rational`.
`tone_response_rational` is the closed-form gain of the chain for a complex tone, images of the zero-stuffing included.
"""
import numpy as np

from ddc_reference import ddc_reference, phasor


def n_outputs_rational(N, L, M):
    """outputs per channel of N inputs at rate L / M: those m with floor(m M / L) <= N - 1, ceil(N L / M)"""
    return -(-N * L // M)


def ddc_reference_rational(x, h1, D1, h2, L, M2, T, S, gain=1.0):
    """The rational down-converter (output rate Fs_in L / (D1 M2)): stage 1 as ddc_reference, then the polyphase form of
    stage 2, v[m] = sum_r h2[phi_m + r L] u[q_m - r] with q_m = floor(m M2 / L), phi_m = m M2 - q_m L, summed in ascending r.
    T, S: tuning words or retune schedules as in ddc_reference; an audio-frequency retune at input s applies to the outputs m
    with floor(m M / L) >= s. Returns (pcm int16 [C, M], value before rounding [C, M], clipped [C], v [C, M])."""
    x = np.asarray(x, dtype=np.complex128)
    h2 = np.asarray(h2, dtype=np.float64)
    N, K2, M = len(x), len(h2), D1 * M2
    Tsch = T if (len(T) and isinstance(T[0], tuple)) else [(0, list(T))]
    Ssch = S if (len(S) and isinstance(S[0], tuple)) else [(0, list(S))]
    C = len(Tsch[0][1])
    # stage 1 alone: ddc_reference with the single-stage h2 = {1} returns u itself
    _, _, _, u = ddc_reference(x, h1, D1, [1.0], 1, Tsch, [0] * C)
    R = -(-K2 // L)
    hp = np.zeros((L, R))
    for phi in range(L):
        taps = h2[phi::L]
        hp[phi, :len(taps)] = taps
    Nout = n_outputs_rational(N, L, M)
    m = np.arange(Nout, dtype=np.int64)
    q = m * M2 // L
    phi = m * M2 - q * L
    up = np.concatenate([np.zeros((C, R), dtype=np.complex128), u], axis=1)
    v = np.zeros((C, Nout), dtype=np.complex128)
    for r in range(R):
        v += hp[phi, r] * up[:, q - r + R]
    val = np.zeros((C, Nout))
    for s, (start, words) in enumerate(Ssch):
        end = Ssch[s + 1][0] if s + 1 < len(Ssch) else None
        a = -(-start * L // M)
        b = Nout if end is None else min(Nout, -(-end * L // M))
        if b > a:
            mm = np.arange(a, b)
            val[:, a:b] = gain * 32768.0 * np.real(v[:, a:b] * np.stack([phasor(mm, w) for w in words]))
    r = np.rint(val)
    clipped = ((r > 32767) | (r < -32768)).sum(axis=1)
    return np.clip(r, -32768, 32767).astype(np.int16), val, clipped, v


def ddc_direct_rational(x, h1, D1, h2, L, M2, T, S, gain=1.0):
    """The rational contract term by term for fixed tuning words: mix, filter and decimate by D1, zero-stuff by L, filter with
    h2 and keep every M2-th sample (np.convolve throughout). Returns (value before rounding [C, M], v [C, M])."""
    x = np.asarray(x, dtype=np.complex128)
    N = len(x)
    n = np.arange(N)
    Nout = n_outputs_rational(N, L, D1 * M2)
    vals, vs = [], []
    for t, s in zip(T, S):
        z = x * np.conj(phasor(n, t))
        u = np.convolve(z, h1)[:N][::D1]
        w = np.zeros(len(u) * L, dtype=np.complex128)
        w[::L] = u
        v = np.convolve(w, h2)[:len(w)][::M2][:Nout]
        assert len(v) == Nout
        m = np.arange(Nout)
        vals.append(gain * 32768.0 * np.real(v * phasor(m, s)))
        vs.append(v)
    return np.array(vals), np.array(vs)


def tone_response_rational(h1, D1, h2, L, fs, freqs, phase):
    """|v| / |u| gain of the rational chain for a complex input tone at f, at an output of polyphase phase `phase`: the x L
    zero-stuffing makes L images f + k fs/D1 of the stage-1 output, each weighted 1/L and rotated by exp(2 pi i k phase / L);
    H2 runs at L fs / D1. Returns |H1(f)| |sum_k H2(f + k fs1) exp(2 pi i k phase / L)| / L."""
    f = np.asarray(freqs, dtype=np.float64)
    fs1 = fs / D1
    H1 = np.exp(-2j * np.pi * f[:, None] * np.arange(len(h1)) / fs) @ np.asarray(h1)
    acc = np.zeros(len(f), dtype=np.complex128)
    for k in range(L):
        g = f + k * fs1
        acc += (np.exp(-2j * np.pi * g[:, None] * np.arange(len(h2)) / (L * fs1)) @ np.asarray(h2)) * np.exp(2j * np.pi * k * phase / L)
    return np.abs(H1) * np.abs(acc) / L
