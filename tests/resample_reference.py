"""float64 numpy reference of the PCM rate converter (include/jaero_b200.h, jaero_resample_plan / jaero_resample_create): output
rate input_rate L / M, one low-pass prototype h at L input_rate.

Two forms of the same sum:
- `resample_direct`: the contract as written, zero-stuff by L, filter with h (np.convolve), keep every M-th sample.
- `resample_reference`: the polyphase sum v[m] = sum_r h[phi_m + r L] x[q_m - r], q_m = floor(m M / L), phi_m = m M - q_m L, in
  ascending r, the order the device sums in.
The two agree to rounding (tests/test_resample_cpu.py); the GPU output is checked against `resample_reference`.
"""
import numpy as np


def n_outputs(N, L, M):
    """outputs per channel of N inputs: those m with floor(m M / L) <= N - 1, ceil(N L / M)"""
    return -(-N * L // M)


def phase_table(h, L):
    """[L][R] per-phase taps, row phi = h[phi + r L], zero-padded to R = ceil(K / L)"""
    h = np.asarray(h, dtype=np.float64)
    R = -(-len(h) // L)
    hp = np.zeros((L, R))
    for phi in range(L):
        taps = h[phi::L]
        hp[phi, :len(taps)] = taps
    return hp


def resample_reference(x, h, L, M):
    """x: int16 [C, N] (x[n < 0] = 0). Returns (pcm int16 [C, ceil(N L / M)], value before rounding [C, ...], clipped [C])."""
    x = np.atleast_2d(np.asarray(x)).astype(np.float64)
    C, N = x.shape
    hp = phase_table(h, L)
    R = hp.shape[1]
    m = np.arange(n_outputs(N, L, M), dtype=np.int64)
    q = m * M // L
    phi = m * M - q * L
    xp = np.concatenate([np.zeros((C, R)), x], axis=1)
    v = np.zeros((C, len(m)))
    for r in range(R):
        v += hp[phi, r] * xp[:, q - r + R]
    rv = np.rint(v)
    clipped = ((rv > 32767) | (rv < -32768)).sum(axis=1)
    return np.clip(rv, -32768, 32767).astype(np.int16), v, clipped


def resample_direct(x, h, L, M):
    """The contract term by term: w = x zero-stuffed by L, v = (h * w)[m M] (np.convolve). Returns v [C, ceil(N L / M)]."""
    x = np.atleast_2d(np.asarray(x)).astype(np.float64)
    C, N = x.shape
    Nout = n_outputs(N, L, M)
    out = np.zeros((C, Nout))
    for c in range(C):
        w = np.zeros(N * L)
        w[::L] = x[c]
        out[c] = np.convolve(w, h)[:N * L][::M][:Nout]
    return out
