"""GPU tests: the streaming overlap-save FFT convolution (fastfir.cu, the 8400 bps pre-filter K6 and the burst Hilbert filter) on
caller data through jaero_probe_fastfir, against the long-double reference of tests/fastfir_reference.py.

Every output block must lie within the bound of fastfir_reference (4 log2(nfft) 2^-52 max|H| ||u||_2); outputs before 2L and
every output of an all-zero channel must be exactly 0.0; the output must be bit-identical whatever the write sizes (each block
transform sees the same data); permuting channels permutes the outputs bit for bit, and identical rows give identical outputs.
About six channels per configuration are checked against the reference; the others are held to the bitwise relations."""
import numpy as np
import pytest

import fastfir_reference as fr
from conftest import has_cuda

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

TAPSETS = ("production", "random", "tap0", "tapmid", "taplast")
_worst = {}


def taps_of(tapset, K, nfft):
    if tapset == "production":
        return fr.production_taps(K, nfft)
    if tapset == "random":
        rng = np.random.default_rng(1000 + K)
        return (rng.standard_normal(K) + 1j * rng.standard_normal(K)) / np.sqrt(K)
    h = np.zeros(K, dtype=np.complex128)
    h[{"tap0": 0, "tapmid": (K - 1) // 2, "taplast": K - 1}[tapset]] = 0.3 - 0.7j
    return h


def impulse_positions(K, nfft):
    """K-2, K-1, L-1, L, 2L-1, 2L, and around the oldest sample of block 2's history (the last sample before it is cut)"""
    L, K1 = fr.block_length(K, nfft), K - 1
    return sorted(set([K - 2, K - 1, L - 1, L, 2 * L - 1, 2 * L, 2 * L - K1 - 1, 2 * L - K1, 3 * L - K1 - 1]))


def row(r, K, nfft, n):
    """channel r's input: 0 full-scale int16/32768 real, 1 complex Gaussian, 2 zeros, 3 DC, then one impulse per position of
    impulse_positions, then Gaussian rows of varied scale (every row differs)"""
    imp = impulse_positions(K, nfft)
    rng = np.random.default_rng(7919 * r + K)
    if r == 0:
        return rng.integers(-32768, 32768, n).astype(np.float64) / 32768.0 + 0j
    if r == 1:
        return rng.standard_normal(n) + 1j * rng.standard_normal(n)
    if r == 2:
        return np.zeros(n, dtype=np.complex128)
    if r == 3:
        return np.full(n, 0.25 - 0.5j)
    if r - 4 < len(imp):
        x = np.zeros(n, dtype=np.complex128)
        x[imp[r - 4]] = 0.6 - 0.8j
        return x
    return (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 10.0 ** rng.uniform(-3, 3)


def inputs(C, K, nfft, n):
    return np.stack([row(r, K, nfft, n) for r in range(C)])


def write_patterns(L, n, seed):
    rng = np.random.default_rng(seed)

    def fill(sizes):
        out, left = [], n
        for s in sizes:
            s = min(s, left)
            if s > 0:
                out.append(s); left -= s
        if left > 0:
            out.append(left)
        return out
    singles = [L - 3] + [1] * 6 + [L - 6] + [1] * 6
    rand = []
    while sum(rand) < n:
        rand.append(int(rng.integers(1, 2 * L)))
    return {"whole": [n], "singles": fill(singles), "L-1,L,L+1": fill([L - 1, L, L + 1] * (n // L + 1)),
            "3L+5": fill([3 * L + 5]), "random": fill(rand)}


_ref_cache = {}


def reference(tapset, K, nfft, r, x):
    key = (tapset, K, nfft, r, len(x))
    if key not in _ref_cache:
        taps = taps_of(tapset, K, nfft)
        L = fr.block_length(K, nfft)
        if tapset.startswith("tap"):                    # one tap: y[n] = h x[n - L - k0], exactly a product
            k0 = int(np.nonzero(taps)[0][0])
            y = np.zeros(len(x), dtype=np.clongdouble)
            src = np.arange(2 * L, len(x)) - L - k0
            y[2 * L:] = taps[k0].astype(np.clongdouble) * x[src].astype(np.clongdouble)
        else:
            y = fr.convolve(taps, x, nfft)
        _ref_cache[key] = y
    return _ref_cache[key]


def check_rows(tapset, K, nfft, x, y, rows, what):
    taps = taps_of(tapset, K, nfft)
    L = fr.block_length(K, nfft)
    worst = 0.0
    for r in rows:
        assert not y[r, :2 * L].any(), "%s: row %d: nonzero output before 2L" % (what, r)
        if not x[r].any():
            assert not y[r].any(), "%s: zero row %d: nonzero output" % (what, r)
            continue
        want = reference(tapset, K, nfft, r, x[r])
        for a, b, bound in fr.block_bounds(taps, x[r], nfft):
            err = float(np.sqrt(np.sum(np.abs(y[r, a:b].astype(np.clongdouble) - want[a:b]) ** 2)))
            ratio = err / bound if bound > 0 else (0.0 if err == 0 else np.inf)
            worst = max(worst, ratio)
            assert ratio <= 1.0, "%s: row %d block [%d, %d): error %.3g, bound %.3g" % (what, r, a, b, err, bound)
    key = (K, nfft, tapset)
    _worst[key] = max(_worst.get(key, 0.0), worst)
    print("FASTFIR-STATS K=%d nfft=%d taps=%s %s: worst error / bound = %.3g" % (K, nfft, tapset, what, worst))


def rows_to_check(C, K, nfft):
    imp = impulse_positions(K, nfft)
    rows = [0, 1, 2, 3, C - 1, 4 + (C % max(1, len(imp)))]
    return sorted(set(r for r in rows if r < C))


# 2048 channels (the burst workload's width) run with the production and the random taps
CASES = [(K, nfft, C, t) for t in TAPSETS for K, nfft in fr.SIZES for C in (1, 3, 33, 257)] + \
        [(2048, 8192, 2048, t) for t in ("production", "random")]


@pytest.mark.parametrize("K,nfft,C,tapset", CASES)
def test_fastfir_against_long_double(K, nfft, C, tapset):
    import jaero_b200
    L = fr.block_length(K, nfft)
    n = 6 * L + 37
    x = inputs(C, K, nfft, n)
    taps = taps_of(tapset, K, nfft)
    pats = write_patterns(L, n, seed=K + C)
    if C == 2048 or tapset != "production":
        pats = {k: pats[k] for k in ("whole", "singles")}
    y0 = None
    for name, w in pats.items():
        y = jaero_b200.probe_fastfir(taps, x, nfft, w)
        if y0 is None:
            y0 = y
            check_rows(tapset, K, nfft, x, y, rows_to_check(C, K, nfft), "C=%d" % C)
        else:
            assert np.array_equal(y.view(np.uint64), y0.view(np.uint64)), "writes %s differ from one whole write" % name
        del y
    if C >= 3:
        rng = np.random.default_rng(C)
        perm = rng.permutation(C)
        x2 = x[perm].copy()
        x2[-1] = x2[0]                                  # identical rows
        y2 = jaero_b200.probe_fastfir(taps, x2, nfft, pats["singles"])
        assert np.array_equal(y2[:-1].view(np.uint64), y0[perm[:-1]].view(np.uint64)), "permuted channels"
        assert np.array_equal(y2[-1].view(np.uint64), y2[0].view(np.uint64)), "identical rows"


def test_fastfir_probe_rejects_bad_arguments():
    import jaero_b200
    x = np.ones((2, 100), dtype=np.complex128)
    for K, nfft in ((2048, 4096), (2049, 8192), (2049, 2048)):
        with pytest.raises(jaero_b200.JaeroError, match="no FFT convolution kernel"):
            jaero_b200.probe_fastfir(np.ones(K), x, nfft, [100])
    with pytest.raises(jaero_b200.JaeroError, match="size <= 0"):
        jaero_b200.probe_fastfir(np.ones(2049), x, 4096, [50, 0, 50])
    with pytest.raises(jaero_b200.JaeroError, match="size <= 0"):
        jaero_b200.probe_fastfir(np.ones(2049), x, 4096, [150, -50])
    with pytest.raises(jaero_b200.JaeroError, match="add up to 99"):
        jaero_b200.probe_fastfir(np.ones(2049), x, 4096, [50, 49])


def test_fastfir_probe_frees_its_buffers():
    """eight probes of about 2 GB each leave the device's free memory where it was (a leak would take 16 GB)"""
    import torch
    import jaero_b200
    torch.cuda.init()
    x = np.zeros((2048, 32768), dtype=np.complex128)
    free0, _ = torch.cuda.mem_get_info(0)
    for _ in range(8):
        jaero_b200.probe_fastfir(np.ones(2049), x, 4096, [32768])
    free1, _ = torch.cuda.mem_get_info(0)
    assert free1 >= free0 - (4 << 30), "free memory fell from %d to %d" % (free0, free1)


def test_fastfir_worst_ratios_summary():
    """prints the worst error / bound of every (K, nfft, taps) the cases above measured"""
    for (K, nfft, tapset), w in sorted(_worst.items()):
        print("FASTFIR-WORST K=%d nfft=%d taps=%s: %.3g" % (K, nfft, tapset, w))
