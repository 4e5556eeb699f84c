"""CPU tests: pin the long-double trident reference (tests/trident_reference.py) to the restated burst oracles, whose outputs
are themselves pinned to the reference build (test_oracle_golden.py): on every fill of the three burst recordings the
reference's bins are the oracle's, apart from counted near-ties, and its minval lies within the spectrum bound."""
import numpy as np
import pytest

import trident_reference as T
from conftest import load_excerpt
from oracle import restated

RECORDINGS = {"burst_msk_1200_a": ("msk", 1200.0), "burst_msk_1200_b": ("msk", 1200.0), "burst_oqpsk_10500": ("oqpsk", 10500.0)}


def oracle_fills(golden, name):
    """(segments [n, tri_sz], trident_log [n, 5]) of the restated oracle on recording `name`, written as its golden case is"""
    case = golden[name]
    kind, fb = RECORDINGS[name]
    g = T.geometry(kind, fb)
    d = restated.OracleDemod(case["kind"], **case["kw"])
    pcm = load_excerpt(case["excerpt"])
    segs, logs = [], []
    for a in range(0, len(pcm), case["chunk"]):
        d.write(pcm[a:a + case["chunk"]])
        segs.append(d.take_aux(3, cap=1 << 22))
        logs.append(d.take_aux(1, cap=1 << 16))
    d.close()
    segs = np.concatenate(segs).reshape(-1, g["tri_sz"])
    logs = np.concatenate(logs).reshape(-1, 5)
    assert len(segs) == len(logs)
    return segs, logs


@pytest.mark.parametrize("name", sorted(RECORDINGS))
def test_trident_reference_matches_oracle(golden, name):
    kind, fb = RECORDINGS[name]
    g = T.geometry(kind, fb)
    segs, logs = oracle_fills(golden, name)
    assert len(segs) >= 3, "too few trident tests on %s" % name
    spec = T.spectra(segs, g)
    ties = 0
    for e in range(len(segs)):
        r = T.search(kind, fb, spec[e])
        mag = np.abs(spec[e]).astype(np.float64)
        tol = np.stack([np.full(T.N, 2 * T.SPECTRUM_REL * float(np.sqrt(np.sum(mag[w] ** 2)))) for w in range(2)])
        o = logs[e]
        # minval (both kinds) within twice the spectrum bound (the oracle's double FFT and the long-double one)
        assert abs(float(r[1]) - o[1]) <= tol[0][0] + 4 * np.spacing(o[1]), (e, r, o)
        if T.near_tie(kind, fb, mag, tol):
            ties += 1
            continue
        assert int(r[0]) == int(o[0]), (e, r, o)
        assert int(r[2]) == int(o[2]), (e, r, o)
        if kind == "msk":
            assert int(r[3]) == int(o[3]), (e, r, o)
        else:
            assert abs(float(r[3]) - o[3]) <= 8 * tol[0][0], (e, r, o)
    assert ties * 100 <= len(segs), "%d near-ties in %d tests (at most 1 %%)" % (ties, len(segs))
    print("TRIDENT-REF %s: %d tests, %d near-ties" % (name, len(segs), ties))


def test_geometry_matches_kernel_constants():
    assert T.geometry("msk", 1200.0) == dict(tri_sz=8000, base_len=5040, top_len=2960, nfft=32768)
    assert T.geometry("msk", 600.0) == dict(tri_sz=17920, base_len=12000, top_len=5920, nfft=32768)
    assert T.geometry("oqpsk", 10500.0)["base_len"] == 1170
