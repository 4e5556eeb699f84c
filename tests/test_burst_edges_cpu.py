"""The burst edge-test streams (tests/burst_edge_streams.py) on the CPU: the oracle's fill log agrees with what the trident log
shows, every stream places its trident-buffer fills where the GPU tests need them, the 600 bps stretched streams acquire, and
the 300-channel layout really puts more trident events in one internal chunk than one trident launch takes."""
import numpy as np
import pytest

import burst_edge_streams as S
from oracle import restated


@pytest.mark.parametrize("mode", list(S.MODES))
def test_fill_log_agrees_with_trident_log(mode):
    """take_aux(2) holds the stream index of the sample at which each trident test ran: written in 16-sample pieces, the trident
    log grows in exactly the piece that holds that index, and writing in other pieces gives the same indices."""
    m = S.MODES[mode]
    x = S.base_stream(mode)[:160000 if mode != "msk600" else 420000]
    d = restated.OracleDemod(m["kind"], **m["kw"])
    seen = []
    for a in range(0, len(x), 16):
        d.write(x[a:a + 16])
        seen += [a] * (len(d.take_aux(1)) // 5)
    f = d.take_aux(2).astype(np.int64)
    d.close()
    assert len(f) == len(seen) >= 2
    assert np.array_equal(f // 16 * 16, seen)
    assert f[0] == m["tri_sz"]                                   # the first fill completes one buffer length into the stream
    assert np.array_equal(S.oracle_fills(mode, x, S.cycle_writes(S.P2, len(x)))[0], f)


@pytest.mark.parametrize("rec", ["burst_msk_1200_a", "burst_msk_1200_b"])
def test_stretched_600_streams_acquire(rec):
    f, acc, soft = S.oracle_fills("msk600", S.stretched_600(rec))
    assert int((soft < 0).sum()) >= 2 and int(acc.sum()) >= 2


@pytest.mark.parametrize("mode", list(S.MODES))
def test_streams_place_their_fills(mode):
    m = S.MODES[mode]
    v = S.variants(mode)
    n = len(v["base"])
    fills = {k: S.oracle_fills(mode, x) for k, x in v.items()}
    f0, acc0, soft0 = fills["base"]
    A = f0[acc0]
    assert len(A) >= 2 and int((soft0 < 0).sum()) >= 2
    # the frequency-offset replicas acquire the same bursts at (nearly) the same samples
    for k in ("off0", "off1"):
        f, acc, soft = fills[k]
        assert int(acc.sum()) == len(A) and np.abs(f[acc] - A).max() <= 2 and int((soft < 0).sum()) == len(A)
    # an accepted fill on the last and on the first sample of a P4 internal chunk
    starts = {s for s, _ in S.chunk_spans(S.cycle_writes(S.P4, n))}
    (fl, al, _), (ff, af, _) = fills["chunk_last"], fills["chunk_first"]
    assert any(int(t) + 1 in starts for t in fl[al]) and any(int(t) in starts for t in ff[af])
    b = min(starts, key=lambda s: abs(s - A[0]))
    assert b - 1 in fl[al] and b in ff[af]
    # ... and at a Hilbert block edge and one sample after it
    (fh, ah, _), (fh1, ah1, _) = fills["hil_edge"], fills["hil_edge1"]
    h = int(round(A[-1] / S.HIL_L)) * S.HIL_L
    assert h in fh[ah] and h + 1 in fh1[ah1] and h % S.HIL_L == 0
    # the stream that starts inside a burst: that burst is not acquired, the recording's last one still is
    fi, ai, si = fills["inside"]
    s = int(A[0]) - m["tri_sz"] // 2
    assert not (fi[ai] < 2 * m["tri_sz"]).any() and np.abs(fi[ai] - (A[-1] - s)).min() <= 2 and int((si < 0).sum()) >= 1
    # two recorded bursts closer together than in the recording, both acquired
    _, planned, first = S.splice(mode, v["base"], A)
    fs, as_, _ = fills["splice"]
    k = S.SPLICE_PAIR[mode]
    assert first in fs[as_] and np.abs(fs[as_] - planned).min() <= 200
    assert planned - first < A[k + 1] - A[k]
    # consecutive fills never complete closer than tri_sz + 1 samples: at most 7 (burst OQPSK), 3 (MSK 1200) or 1 (MSK 600)
    # per internal chunk, inside the 8 trident-buffer slots per channel
    for f, _, _ in fills.values():
        assert np.diff(f).min() >= m["tri_sz"] + 1
    assert (S.CHUNK - 1) // (m["tri_sz"] + 1) + 1 == {"msk1200": 3, "msk600": 1, "oqpsk": 7}[mode]


def test_dense_stream_fills_an_internal_chunk_to_the_bound():
    """the burst OQPSK gated carrier completes a fill every tri_sz + 1 samples at its closest, and 7 fills (every one of them
    accepted) inside one P4 internal chunk: the most any stream can put there"""
    f, acc, soft = S.oracle_fills("oqpsk", S.variants("oqpsk")["dense"])
    assert np.diff(f).min() == S.MODES["oqpsk"]["tri_sz"] + 1
    spans = S.chunk_spans(S.cycle_writes(S.P4, len(S.variants("oqpsk")["dense"])))
    best = max(spans, key=lambda sp: int(((f >= sp[0]) & (f < sp[1])).sum()))
    inside = (f >= best[0]) & (f < best[1])
    assert int(inside.sum()) == 7 and acc[inside].all()
    assert int((soft < 0).sum()) >= 100


@pytest.mark.parametrize("mode", list(S.MODES))
def test_layout_b_crosses_a_trident_round(mode):
    """more than EV_ROUND channels of the 300-channel layout complete an accepted fill inside one internal chunk (P1 writes),
    so a second trident launch has to run for it"""
    names, idx = S.layout_b(mode)
    v = S.variants(mode)
    assert len(idx) == S.N_LAYOUT_B and set(idx) == set(range(len(names)))
    acc_fills = {k: (lambda r: r[0][r[1]])(S.oracle_fills(mode, v[k])) for k in names}
    spans = S.chunk_spans(S.cycle_writes(S.P1, len(v["base"])))
    per_chunk = [sum(int(((acc_fills[names[i]] >= s0) & (acc_fills[names[i]] < s1)).any()) for i in idx) for s0, s1 in spans]
    assert max(per_chunk) > S.EV_ROUND
