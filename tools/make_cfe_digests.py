"""SHA-256 digests of what the cluster-resident coarse estimator (cfe_cluster_kernel) returns, epoch by epoch, on seeded rings
of the kinds tests/test_gpu_cfe.py builds: the smoothed spectrum y, the raw estimate and the emitted estimate.

    python tools/make_cfe_digests.py            # writes tests/golden/cfe_cluster_digests.json (needs a GPU)

The fixture pins the kernel's output bit for bit, so that a change to how the kernel schedules its arithmetic (where values sit
between FFT passes, how threads map onto sequences) can be shown to compute exactly what it computed before.
tests/test_gpu_cfe_digest.py recomputes the digests with the same cases and compares them."""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "cfe_cluster_digests.json")

EPOCHS = 6
# name -> (fb, channels, max_clusters). "wide" has more than twice as many channels as an H100 can hold clusters of the
# kernel, so every cluster runs several channels in turn.
CASES = {
    "10500_c7": (10500.0, 7, 0),
    "8400_c7": (8400.0, 7, 0),
    "10500_c20_mc1": (10500.0, 20, 1),
    "10500_c20_mc2": (10500.0, 20, 2),
    "10500_c20_mc7": (10500.0, 20, 7),
    "8400_wide": (8400.0, 160, 0),
}


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def run_case(name):
    """-> dict(clusters=co-resident clusters of the batch, epochs=[dict(y, raw, emitted) digests per epoch])"""
    import cfe_reference as R
    import jaero_b200
    fb, C, max_clusters = CASES[name]
    lockingbw = 10500.0
    b = jaero_b200.DemodBatch("oqpsk", C, fb=fb, lockingbw=lockingbw, fft_power=14)
    try:
        geo = b.cfe_geometry()
        n = geo["bb_len"]
        rng = np.random.default_rng(sum(map(ord, name)))
        kinds = [R.KINDS[c % len(R.KINDS)] for c in range(C)]
        offsets = rng.uniform(-0.4, 0.4, C) * lockingbw / 2
        c = np.arange(C)
        flags = {0: c % 3 == 0, 3: c % 3 == 1}                  # bigchange() before epoch 0 and mid-sequence
        oldests = [0, 1, None, n - 1, n - 2, n - 17]            # the last ones cross the wrap of the ring
        epochs = []
        for e in range(EPOCHS):
            oldest = oldests[e % len(oldests)]
            oldest = int(rng.integers(0, n)) if oldest is None else oldest
            ring = np.stack([R.make_ring(k, n, fb, lockingbw, offsets[ch], rng) for ch, k in enumerate(kinds)])
            bc = np.asarray(flags.get(e, np.zeros(C, dtype=bool)), dtype=np.int32)
            y, raw, emitted = b.probe_cfe(ring, oldest, bc, impl=2, max_clusters=max_clusters)
            epochs.append(dict(y=_sha(y), raw=_sha(raw), emitted=_sha(emitted)))
        return dict(clusters=geo["clusters"], epochs=epochs)
    finally:
        b.close()


if __name__ == "__main__":
    out = {name: run_case(name)["epochs"] for name in CASES}
    with open(OUT, "w") as fh:
        json.dump(out, fh, indent=1, sort_keys=True)
        fh.write("\n")
    print("wrote %s (%d cases x %d epochs)" % (OUT, len(out), EPOCHS))
