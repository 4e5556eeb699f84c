"""GPU test (pytest -m gpu): the streaming FFT convolutions behind the 8400 bps pre-filter and the burst Hilbert filter, and the
burst demodulators behind them, give, bit for bit, the soft bits and full per-channel status recorded in
tests/golden/fastfir_digests.json (tools/make_fastfir_digests.py): 8400 bps OQPSK under writes that cut the 2048-sample
pre-filter blocks at every edge, the three burst modes on streams whose fills complete at and one sample after a 6145-sample
Hilbert block boundary, and the three burst modes on every burst edge stream at once (with AFC off for MSK 1200 and the
squelch on for burst OQPSK as well)."""
import importlib.util
import json
import os

import pytest

from conftest import ROOT, has_cuda

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]


def _tool():
    spec = importlib.util.spec_from_file_location("make_fastfir_digests", os.path.join(ROOT, "tools", "make_fastfir_digests.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


T = _tool()
with open(T.OUT) as fh:
    GOLDEN = json.load(fh)


@pytest.mark.parametrize("name", T.cases())
def test_fastfir_outputs_are_bit_identical(name):
    got = T.run_case(name)
    assert got == GOLDEN[name], "%s: digests differ (%s)" % (name, ", ".join(k for k in GOLDEN[name] if got[k] != GOLDEN[name][k]))
