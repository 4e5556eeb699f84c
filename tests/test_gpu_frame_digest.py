"""GPU test (pytest -m gpu): the P-channel, C-channel and R/T frame layers return, bit for bit, the records, per-read counts,
stats and demodulator DCD recorded in tests/golden/frame_digests.json (tools/make_frame_digests.py): P at 10500, 1200 and
600 bps and C at 8400 bps through write_batch and through process_softbits cut across the fast-path / bit-serial edges, and
R/T on the three burst recordings through process_burst (vector mode off and on) and through host soft bits with
start-of-burst markers, with ticks and lost-signal events at fixed points."""
import importlib.util
import json
import os

import pytest

from conftest import ROOT, has_cuda

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]


def _tool():
    spec = importlib.util.spec_from_file_location("make_frame_digests", os.path.join(ROOT, "tools", "make_frame_digests.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


T = _tool()
with open(T.OUT) as fh:
    GOLDEN = json.load(fh)


@pytest.mark.parametrize("name", T.cases())
def test_frame_layer_outputs_are_bit_identical(name):
    got = T.run_case(name)
    assert got == GOLDEN[name], "%s: digests differ (%s)" % (name, ", ".join(k for k in GOLDEN[name] if got[k] != GOLDEN[name][k]))
