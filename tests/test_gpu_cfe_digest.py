"""GPU test (pytest -m gpu): the cluster-resident coarse estimator returns, bit for bit, the smoothed spectrum y, raw estimate and
emitted estimate recorded in tests/golden/cfe_cluster_digests.json (tools/make_cfe_digests.py) for every epoch of seeded rings:
both spectrum shapes, few clusters for many channels, more channels than twice the device's cluster capacity, and bigchange()
before the first and in a later epoch."""
import importlib.util
import json
import os

import pytest

from conftest import ROOT, has_cuda

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]


def _tool():
    spec = importlib.util.spec_from_file_location("make_cfe_digests", os.path.join(ROOT, "tools", "make_cfe_digests.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


T = _tool()
with open(T.OUT) as fh:
    GOLDEN = json.load(fh)


@pytest.mark.parametrize("name", sorted(T.CASES))
def test_cluster_estimator_output_is_bit_identical(name):
    got = T.run_case(name)
    if name == "8400_wide":
        assert T.CASES[name][1] > 2 * got["clusters"], "the case no longer reuses every cluster for several channels"
    assert got["clusters"] > 0, "the cluster estimator cannot run on this device"
    assert len(got["epochs"]) == len(GOLDEN[name])
    for e, (g, want) in enumerate(zip(got["epochs"], GOLDEN[name])):
        assert g == want, "%s epoch %d: digests differ (%s)" % (name, e, ", ".join(k for k in want if g[k] != want[k]))
