"""CPU checks of tests/math_reference.py, the reference side of tests/test_gpu_math.py: the ulp helpers, the x86 conversion model
against the reference build's own qRound and WaveTable, the generators' claims, and the build flags the primitives rely on."""
import math
import os
import re
from fractions import Fraction

import numpy as np
import pytest

import math_reference as mr
from conftest import ROOT
from oracle import ref

needs_ref = pytest.mark.skipif(not ref.available(), reason="oracle/_ref not built (needs /root/reference)")
needs_script = pytest.mark.skipif(not ref.wavetable_script_available() if ref.available() else True,
                                  reason="oracle/_ref/libjaero_ref.so has no jref_wavetable_script")


def test_ulp_distance_on_known_pairs():
    cases = [(1.0, 1.0, 0), (0.0, -0.0, 0), (1.0, np.nextafter(1.0, 2.0), 1), (1.0, np.nextafter(1.0, 0.0), 1),
             (5e-324, -5e-324, 2), (0.0, 5e-324, 1), (2.0, 1.0, 2 ** 52), (-1.0, 1.0, 2 * 0x3FF0000000000000),
             (1.7976931348623157e308, np.inf, 1), (np.nextafter(2.0, 0.0), np.nextafter(2.0, 3.0), 2)]
    for a, b, d in cases:
        assert mr.ulp_distance(np.array([a]), np.array([b]))[0] == d, (a, b)
    assert mr.ulp_error(np.array([1.0 + 2 ** -52]), np.array([1.0], dtype=np.longdouble))[0] == 1.0
    assert mr.ulp_error(np.array([1.0]), np.longdouble(1.0) + np.longdouble(2.0) ** -54)[0] == 0.25
    assert mr.ulp_error(np.array([5e-324]), np.array([0.0], dtype=np.longdouble) + np.longdouble(2.0) ** -1075)[0] == 0.5
    assert mr.same_bits(np.array([np.nan, 0.0, -0.0]), np.array([-np.nan, 0.0, 0.0])).tolist() == [True, True, False]


def test_x86_int_model():
    d = np.array([0.9, -0.9, 2147483647.9, 2147483648.0, -2147483648.9, -2147483649.0, np.nan, np.inf, -np.inf, 1e300, -0.0])
    assert mr.x86_int(d).tolist() == [0, 0, 2147483647, mr.INT_MIN, -2147483648, mr.INT_MIN, mr.INT_MIN, mr.INT_MIN, mr.INT_MIN,
                                      mr.INT_MIN, 0]
    assert mr.wt_index(np.array([0.0, 19998.9, 19999.0, -0.5, -1.0, np.nan, 3e9])).tolist() == [0, 19998, 0, 0, 19998, 19998, 19998]


@needs_ref
def test_x86_rule_agrees_with_the_reference_qround():
    """the Python model of qRound with x86 conversions equals the reference build's own qRound (jref_qround) on the q_round
    operand set, including NaN, infinities and values outside the int range"""
    d = mr.q_round_cases(n=1 << 14)
    L = ref.lib()
    want = np.array([L.jref_qround(float(v)) for v in d])
    got = mr.qround_x86(d)
    bad = np.nonzero(want != got)[0]
    assert len(bad) == 0, [(d[i], want[i], got[i]) for i in bad[:10]]
    assert want[d == 2147483648.0][0] == mr.INT_MIN and want[d == 0.49999999999999994][0] == 1   # d + 0.5 rounds up to 1.0


def test_near_midpoint_numerators_are_as_close_as_the_divisor_allows():
    rng = np.random.default_rng(0)
    for d in (3, 5, 6, 7, 45, 75, 360, 400, 401, 19999, 48000, 192000, 131071):
        o = mr.odd_part(d)
        for x in mr.near_midpoint_numerators(rng, d, 16):
            assert mr.midpoint_distance(x, d) == Fraction(1, 2 * o), (x, d)
            q = Fraction(float(x)) / d
            assert abs(q) >= Fraction(2) ** -1022 and math.isfinite(x)
    assert Fraction(1, 2 * mr.odd_part(131071)) < Fraction(1, 2 ** 17)


def test_divisor_sets():
    ds = mr.production_divisors()
    for d in (360, 19999, 48000, 192000, 4 * 48000, 96000, 800, 401, 400, 600, 80, 41, 40, 21, 5040, 6000, 75, 128):
        assert d in ds, d
    x, d = mr.div_exact_cases()
    assert set(np.arange(1, 2 ** 17 + 1)) <= set(d.tolist())
    assert np.all(np.isfinite(x)) and np.any(x == 0) and np.any(np.signbit(x) & (x == 0))
    assert np.any((x != 0) & (np.abs(x) < 2.2250738585072014e-308)) and np.any(np.abs(x) > 1e308)


def test_div_fast_domains():
    a, b, dom = mr.div_fast_cases(n=1 << 12)
    assert np.all(a[dom == 0] == mr.AGC_NUMERATOR) and b[dom == 0].min() >= 1e-6 and b[dom == 0].max() <= 1e6 * (1 + 1e-15)
    assert np.all((b[dom == 1] >= 2) & (b[dom == 1] < 3) & (np.abs(a[dom == 1]) <= b[dom == 1]))
    q = a[dom == 2] / b[dom == 2]
    assert np.all((b[dom == 2] > 1e-290) & (np.abs(q) <= 1) & (np.abs(q) >= 2.2250738585072014e-308) &
                  (np.abs(a[dom == 2]) >= 2.0 ** -968))


def test_atan2_cases_reach_every_branch():
    y, x = mr.atan2_cases(n=1 << 14)
    ay, ax = np.abs(y), np.abs(x)
    fin = np.isfinite(y) & np.isfinite(x) & (ay > 0) & (ax > 0)
    mn, mx = np.minimum(ay, ax)[fin], np.maximum(ay, ax)[fin]
    for r in (0.4375, 0.6875):
        assert np.any(mn == r * mx) and np.any(mn == np.nextafter(r * mx, 0)) and np.any(mn == np.nextafter(r * mx, np.inf))
    assert np.any(mn == mx)
    for g in (1e-290, 1e300):
        for v in (np.nextafter(g, 0), g, np.nextafter(g, np.inf)):
            assert np.any(ax == v) and np.any(ay == v)
    for sy in (1, -1):
        for sx in (1, -1):
            assert np.any(fin & (np.sign(y) == sy) & (np.sign(x) == sx))
    assert np.any(np.isnan(y)) and np.any(np.isinf(x)) and np.any((y == 0) & np.signbit(y))


def test_log10_and_index_cases():
    x = mr.log10_cases(n=1 << 10)
    assert np.all(x >= 1) and 1.0 in x and all(v in x for v in mr.powers_of_ten())
    assert np.nextafter(math.sqrt(2.0) * 2.0 ** 100, 0) in x
    p = mr.osc_index_cases(n=1 << 10)
    assert all(np.any(p == v) for v in (0.0, 19998.0, 19999.0, 20000.0, 2147483647.0, 2147483648.0, np.inf, -np.inf))
    assert np.any(np.isnan(p)) and np.any(p == np.nextafter(19999.0, 0))
    assert np.any((p == 0) & np.signbit(p))


@needs_script
def test_osc_scripts_exercise_every_operation_after_a_wrap():
    """every operation runs right after a frame that wrapped the pointer, and the tame lanes keep their pointers in the table"""
    op, arg = mr.osc_scripts(n_lanes=256, n_ops=256)
    log = ref.wavetable_script(op, arg, 48000.0)
    wrapped = (op[:, :-1] == mr.NEXT_FRAME) & (log[:, :-1, 0] < log[:, :-1, 1])
    for o in mr.OSC_OPS:
        assert np.any(wrapped & (op[:, 1:] == o)), o
    tame = np.arange(256) % 4 != 3
    assert np.all(log[tame, :, 0] <= mr.WTSIZE) and np.all(log[tame, :, 0] >= 0)
    assert np.any(log[~tame, :, 0] >= 2.0 ** 31) and np.any(np.isnan(log[~tame, :, 0]))
    assert np.any(log[:, :, 5] == 1)
    # the model of the table index is the reference's, wherever the pointer is
    idx = np.where(op == mr.NEXT_INDEX, -1, mr.wt_index(log[:, :, 0]))
    sel = op != mr.NEXT_INDEX
    assert np.array_equal(idx[sel], log[:, :, 4][sel])


def test_primitives_are_built_with_the_flags_they_rely_on():
    """every unit that calls div_exact, atan2_fast, q_round or an osc_* helper is compiled with -fmad=false, so that a*b+c rounds as
    the reference's x86 build rounds it; cfe.cu, compiled with contraction, calls none of them (log10_ge1 and div_fast only)"""
    from jaero_b200 import build
    units = dict(build.UNITS)
    csrc = os.path.join(ROOT, "jaero_b200", "csrc")
    uses = re.compile(r"\b(div_exact|atan2_fast|q_round|osc_[a-z_]+)\s*\(")
    src = {f: open(os.path.join(csrc, f)).read() for f in os.listdir(csrc) if f.endswith(".cu")}
    includes = {f: set(re.findall(r'#include "([a-z_]+\.cu)"', s)) for f, s in src.items()}
    calls = {f for f, s in src.items() if uses.search(s)}
    assert {"msk_pipe.cu", "oqpsk_pipe.cu", "oqpsk_demod.cu", "burst.cu", "prefilter.cu", "demod_kernels.cu"} <= calls
    for f in calls:
        owners = [u for u in units if u == f or f in includes[u]]
        assert owners, f + " is compiled by no unit"
        for u in owners:
            assert "-fmad=false" in units[u], (u, f)
    assert "cfe.cu" not in calls and "-fmad=false" not in units["cfe.cu"]
