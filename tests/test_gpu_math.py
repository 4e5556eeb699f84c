"""GPU tests: the demodulators' device arithmetic primitives (demod_device.cuh, cfe.cu), compiled with the product's flags and run
through jaero_probe_math / jaero_probe_osc, against the exact, glibc and long-double references of tests/math_reference.py.

- div_exact: bit-equal to the IEEE quotient where that is normal (-0 / d gives +0); within 1 ulp where it is subnormal.
- div_fast, in both units that compile it: bit-equal to the IEEE quotient on the domains of its three call sites.
- atan2_fast: <= 1 ulp from glibc's atan2 and <= 1.5 ulp from atan2l; the arguments it forwards are bit-equal to glibc.
- hypot_fast: <= 2 ulp from glibc's hypot. log10_ge1 as cfe.cu compiles it: <= 2 ulp from glibc, exactly k at 10^k.
- osc_index, q_round, fmod360: bit-equal to the reference's x86 behaviour over the whole double range.
- The Osc helpers: bit-equal, in every logged field, to the reference's own WaveTable running the same scripts."""
import numpy as np
import pytest

import jaero_b200
import math_reference as mr
from conftest import has_cuda
from oracle import ref

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]
needs_script = pytest.mark.skipif(not ref.wavetable_script_available() if ref.available() else True,
                                  reason="oracle/_ref/libjaero_ref.so has no jref_wavetable_script")
FINITE_NORMAL_MIN = 2.2250738585072014e-308


def _report(name, **kv):
    print("\n%s: %s" % (name, ", ".join("%s=%s" % (k, v) for k, v in kv.items())))


def _first_bad(ok, *cols):
    i = np.nonzero(~ok)[0][:8]
    return [tuple(float(c[k]) for c in cols) for k in i]


def test_div_exact_is_the_ieee_quotient():
    x, d = mr.div_exact_cases()
    got = jaero_b200.probe_math(mr.DIV_EXACT, x, d)
    want = x / d
    negzero = (x == 0) & np.signbit(x)
    assert negzero.sum() > 0
    assert np.all((got[negzero] == 0) & ~np.signbit(got[negzero])), "-0 / d must come out as +0"
    ok = mr.same_bits(got, np.where(negzero, 0.0, want))
    sub = np.abs(want) < FINITE_NORMAL_MIN
    dist = mr.ulp_distance(got, want)
    _report("div_exact", operands=len(x), subnormal_quotients=int(sub.sum()), mismatches_subnormal=int((~ok & sub).sum()),
            worst_ulp_subnormal=float(dist[sub].max()))
    assert ok[~sub].all(), _first_bad(ok | sub, x, d, got, want)
    assert dist[sub].max() <= 1                                   # a subnormal quotient's remainder is not exact: within 1 ulp


@pytest.mark.parametrize("op", [mr.DIV_FAST, mr.DIV_FAST_CFE], ids=["demod_kernels", "cfe"])
def test_div_fast_is_the_ieee_quotient_on_its_call_sites(op):
    a, b, dom = mr.div_fast_cases()
    got = jaero_b200.probe_math(op, a, b)
    with np.errstate(all="ignore"):
        want = a / b
    ok = mr.same_bits(got, want)
    outside = dom == 3
    _report("div_fast (%s)" % ("cfe.cu" if op == mr.DIV_FAST_CFE else "demod_kernels.cu"), operands=len(a),
            mismatches_in_domain=int((~ok & ~outside).sum()), mismatches_outside=int((~ok & outside).sum()),
            worst_ulp_in_domain=float(mr.ulp_distance(got[~outside], want[~outside]).max()),
            bad_by_domain=[int((~ok & (dom == k)).sum()) for k in range(4)], first=_first_bad(ok | outside, a, b, got, want))
    assert ok[~outside].all(), _first_bad(ok | outside, a, b, got, want)


def test_atan2_fast_is_within_one_ulp_of_glibc():
    y, x = mr.atan2_cases()
    got = jaero_b200.probe_math(mr.ATAN2_FAST, y, x)
    want = mr.atan2_glibc(y, x)
    ay, ax = np.abs(y), np.abs(x)
    with np.errstate(invalid="ignore"):
        fwd = ~(ax > 0) | ~(ay > 0) | ~(ax < 1e300) | ~(ay < 1e300) | (ax < 1e-290) | (ay < 1e-290)
    ok = mr.same_bits(got, want)
    special = ~np.isfinite(y) | ~np.isfinite(x) | (y == 0) | (x == 0)
    assert ok[special].all(), _first_bad(ok | ~special, y, x, got, want)       # zero signs and NaN / inf results are glibc's
    fdist = mr.ulp_distance(got[fwd & ~special], want[fwd & ~special])        # the device library beyond the 1e-290 / 1e300 gates
    dist = mr.ulp_distance(got[~fwd], want[~fwd])
    ld = mr.atan2_ld(y[~fwd], x[~fwd])
    err = mr.ulp_error(got[~fwd], ld)
    _report("atan2_fast", operands=len(y), forwarded=int(fwd.sum()), worst_ulp_glibc=float(dist.max()), library_beyond_gates_worst_ulp=float(fdist.max()),
            worst_ulp_atan2l=float(err.max()), beyond_1ulp_atan2l=int((err > 1).sum()), glibc_worst_atan2l=float(mr.ulp_error(want[~fwd], ld).max()))
    assert dist.max() <= 1, _first_bad(dist <= 1, y[~fwd], x[~fwd], got[~fwd], want[~fwd])
    assert err.max() <= 1.5
    assert fdist.max() <= 2                                                    # CUDA's atan2: 2 ulp


def test_hypot_fast_is_within_two_ulp_of_glibc():
    x, y, dom = mr.hypot_cases()
    got = jaero_b200.probe_math(mr.HYPOT_FAST, x, y)
    want = mr.hypot_glibc(x, y)
    dist = mr.ulp_distance(got, want)
    nz = want > 0
    _report("hypot_fast", operands=len(x), worst_ulp_glibc_call_site=float(dist[dom == 0].max()),
            worst_ulp_glibc_wide=float(dist[dom == 1].max()), worst_ulp_hypotl=float(mr.ulp_error(got[nz], mr.hypot_ld(x[nz], y[nz])).max()))
    assert dist.max() <= 2, _first_bad(dist <= 2, x, y, got, want)


def test_log10_ge1_as_the_estimator_compiles_it():
    x = mr.log10_cases()
    got = jaero_b200.probe_math(mr.LOG10_GE1, x)
    want = mr.log10_glibc(x)
    dist = mr.ulp_distance(got, want)
    nz = x > 1
    _report("log10_ge1 (cfe.cu)", operands=len(x), worst_ulp_glibc=float(dist.max()),
            worst_ulp_log10l=float(mr.ulp_error(got[nz], mr.log10_ld(x[nz])).max()))
    assert got[x == 1.0][0] == 0.0 and not np.signbit(got[x == 1.0][0])
    p10 = mr.powers_of_ten()
    assert np.array_equal(jaero_b200.probe_math(mr.LOG10_GE1, p10), np.arange(23, dtype=np.float64))
    assert dist.max() <= 2, _first_bad(dist <= 2, x, got, want)


@pytest.mark.parametrize("op", [mr.OSC_INDEX, mr.Q_ROUND, mr.FMOD360], ids=["osc_index", "q_round", "fmod360"])
def test_conversions_are_bit_equal_to_the_x86_reference(op):
    """over the whole double range, NaN, infinities and values outside the int range included"""
    x = {mr.OSC_INDEX: mr.osc_index_cases, mr.Q_ROUND: mr.q_round_cases, mr.FMOD360: mr.fmod360_cases}[op]()
    got = jaero_b200.probe_math(op, x)
    with np.errstate(invalid="ignore"):
        want = {mr.OSC_INDEX: lambda: mr.wt_index(x).astype(np.float64), mr.Q_ROUND: lambda: mr.qround_x86(x).astype(np.float64),
                mr.FMOD360: lambda: np.fmod(x, 360.0)}[op]()
    ok = mr.same_bits(got, want)
    assert ok.all(), _first_bad(ok, x, got, want)


@needs_script
@pytest.mark.parametrize("samplerate,n_lanes", [(48000.0, 4096), (44100.0, 1024)])
def test_oscillator_scripts_are_bit_equal_to_the_reference_wavetable(samplerate, n_lanes):
    op, arg = mr.osc_scripts(seed=int(samplerate), n_lanes=n_lanes, n_ops=256, samplerate=samplerate)
    dev = jaero_b200.probe_osc(op, arg, samplerate)
    want = ref.wavetable_script(op, arg, samplerate)
    # the one deviation is div_exact's: where the reference computes -0 (SetPhaseDeg(-360 k) for WTptr, SetFreq(-0) for WTstep)
    # the device has +0. The zero's sign travels into last_WTptr, and a point passed with a -0 step gives the fraction t / -0
    # there and t / +0 here, infinities of opposite signs
    negzero = lambda v: (v == 0) & np.signbit(v)
    for f, name in ((0, "ptr"), (1, "last"), (2, "step"), (3, "freq"), (5, "passed"), (6, "fraction")):
        ok = mr.same_bits(dev[..., f], want[..., f]) | (negzero(want[..., f]) & (dev[..., f] == 0))
        if f == 6:                                                # the step at the latest passed point, whose fraction is logged
            k = np.where(want[..., 5] == 1, np.arange(op.shape[1]), 0)
            step_then = np.take_along_axis(want[..., 2], np.maximum.accumulate(k, axis=1), axis=1)
            ok |= negzero(step_then) & np.isinf(want[..., 6]) & (dev[..., 6] == -want[..., 6])
        if not ok.all():
            l, k = np.argwhere(~ok)[0]
            pytest.fail("%s differs first at lane %d op %d (%d, arg %r): device %r, reference %r; script ops %s"
                        % (name, l, k, op[l, k], arg[l, k], dev[l, k, f], want[l, k, f], op[l, max(0, k - 4):k + 1].tolist()))
    assert np.array_equal(dev[..., 4], want[..., 4]), "table index differs"
    sin_t, cos_t = np.zeros(mr.WTSIZE), np.zeros(mr.WTSIZE)
    ref.lib().jref_trig_tables(ref._p(sin_t), ref._p(cos_t))
    idx = dev[..., 4].astype(np.int64)
    assert np.array_equal(cos_t[idx], want[..., 7]) and np.array_equal(sin_t[idx], want[..., 8])
    _report("osc scripts @%g" % samplerate, lanes=n_lanes, ops=op.size, wrapped_frames=int(((op == mr.NEXT_FRAME) & (want[..., 0] < want[..., 1])).sum()),
            passed_points=int(want[..., 5].sum()), pointers_beyond_int=int((np.abs(want[..., 0]) >= 2.0 ** 31).sum()))


def test_probes_reject_bad_arguments():
    x = np.ones(4)
    with pytest.raises(jaero_b200.JaeroError, match="unknown op"):
        jaero_b200.probe_math(9, x, x)
    with pytest.raises(jaero_b200.JaeroError, match="null argument"):
        jaero_b200.probe_math(mr.DIV_EXACT, x)
    with pytest.raises(jaero_b200.JaeroError, match="unknown op"):
        jaero_b200.probe_osc(np.array([[0, 8]]), np.zeros((1, 2)), 48000.0)
    with pytest.raises(jaero_b200.JaeroError, match="samplerate"):
        jaero_b200.probe_osc(np.array([[0]]), np.zeros((1, 1)), 0.0)
