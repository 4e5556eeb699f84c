"""References and hard-case operand generators for the demodulators' device arithmetic primitives (demod_device.cuh, cfe.cu),
which tests/test_gpu_math.py runs through jaero_probe_math / jaero_probe_osc.

- Exact: numpy float64 `/` (IEEE, correctly rounded) and np.fmod (exact).
- libm: glibc through math.atan2 / math.hypot / math.log10, one element at a time (np.arctan2 on float64 may take numpy's own
  SIMD code instead of glibc).
- Long double: np.longdouble (x87, 64-bit significand) through atan2l / hypotl / log10l.
- x86 conversions: (int)d as the reference's x86-64 build evaluates it (cvttsd2si): truncation where -2^31 - 1 < d < 2^31,
  INT_MIN otherwise and for NaN. The device's own conversion saturates and gives 0 for NaN, so the primitives that stand for
  the reference's (int) (osc_index, q_round, the oscillator wrap loops) must follow this rule to stay bit-equal."""
import math
from fractions import Fraction

import numpy as np

assert np.finfo(np.longdouble).nmant >= 63, "the long-double references need x87 extended precision"

WTSIZE = 19999
INT_MIN = -2 ** 31
# JAERO_MATH_* / JAERO_OSC_* of include/jaero_b200.h
DIV_EXACT, DIV_FAST, ATAN2_FAST, HYPOT_FAST, LOG10_GE1, OSC_INDEX, Q_ROUND, FMOD360, DIV_FAST_CFE = range(9)
SET_FREQ, NEXT_FRAME, NEXT_INDEX, INCREASE_PHASE_DEG, SET_PHASE_DEG, ADVANCE_FRACTION, HAVE_PASSED_POINT, SET_FREQ_SR = range(8)
OSC_OPS = range(8)
AGC_NUMERATOR = 1.414213562           # the AGC gain 1.414213562 / max(mean, 1e-6)


# ---------------------------------------------------------------- ulp helpers
def ordered(x):
    """int64 keys whose order and differences are those of the doubles (+0 and -0 share key 0)"""
    i = np.ascontiguousarray(x, dtype=np.float64).view(np.int64)
    return np.where(i < 0, np.int64(-2 ** 63) - i, i)


def ulp_distance(a, b):
    """number of doubles between a and b (0 for a == b, and for +0 / -0); as float64, exact below 2^53"""
    return np.abs((ordered(a) - ordered(b)).astype(np.float64))


def ulp_error(x, ref):
    """|x - ref| in units of the double ulp at ref (ref long double, nonzero and finite)"""
    ref = np.asarray(ref, dtype=np.longdouble)
    _, e = np.frexp(np.abs(ref))                                  # |ref| in [2^(e-1), 2^e)
    u = np.ldexp(np.longdouble(1), np.maximum(e - 53, -1074))
    return np.abs(np.asarray(x, dtype=np.longdouble) - ref) / u


def same_bits(a, b):
    """element-wise: equal bit patterns, or both NaN"""
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return (a.view(np.int64) == b.view(np.int64)) | (np.isnan(a) & np.isnan(b))


def neighbours(x, k):
    """x and its k nearest doubles on each side, flattened"""
    x = np.asarray(x, dtype=np.float64)
    out, up, dn = [x], x.copy(), x.copy()
    for _ in range(k):
        up = np.nextafter(up, np.inf); dn = np.nextafter(dn, -np.inf)
        out += [up, dn]
    return np.concatenate([o.ravel() for o in out])


# ---------------------------------------------------------------- x86 conversion rule and what is built on it
def x86_int(d):
    d = np.asarray(d, dtype=np.float64)
    ok = (d > -2147483649.0) & (d < 2147483648.0)
    return np.where(ok, np.trunc(np.where(ok, d, 0.0)), INT_MIN).astype(np.int64)


def qround_x86(d):
    """Qt5's qRound, d >= 0 ? int(d + 0.5) : int(d - double(int(d - 1)) + 0.5) + int(d - 1), with x86 conversions and a
    wrapping 32-bit addition"""
    d = np.asarray(d, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        k = x86_int(d - 1.0)
        neg = x86_int((d - k.astype(np.float64)) + 0.5) + k
        neg = (neg + 2 ** 31) % 2 ** 32 - 2 ** 31
        return np.where(d >= 0.0, x86_int(d + 0.5), neg)


def wt_index(ptr):
    """WaveTable::WTCISValue's table index (DSP.cpp:81-83)"""
    t = x86_int(ptr)
    return np.where(t >= WTSIZE, 0, np.where(t < 0, WTSIZE - 1, t))


# ---------------------------------------------------------------- libm and long-double references
def libm(f, *args):
    return np.array([f(*v) for v in zip(*[np.asarray(a, dtype=np.float64).tolist() for a in args])], dtype=np.float64)


def atan2_glibc(y, x):
    return libm(math.atan2, y, x)


def atan2_ld(y, x):
    return np.arctan2(np.asarray(y, dtype=np.longdouble), np.asarray(x, dtype=np.longdouble))


def hypot_glibc(x, y):
    return libm(math.hypot, x, y)


def hypot_ld(x, y):
    return np.hypot(np.asarray(x, dtype=np.longdouble), np.asarray(y, dtype=np.longdouble))


def log10_glibc(x):
    return libm(math.log10, x)


def log10_ld(x):
    return np.log10(np.asarray(x, dtype=np.longdouble))


# ---------------------------------------------------------------- operand generators
def _log_uniform(rng, n, lo, hi):
    return np.exp(rng.uniform(math.log(lo), math.log(hi), n))


def production_divisors():
    """every divisor the demodulators hand div_exact: the moving-average lengths that jaero_batch_create and the burst create
    functions derive (capi.cu) for each mode at the sample rates they accept, Fs itself (osc_set_freq), 360 and WTSIZE"""
    out = {360, WTSIZE}
    qr = lambda d: int(math.floor(d + 0.5))
    for Fs in (12000, 24000, 32000, 48000, 64000, 96000, 128000, 144000, 192000):
        out.add(Fs)
        for fb in (8400, 10500):                                   # continuous OQPSK
            out |= {int(round(4 * Fs)), 2 * 48000, 800, 401, 400}
        for fb in (600, 1200):                                     # continuous MSK
            sps = int(Fs / fb)
            out |= {int(round(Fs)), int(2.0 * Fs), sps, sps // 2 + 1, 600}
        for kind, fb in ((0, 600), (0, 1200), (1, 10500)):         # burst MSK / burst OQPSK
            sps = int(Fs / fb)
            SPS = 2.0 * Fs / fb if kind == 1 else float(sps)
            if SPS < 1:
                continue
            n = {0: 126.0 if fb >= 1200 else 150.0, 1: 128.0}[kind]
            out |= {int(round(Fs)), qr(n * SPS), int(SPS * n), int(SPS * n / 2.0)}
            out |= {int(0.15 * Fs), int(round((SPS * 128.0 / Fs) * Fs)), 75} if kind == 0 else \
                   {int(SPS * 256.0), int(round((SPS * 64.0 / Fs) * Fs)), 128}
    return np.array(sorted(d for d in out if d >= 1), dtype=np.float64)


def odd_part(d):
    d = int(d)
    while d % 2 == 0:
        d //= 2
    return d


def near_midpoint_numerators(rng, d, n):
    """n numerators x whose exact quotient x / d (d an integer with an odd part o > 1) lies 1 / (2o) of an ulp from the midpoint
    between two doubles: the closest any double numerator comes for that divisor. x = N 2^E with N = rho 2^-(t - j) mod o
    (d = 2^j o, t = ceil(log2 d)), so that N 2^t / d = integer + rho / o with rho = (o -+ 1) / 2. Normal quotients, random sign."""
    di = int(d)
    o = odd_part(di); j = (di // o).bit_length() - 1
    assert o > 1
    t = (di - 1).bit_length()                                          # ceil(log2 d)
    hi = di << (53 - t)                                                # N < hi keeps N 2^t / d below 2^53
    inv = pow(pow(2, t - j, o), -1, o)
    out = np.empty(n)
    for i in range(n):
        rho = (o - 1) // 2 + int(rng.integers(0, 2))
        base = rho * inv % o
        k0 = (2 ** 52 - base + o - 1) // o
        k1 = (hi - 1 - base) // o
        N = base + o * int(rng.integers(k0, k1 + 1))
        E = int(rng.integers(-1074 + t, 971))
        out[i] = math.ldexp(float(N), E) * (1 if rng.integers(0, 2) else -1)
    return out


def midpoint_distance(x, d):
    """exact distance of x / d from the nearest midpoint between two doubles, in ulps of the quotient (Fraction)"""
    q = Fraction(float(x)) / Fraction(float(d))
    qa = abs(q)
    e = math.frexp(float(qa))[1]
    if qa >= Fraction(2) ** (e - 1) * 2:
        e += 1
    while qa < Fraction(2) ** (e - 1):
        e -= 1
    u = Fraction(2) ** max(e - 53, -1074)
    frac = (qa / u) % 1
    return abs(frac - Fraction(1, 2))


def div_exact_cases(seed=1, per_divisor=64, dense_numerators=8):
    """(x, d): near-midpoint numerators +-3 ulp for every production divisor; random numerators over all exponents, 0, -0,
    subnormals and values near DBL_MAX; every integer divisor 1 .. 2^17 on a smaller numerator set"""
    rng = np.random.default_rng(seed)
    xs, ds = [], []
    for d in production_divisors():
        if odd_part(d) > 1:
            x = neighbours(near_midpoint_numerators(rng, d, per_divisor), 3)
            xs.append(x); ds.append(np.full(len(x), d))
        x = np.concatenate([rng.uniform(-1, 1, 256) * np.exp2(rng.integers(-1070, 1023, 256)).astype(np.float64),
                            [0.0, -0.0, 5e-324, -5e-324, 2.2250738585072014e-308, 1.7976931348623157e308, -1.7976931348623157e308],
                            np.nextafter(1.7976931348623157e308, 0) - rng.integers(0, 1 << 40, 8) * 2.0 ** 971,
                            rng.integers(1, 1 << 52, 16) * 5e-324])
        xs.append(x); ds.append(np.full(len(x), d))
    all_d = np.arange(1, 2 ** 17 + 1, dtype=np.float64)
    for k in range(dense_numerators):
        x = rng.uniform(-1, 1, len(all_d)) * np.exp2(rng.integers(-1000, 1000, len(all_d))).astype(np.float64)
        xs.append(x); ds.append(all_d)
    odd = all_d[[odd_part(d) > 1 for d in all_d]]
    x = np.array([near_midpoint_numerators(rng, d, 1)[0] for d in odd])
    xs.append(neighbours(x, 1)); ds.append(np.tile(odd, 3))
    return np.concatenate(xs), np.concatenate(ds)


def div_fast_cases(seed=2, n=1 << 21):
    """(a, b, domain): domain 0 the AGC call (1.414213562 over b in [1e-6, 1e6], log-uniform, plus b next to the divisors that put
    the quotient on a midpoint), 1 the log10 call (|a| <= b, b in [2, 3)), 2 the atan2 call (|a| <= b, b in (1e-290, 1e300],
    |a| >= 2^-968, quotient normal), 3 outside those domains (reported, not asserted)"""
    rng = np.random.default_rng(seed)
    b0 = _log_uniform(rng, n, 1e-6, 1e6)
    q = AGC_NUMERATOR / _log_uniform(rng, n // 8, 1e-6, 1e6)
    mid = q + np.spacing(q) / 2
    b0 = np.concatenate([b0, neighbours(AGC_NUMERATOR / mid, 3), [1e-6, 1.0, 2.0, 1e6]])
    b1 = rng.uniform(2.0, 3.0, n)
    a1 = b1 * rng.uniform(-1, 1, n) * np.exp2(-rng.integers(0, 60, n))
    b2 = _log_uniform(rng, n, 1e-290, 1e300)
    a2 = b2 * rng.uniform(-1, 1, n) * np.exp2(-rng.integers(0, 900, n).astype(np.float64))
    # the quotient's remainder must stay normal for the correction step to be exact: numerators below 2^-968 are reported only
    # (atan2_fast's smallest numerators, differences of arguments next to its 1e-290 gate, can be that small; its own test covers them)
    keep = np.abs(a2 / b2) >= 2.2250738585072014e-308
    a2, b2 = a2[keep], b2[keep]
    tiny = np.abs(a2) < 2.0 ** -968
    b3 = np.concatenate([_log_uniform(rng, 4096, 1e-308, 1e-290), _log_uniform(rng, 4096, 1e300, 1.7e308), [0.0, -1.0, np.inf]])
    a3 = rng.uniform(-1, 1, len(b3)) * _log_uniform(rng, len(b3), 1e-300, 1e300)
    a = np.concatenate([np.full(len(b0), AGC_NUMERATOR), a1, a2, a3])
    b = np.concatenate([b0, b1, b2, b3])
    dom = np.concatenate([np.zeros(len(b0)), np.ones(len(b1)), np.where(tiny, 3, 2), np.full(len(b3), 3)]).astype(np.int8)
    return a, b, dom


def atan2_cases(seed=3, n=1 << 21):
    """(y, x): every sign combination of random magnitudes; min/max ratios at 0.4375, 0.6875 and 1 +- 4 ulp; |y| = |x|; the
    1e-290 and 1e300 gates +- 1 ulp; extreme ratios; +-0, +-inf and NaN against finite and special partners"""
    rng = np.random.default_rng(seed)
    sgn = lambda m: np.where(rng.integers(0, 2, m) == 1, 1.0, -1.0)
    mx = _log_uniform(rng, n, 1e-280, 1e290)
    mn = mx * rng.uniform(0, 1, n)
    cases = [(mn, mx)]
    for r in (0.4375, 0.6875, 1.0):
        m = _log_uniform(rng, n // 16, 1e-200, 1e200)
        for k in range(-4, 5):
            v = r * m
            for _ in range(abs(k)):
                v = np.nextafter(v, np.inf if k > 0 else -np.inf)
            cases.append((np.minimum(v, m), np.maximum(v, m)))
    m = _log_uniform(rng, n // 8, 1e-289, 1e299)
    cases.append((m * _log_uniform(rng, len(m), 1e-300, 1e-12), m))            # extreme ratios (small quotient may underflow)
    cases.append((_log_uniform(rng, n // 8, 0.01, 10.0), _log_uniform(rng, n // 8, 0.01, 10.0)))   # the timing-error phasor
    gates = neighbours(np.array([1e-290, 1e300]), 1)
    g = np.repeat(gates, 64)
    other = _log_uniform(rng, len(g), 1e-289, 1e299)
    cases += [(g, other), (other, g)]
    ys = np.concatenate([np.concatenate([c[0], c[1]]) for c in cases])
    xs = np.concatenate([np.concatenate([c[1], c[0]]) for c in cases])          # both orders: swap and no swap
    ys *= sgn(len(ys)); xs *= sgn(len(xs))
    sp = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1.0, -1.0, 1e-300, -1e-300, 1e305, -1e305, 5e-324])
    sy, sx = np.meshgrid(sp, sp)
    return np.concatenate([ys, sy.ravel()]), np.concatenate([xs, sx.ravel()])


def hypot_cases(seed=4, n=1 << 21):
    """(x, y, domain): 0 the call site |sig2| (0 .. 1e12, zeros included), 1 log-uniform over [1e-150, 1e150]"""
    rng = np.random.default_rng(seed)
    sgn = lambda m: np.where(rng.integers(0, 2, m) == 1, 1.0, -1.0)
    x0 = np.concatenate([_log_uniform(rng, n, 1e-6, 1e12), [0.0, 0.0, 1.0]]) * sgn(n + 3)
    y0 = np.concatenate([_log_uniform(rng, n, 1e-6, 1e12), [0.0, 1.0, 0.0]]) * sgn(n + 3)
    x1 = _log_uniform(rng, n, 1e-150, 1e150) * sgn(n)
    y1 = x1 * _log_uniform(rng, n, 1e-20, 1e20) * sgn(n)
    keep = (np.abs(y1) >= 1e-150) & (np.abs(y1) <= 1e150)
    x1, y1 = x1[keep], y1[keep]
    return np.concatenate([x0, x1]), np.concatenate([y0, y1]), np.concatenate([np.zeros(len(x0)), np.ones(len(x1))]).astype(np.int8)


def log10_cases(seed=5, n=1 << 21):
    """x >= 1: 1, powers of two, 10^0 .. 10^22 (exact doubles), the sqrt(2) 2^k boundary where the 0x95f64 carry halves the
    significand +- 8 ulp, log-uniform up to DBL_MAX and dense over [1, 4)"""
    rng = np.random.default_rng(seed)
    p2 = np.exp2(np.arange(0, 1024, dtype=np.float64))
    s2 = np.array([math.sqrt(2.0) * 2.0 ** k for k in range(0, 1023)])
    x = np.concatenate([[1.0], p2, powers_of_ten(), neighbours(s2, 8), neighbours(p2[1:], 2),
                        np.exp(rng.uniform(0, math.log(1.7976931348623157e308), n)), rng.uniform(1.0, 4.0, n // 4)])
    return x[x >= 1.0]


def powers_of_ten():
    return np.array([float(10 ** k) for k in range(23)])


def osc_index_cases(seed=6, n=1 << 20):
    """every integer 0 .. 20000 and its neighbouring doubles, -0, tiny negatives, 2^31 - 1 and 2^31 +- ulps, +-1e300, +-inf, NaN,
    random values around the table and random bit patterns over the whole double range"""
    rng = np.random.default_rng(seed)
    ints = np.arange(0, 20001, dtype=np.float64)
    special = np.array([-0.0, -5e-324, -1e-300, -1e-17, -1.0, -19999.0, 2147483647.0, 2147483648.0, -2147483648.0, -2147483649.0,
                        1e300, -1e300, np.inf, -np.inf, np.nan, -np.nan, 4503599627370496.0, 9007199254740992.0])
    return np.concatenate([neighbours(ints, 1), neighbours(special, 3), rng.uniform(-30000, 60000, n),
                           rng.integers(-2 ** 63, 2 ** 63, n, dtype=np.int64).view(np.float64)])


def q_round_cases(seed=7, n=1 << 20):
    """half-integers and their neighbours over the soft-bit range and beyond, 0.49999999999999994, +-2^31 +- ulps, +-inf, NaN,
    random values and random bit patterns"""
    rng = np.random.default_rng(seed)
    halves = np.arange(-2000, 2001, dtype=np.float64) + 0.5
    special = np.array([0.49999999999999994, -0.49999999999999994, 0.5, -0.5, 0.0, -0.0, 2147483647.0, 2147483647.5, 2147483648.0,
                        -2147483648.0, -2147483648.5, -2147483649.0, 4294967296.0, -4294967296.0, 1e300, -1e300, np.inf, -np.inf, np.nan])
    return np.concatenate([neighbours(halves, 2), neighbours(special, 3), rng.uniform(-1000, 1000, n),
                           rng.uniform(-1, 1, n) * 2.0 ** 33, rng.integers(-2 ** 63, 2 ** 63, n, dtype=np.int64).view(np.float64)])


def fmod360_cases(seed=8, n=1 << 20):
    rng = np.random.default_rng(seed)
    edges = np.array([0.0, 360.0, 720.0, 1080.0, 1e300, np.inf, np.nan])
    return np.concatenate([neighbours(np.concatenate([edges, -edges]), 3), rng.uniform(-1000, 1000, n),
                           rng.uniform(-1, 1, n) * np.exp2(rng.integers(-60, 80, n)).astype(np.float64)])


def osc_scripts(seed=9, n_lanes=4096, n_ops=256, samplerate=48000.0):
    """(op, arg) [n_lanes, n_ops] scripts of oscillator operations. Tame lanes (3 in 4) keep frequencies in [-Fs/2, 5 Fs] (negative,
    0, near and above Fs included), so that their pointer stays below a few table lengths and every operation, advance fractions
    below 0 and above 1 included, follows wraps many times. Wild lanes add frequencies whose step is 2^31 +- a few table lengths,
    >= 1e10 Hz, 1e300 Hz and NaN, and phases of +-inf, NaN and 1e300: their pointers leave the range of (int). They never
    advance by a fraction of a wave, whose loops (the reference's and the device's alike) would take ptr / 19999 turns there."""
    rng = np.random.default_rng(seed)
    Fs, shape = samplerate, (n_lanes, n_ops)
    wild = (np.arange(n_lanes) % 4 == 3)[:, None] & np.ones(shape, dtype=bool)
    tame_ops = np.array([SET_FREQ, SET_FREQ_SR, NEXT_FRAME, NEXT_FRAME, NEXT_FRAME, NEXT_FRAME, NEXT_INDEX, INCREASE_PHASE_DEG,
                         SET_PHASE_DEG, ADVANCE_FRACTION, HAVE_PASSED_POINT, HAVE_PASSED_POINT])
    wild_ops = tame_ops[tame_ops != ADVANCE_FRACTION]
    op = np.where(wild, rng.choice(wild_ops, shape), rng.choice(tame_ops, shape)).astype(np.int32)

    def pick(tame, extra):
        """per element one of the columns of tame (or, in wild lanes, of tame + extra)"""
        cand = np.stack([np.broadcast_to(c, shape) for c in tame + extra], axis=-1)
        k = np.where(wild, rng.integers(0, len(tame) + len(extra), shape), rng.integers(0, len(tame), shape))
        return np.take_along_axis(cand, k[..., None], axis=-1)[..., 0]

    u = lambda lo, hi: rng.uniform(lo, hi, shape)
    step31 = np.array([2.0 ** 31 + k * WTSIZE for k in (-3, -1, 0, 1)]) * Fs / WTSIZE
    freq = pick([u(-0.5, 1.5) * Fs, u(0, 5) * Fs, Fs * (1 + rng.integers(-4, 5, shape) * 2.0 ** -52), 0.0, -0.0, -u(0, 1e4),
                 u(0, Fs / 2), Fs / 2],
                [rng.choice(step31, shape), u(1e10, 1e12), 1e20, 1e300, np.nan])
    phases = np.array([0.0, -0.0, 360.0, -360.0, 720.0, -720.0, 359.99999999999994, -359.99999999999994, 1e6, -1e6, 1e15, -1e15])
    phase = pick([u(-10, 10), rng.choice(phases, shape), u(-1000, 1000), u(-1, 1) * 1e-9], [np.inf, -np.inf, np.nan, 1e300, -1e300])
    frac = pick([u(-3, 3), u(-1, 1) * 1e-3, -1.0, 1.0, 0.0, -1e-17, 1 - 2 ** -53, u(-1.5, -1)], [])
    ees = np.array([0.4, 0.65, 0.025, 0.015, 0.05, 0.0125, 0.0, 1.0, -0.25, 1.25, 0.75, 0.25])
    ee = pick([rng.choice(ees, shape), u(-0.5, 1.5)], [])
    arg = np.zeros(shape)
    arg = np.where((op == SET_FREQ) | (op == SET_FREQ_SR), freq, arg)
    arg = np.where((op == INCREASE_PHASE_DEG) | (op == SET_PHASE_DEG), phase, arg)
    arg = np.where(op == ADVANCE_FRACTION, frac, arg)
    arg = np.where(op == HAVE_PASSED_POINT, ee, arg)
    return op, arg
