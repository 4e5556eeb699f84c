// Device primitives shared by the OQPSK and MSK segment kernels. Each one restates, in the
// reference's own operation order and in double precision, a class of JAERO/DSP.h / DSP.cpp.
// These kernels are compiled with -fmad=false so that a*b+c is rounded exactly as the CPU
// reference rounds it; the only arithmetic that can differ in the last ulp is libm
// (hypot / atan2 / tanh / cos / sin / log10).
#pragma once
#include "demod.cuh"
#include "common.cuh"
#include "fft_device.cuh"                  // c_mul

namespace jb {

// x / d, correctly rounded, for a divisor whose reciprocal rcp = RN(1/d) is loop-invariant (Markstein's sequence:
// q = RN(x*rcp), r = x - q*d exactly by FMA, result RN(q + r*rcp)). Same value as the IEEE division the reference
// performs (checked against 3e8 random operands for every divisor used here), in 3 dependent instructions instead of
// the ~25-deep DDIV expansion. The only deviation: a zero result is always +0.
__device__ __forceinline__ double div_exact(double x, double d, double rcp)
{
    const double q = x * rcp;
    const double r = __fma_rn(-q, d, x);
    return __fma_rn(r, rcp, q);
}
// fmod(p, 360.0), exact: identity for |p| < 360, one exact subtraction for 360 <= p < 720 (Sterbenz), libm otherwise
__device__ __forceinline__ double fmod360(double p)
{
    if (fabs(p) < 360.0) return p;
    if (p >= 360.0 && p < 720.0) return p - 360.0;
    return fmod(p, 360.0);
}

// ---- shorter transcendental functions for the feedback loop of the pipelined demodulators. The library versions are exact
// enough but long dependent chains (tools/micro/fastlat.cu measures the cycles per dependent call);
// these keep the same error class (<= 2 ulp, i.e. the same last-bit differences from glibc that the library calls have) with
// about half the chain length. Zero / non-finite arguments go to the library call, so the special cases are the library's.

// a / b for finite a and normal positive b: reciprocal seed + two Newton steps + one correction step (<= 1 ulp, usually exact)
__device__ __forceinline__ double div_fast(double a, double b)
{
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(b));
    double e = __fma_rn(-b, r, 1.0); r = __fma_rn(r, e, r);
    e = __fma_rn(-b, r, 1.0); r = __fma_rn(r, e, r);
    const double q = a * r;
    return __fma_rn(__fma_rn(-q, b, a), r, q);
}
// atan2(y, x) (std::arg of the timing-error phasor, oqpskdemodulator.cpp:480). fdlibm's scheme with ONE division: the argument
// reduction (t-c)/(1+tc) of t = min/max is formed directly from min and max.
__device__ __forceinline__ double atan2_fast(double y, double x)
{
    const double ax = fabs(x), ay = fabs(y);
    if (!(ax > 0.0) || !(ay > 0.0) || !(ax < 1.0e300) || !(ay < 1.0e300) || ax < 1.0e-290 || ay < 1.0e-290) return atan2(y, x);
    const bool swap = ay > ax;
    const double mn = swap ? ax : ay, mx = swap ? ay : ax;
    double num, den, hi, lo;
    if (mn < 0.4375 * mx) { num = mn; den = mx; hi = 0.0; lo = 0.0; }
    else if (mn < 0.6875 * mx) { num = __fma_rn(2.0, mn, -mx); den = __fma_rn(2.0, mx, mn); hi = 4.63647609000806093515e-01; lo = 2.26987774529616870924e-17; }
    else { num = mn - mx; den = mn + mx; hi = 7.85398163397448278999e-01; lo = 3.06161699786838301793e-17; }
    const double t = div_fast(num, den);
    const double z = t * t, w = z * z;
    const double s1 = z * __fma_rn(w, __fma_rn(w, __fma_rn(w, __fma_rn(w, __fma_rn(w, 1.62858201153657823623e-02, 4.97687799461593236017e-02),
                                   6.66107313738753120669e-02), 9.09088713343650656196e-02), 1.42857142725034663711e-01), 3.33333333333329318027e-01);
    const double s2 = w * __fma_rn(w, __fma_rn(w, __fma_rn(w, __fma_rn(w, -3.65315727442169155270e-02, -5.83357013379057348645e-02),
                                   -7.69187620504482999495e-02), -1.11111104054623557880e-01), -1.99999999998764832476e-01);
    double r = hi - ((t * (s1 + s2) - lo) - t);                       // atan(mn/mx) in [0, pi/4]
    if (swap) r = 1.57079632679489655800e+00 - (r - 6.12323399573676603587e-17);
    if (x < 0.0) r = 3.14159265358979311600e+00 - (r - 1.22464679914735317720e-16);
    return y < 0.0 ? -r : r;
}

// |(x, y)| within 2 ulp of hypot (the pipelined OQPSK kernel's |sig2|). A shorter tanh, 1 - 2/(exp(2|x|)+1), made the kernels
// slower (divergent branches), so tanh stays the library's.
__device__ __forceinline__ double hypot_fast(double x, double y) { return sqrt(__fma_rn(x, x, y * y)); }

struct Osc {                       // WaveTable (DSP.h:40-81)
    double ptr, step, freq, last;
};

__device__ __forceinline__ int osc_index(double ptr)                 // DSP.cpp:81-83
{
    // (int)ptr for 0 <= ptr < 2^31 without the FP64 -> int conversion (50 cycles on this part): adding 2^52 leaves the
    // round-to-nearest integer in the low word; one step down where that rounded up gives the truncation, exactly.
    int t;
    if (ptr >= 0.0 && ptr < 2147483647.0) {
        const double m = ptr + 4503599627370496.0;
        t = __double2loint(m);
        if ((m - 4503599627370496.0) > ptr) t -= 1;
    } else t = (int)ptr;
    if (t >= WTSIZE) t = 0;
    if (t < 0) t = WTSIZE - 1;
    return t;
}
__device__ __forceinline__ void osc_set_freq(Osc &o, double f, double samplerate)   // DSP.cpp:151-156
{
    o.freq = f;
    if (o.freq < 0) o.freq = 0;
    o.step = div_exact((o.freq) * ((double)WTSIZE), samplerate, 1.0 / samplerate);
}
__device__ __forceinline__ void osc_next_frame(Osc &o)               // DSP.cpp:70-77
{
    if (o.step < 0) o.step = 0;
    o.last = o.ptr;
    o.ptr += o.step;
    // `while(((int)WTptr)>=WTSIZE)`: for the non-negative finite pointer, (int)x >= N  <=>  x >= (double)N. The step is below N
    // (frequencies below Fs), so the loop body runs at most once: written as a branch around the (then idle) loop, which costs
    // a compare instead of a divergent loop on every sample
    if (o.ptr >= (double)WTSIZE) { o.ptr -= WTSIZE; while (o.ptr >= (double)WTSIZE) o.ptr -= WTSIZE; }
}
// table index the oscillator will have after its next WTnextFrame(), without committing the advance
__device__ __forceinline__ int osc_next_index(const Osc &o)
{
    double s = o.step; if (s < 0) s = 0;
    double q = o.ptr + s;
    if (q >= (double)WTSIZE) { q -= WTSIZE; while (q >= (double)WTSIZE) q -= WTSIZE; }
    return osc_index(q);
}
__device__ __forceinline__ void osc_set_phase_deg(Osc &o, double p)  // DSP.cpp:175-180
{
    p = fmod360(p);
    while (p < 0) p += 360.0;
    o.ptr = div_exact(p, 360.0, 1.0 / 360.0) * ((double)WTSIZE);
}
__device__ __forceinline__ void osc_increase_phase_deg(Osc &o, double p)   // DSP.cpp:169-173
{
    p += div_exact(360.0 * o.ptr, (double)WTSIZE, 1.0 / ((double)WTSIZE));
    osc_set_phase_deg(o, p);
}
__device__ __forceinline__ void osc_advance_fraction_of_wave(Osc &o, double x)   // DSP.h:56
{
    o.ptr += x * WTSIZE;
    if (o.ptr >= WTSIZE) { o.ptr -= WTSIZE; while (o.ptr >= WTSIZE) o.ptr -= WTSIZE; }
    if (o.ptr < 0) { o.ptr += WTSIZE; while (o.ptr < 0) o.ptr += WTSIZE; }
}
// IfHavePassedPoint (DSP.cpp:222-238); frac receives FractionOfSampleItPassesBy
__device__ __forceinline__ bool osc_have_passed_point(const Osc &o, double fraction_of_wave, double &frac)
{
    double t_last = o.last, t = o.ptr, pt = (fraction_of_wave * WTSIZE);
    t_last -= pt;
    t -= pt;
    if (t_last < 0.0) t_last += WTSIZE;
    if (t < 0.0) t += WTSIZE;
    if ((t_last > 3.0 * WTSIZE / 4.0) && (t < 1.0 * WTSIZE / 4.0)) {
        frac = t / o.step;
        return true;
    }
    return false;
}

// IIR biquad, direct form as DSP.cpp:659-705 evaluates it:
//   y = 0; y += x[n-2]*b2; y += x[n-1]*b1; y += x[n]*b0; y -= y[n-2]*a2; y -= y[n-1]*a1; y /= a0 (=1)
struct Biquad {
    double x1, x2, y1, y2;
};
__device__ __forceinline__ double biquad_update(Biquad &q, double sig, double a1, double a2, double b0, double b1, double b2)
{
    double y = 0;
    y += q.x2 * b2;
    y += q.x1 * b1;
    y += sig * b0;
    y -= q.y2 * a2;
    y -= q.y1 * a1;
    q.x2 = q.x1; q.x1 = sig;
    q.y2 = q.y1; q.y1 = y;
    return y;
}

// qRound (Qt5 qglobal.h) as used at oqpskdemodulator.cpp:569 / mskdemodulator.cpp:453
__device__ __forceinline__ int q_round(double d)
{
    return d >= 0.0 ? int(d + 0.5) : int(d - double(int(d - 1)) + 0.5) + int(d - 1);
}

__device__ __forceinline__ void push_soft(const DemodParams &p, int ch, int &count, int &pending, int &overflow, int ibit)
{
    if (ibit > 255) ibit = 255;
    if (ibit < 0) ibit = 0;
    int pos = count + pending;
    if (pos < p.soft_cap) p.soft[(size_t)ch * p.soft_cap + pos] = (int16_t)ibit;
    else overflow = 1;
    pending++;
}


// ---- bulk asynchronous copies (TMA engine, 1-D form) + mbarrier completion, sm_90 PTX
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, int count)
{ asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes)
{ asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity)
{
    asm volatile("{\n\t.reg .pred p;\n\tMBW_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra MBD_%=;\n\tbra MBW_%=;\n\tMBD_%=:\n\t}"
                 ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// the same for a waiter that is far ahead of its producer (it must not burn the issue slots of the warp it shares a sub-partition with)
__device__ __forceinline__ void mbar_wait_relaxed(unsigned long long *bar, unsigned parity)
{
    unsigned done = 0;
    while (true) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
        if (done) break;
        __nanosleep(400);
    }
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, unsigned bytes, unsigned long long *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void *dst_gmem, const void *src_smem, unsigned bytes)
{ asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }   // all but the newest group
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

} // namespace jb
