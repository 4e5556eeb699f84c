// Stages of the continuous demodulator kernels (oqpsk_demod.cu, oqpsk_pipe.cu, msk_pipe.cu). Each restates one piece of
// JAERO/oqpskdemodulator.cpp, mskdemodulator.cpp or DSP.h / DSP.cpp, in the reference's operation order (see
// demod_device.cuh for the rounding rules).
//
// The symbol-rate tails divide a moving sum by its length as `x / len` in the single-warp OQPSK kernel and by div_exact in
// the pipelined ones; the `Mean` policy below carries that choice, so each kernel keeps its form. The OQPSK EbNo read-out
// divides with `/` in both OQPSK kernels.
#pragma once
#include "demod_device.cuh"

namespace jb {

static const int OQ_EBNO_TAIL = 256;      // samples before the end of a launch over which the EbNo read-out is evaluated
static const int OQ_T = 32;               // tile length (samples) of the staged HBM streams; one 256 B ring row per lane
static const int OQ_SM_RING = OQ_T * 32 * 8;   // one ring tile [T][32] doubles
static const int RING_NBUF = 3;           // ring-tile buffers of the pipelined kernels: a tile is reloaded into the buffer stored a
                                          // whole tile earlier, so the writer never waits for a bulk store to drain (with 2
                                          // buffers it stalled ~12 000 cycles at every 32-sample tile boundary: 19 % of the launch)
static const int OQ_NT1 = 56;             // OQPSK: 55 taps + 1 (FIR ring, DSP.cpp:277)
static const int OQ_FIRROWS = 2 * OQ_NT1; // every entry is stored twice so any 55-entry window is contiguous
static const int OQ_SM_FIR = 2 * OQ_FIRROWS * 32 * 8;   // FIR windows re/im [OQ_FIRROWS][32] (bytes)

// per-channel state: D[idx][ch], I[idx][ch] (demod.cuh); `p`, `cpad` and `ch` are the caller's
#define LD(idx) p.D[(size_t)(idx) * cpad + ch]
#define LI(idx) p.I[(size_t)(idx) * cpad + ch]

// ---- mean of a moving sum: sum / len
struct MeanDiv {                          // the IEEE quotient
    int len;
    __device__ __forceinline__ MeanDiv(int n) : len(n) {}
    __device__ __forceinline__ double operator()(double x) const { return x / ((double)len); }
};
struct MeanDivExact {                     // the same quotient in three dependent instructions (div_exact)
    int len;
    double rcp;
    __device__ __forceinline__ MeanDivExact(int n) : len(n), rcp(1.0 / ((double)n)) {}
    __device__ __forceinline__ double operator()(double x) const { return div_exact(x, (double)len, rcp); }
};

// ---- per-channel state access
// WaveTable (DSP.h:64,75-79): the four fields follow `ptr_idx` (D_*_PTR) in the order PTR, STEP, FREQ, LAST
__device__ __forceinline__ Osc load_osc(const DemodParams &p, int ptr_idx, int ch)
{ const size_t cpad = p.cpad; return Osc{LD(ptr_idx), LD(ptr_idx + 1), LD(ptr_idx + 2), LD(ptr_idx + 3)}; }
__device__ __forceinline__ void store_osc(const DemodParams &p, int ptr_idx, int ch, const Osc &o)
{ const size_t cpad = p.cpad; LD(ptr_idx) = o.ptr; LD(ptr_idx + 1) = o.step; LD(ptr_idx + 2) = o.freq; LD(ptr_idx + 3) = o.last; }
// IIR history (x[n-1], x[n-2], y[n-1], y[n-2]) from `x1_idx` (D_RES_X1 / D_LF_X1) on
__device__ __forceinline__ Biquad load_biquad(const DemodParams &p, int x1_idx, int ch)
{ const size_t cpad = p.cpad; return Biquad{LD(x1_idx), LD(x1_idx + 1), LD(x1_idx + 2), LD(x1_idx + 3)}; }
__device__ __forceinline__ void store_biquad(const DemodParams &p, int x1_idx, int ch, const Biquad &q)
{ const size_t cpad = p.cpad; LD(x1_idx) = q.x1; LD(x1_idx + 1) = q.x2; LD(x1_idx + 2) = q.y1; LD(x1_idx + 3) = q.y2; }

// FIR delay line (DSP.cpp:277, nt1 = taps + 1 entries) in shared memory as [row][32 lanes].
// OQPSK keeps every entry twice (rows k and k + nt1) so that any 55-entry window is contiguous.
__device__ __forceinline__ void fir_window_load2(const DemodParams &p, double *s_re, double *s_im, int nt1, int ch, int lane)
{
    for (int k = 0; k < nt1; k++) {
        const double vr = p.fir_re[(size_t)k * p.cpad + ch], vi = p.fir_im[(size_t)k * p.cpad + ch];
        s_re[k * 32 + lane] = vr; s_re[(k + nt1) * 32 + lane] = vr;
        s_im[k * 32 + lane] = vi; s_im[(k + nt1) * 32 + lane] = vi;
    }
}
__device__ __forceinline__ void fir_window_load(const DemodParams &p, double *s_re, double *s_im, int nt1, int ch, int lane)
{
    for (int k = 0; k < nt1; k++) {
        s_re[k * 32 + lane] = p.fir_re[(size_t)k * p.cpad + ch];
        s_im[k * 32 + lane] = p.fir_im[(size_t)k * p.cpad + ch];
    }
}
// rows k0, k0 + step, ... back to HBM (the warps of a pipelined kernel share the rows out)
__device__ __forceinline__ void fir_window_store(const DemodParams &p, const double *s_re, const double *s_im, int nt1, int ch, int lane,
                                                 int k0, int step)
{
    for (int k = k0; k < nt1; k += step) {
        p.fir_re[(size_t)k * p.cpad + ch] = s_re[k * 32 + lane];
        p.fir_im[(size_t)k * p.cpad + ch] = s_im[k * 32 + lane];
    }
}
// a mixed sample enters the delay line (DSP.cpp:292-295) at slot pos, which then advances
__device__ __forceinline__ void fir_push2(double *s_re, double *s_im, int nt1, int lane, int &pos, double re, double im)
{
    s_re[pos * 32 + lane] = re; s_re[(pos + nt1) * 32 + lane] = re;
    s_im[pos * 32 + lane] = im; s_im[(pos + nt1) * 32 + lane] = im;
    pos++; if (pos >= nt1) pos = 0;
}
__device__ __forceinline__ void fir_push(double *s_re, double *s_im, int nt1, int lane, int &pos, double re, double im)
{
    s_re[pos * 32 + lane] = re; s_im[pos * 32 + lane] = im;
    pos++; if (pos >= nt1) pos = 0;
}
// OQPSK: the first 54 terms of the 55-tap FIR over a contiguous window (oldest first), exactly the accumulation order of
// FIR::FIRUpdateAndProcess (DSP.cpp:296-303): outsum += points[i]*buff[tptr], i = 0..53; the caller adds the newest term.
__device__ __forceinline__ void fir54(const DemodParams &p, const double *__restrict__ wre, const double *__restrict__ wim, double &ore, double &oim)
{
    double sre = 0, sim = 0;
#pragma unroll
    for (int k = 0; k < 54; k++) {
        sre += p.taps[k] * wre[k * 32];
        sim += p.taps[k] * wim[k * 32];
    }
    ore = sre; oim = sim;
}

// ---- moving sums
// MovingAverage::Update and the running sums of AGC / EbNo / MSEcalc (DSP.cpp:370-379, 451-463, 493-505, 729-744):
// sum -= oldest; sum += |v|; the slot of the oldest keeps |v|
__device__ __forceinline__ void ma_push(double &sum, double old, double &slot, double v)
{ sum = sum - old; sum = sum + fabs(v); slot = fabs(v); }
__device__ __forceinline__ void ma_push(double &sum, double &slot, double v) { ma_push(sum, slot, slot, v); }
// MovingAverage::UpdateSigned (DSP.cpp:418-426): the same without the fabs
__device__ __forceinline__ void ma_push_signed(double &sum, double old, double &slot, double v)
{ sum = sum - old; sum = sum + (v); slot = (v); }

// ---- EbNo read-outs. The smoothed EbNo <- 0.8 EbNo + 0.2 tebno forgets its past by 0.8^k: evaluating it over the last
// OQ_EBNO_TAIL samples of a launch reproduces the value a per-sample evaluation has at the end of the launch to below 1e-24
// relative, without a log10 and three divisions on every sample. Observable only (DSP.h:250).
// OQPSKEbNoMeasure::Update (DSP.cpp:729-744) over moving sums of length len
__device__ __forceinline__ void oqpsk_ebno_readout(int len, double Fs, double fb, double &ebno, double sum1, double sum2)
{
    const double e2val = sum2 / ((double)len), mean = sum1 / ((double)len);
    const double mean_sq = mean * mean;
    double var = (e2val) - (mean * mean);
    var -= (0.024709 * mean_sq);
    double mvr = (((Fs * mean_sq / (2.0 * fb * var))) * 0.13743);
    if (mvr < 0.000000001) mvr = 0.000000001;
    double tebno = 10.0 * log10(mvr);
    if (isnan(tebno)) tebno = 50;
    if (tebno > 50.0) tebno = 50;
    if (tebno < 0.0) tebno = 0;
    ebno = ebno * 0.8 + 0.2 * tebno;
}
// MSKEbNoMeasure::Update (DSP.cpp:493-505)
template <class Mean>
__device__ __forceinline__ void msk_ebno_readout(const Mean &mean_of, double &ebno, double sum1, double sum2)
{
    const double e2val = mean_of(sum2), mean = mean_of(sum1);
    const double var = (e2val) - (mean * mean);
    const double alpha = sqrt(2.0) / mean;
    double tebno = 10.0 * (log10(2.0) - log10(((var * alpha * alpha) - 0.0085))) - 5.0;
    if (isnan(tebno)) tebno = 50;
    if (tebno > 50.0) tebno = 50;
    ebno = ebno * 0.8 + 0.2 * tebno;
}

// AGC::Update's gain (DSP.cpp:370-379) from the moving sum of |x|
template <class Mean>
__device__ __forceinline__ double agc_gain(const Mean &mean_of, double sum)
{
    const double g = 1.414213562 / fmax(mean_of(sum), 0.000001);
    return fmax(g, 0.000001);
}

// ---- carrier and symbol timing
// ct_ec of a strobe (oqpskdemodulator.cpp:513-517, mskdemodulator.cpp:412-416, burstmskdemodulator.cpp:671-676,
// burstoqpskdemodulator.cpp:632-636): the phase error of point pt against the half-symbol-delayed point pt_d, clamped to
// +-pi. The callers' loop filters and clamps follow.
__device__ __forceinline__ double ct_error(double2 pt, double2 pt_d)
{
    const double ct_xt = tanh(pt.y) * pt.x;
    const double ct_xt_d = tanh(pt_d.x) * pt_d.y;
    double ct_ec = ct_xt_d - ct_xt;
    if (ct_ec > M_PI) ct_ec = M_PI;
    if (ct_ec < -M_PI) ct_ec = -M_PI;
    return ct_ec;
}

// ---- FreqOffsetEstimateSlot
// SignalStatus(false) wired to AeroL::LostSignal (see DemodParams::wire_sigstat): record the soft-bit position, clear DCD
__device__ __forceinline__ void record_lost_signal(const DemodParams &p, int ch)
{
    const size_t cpad = p.cpad;
    const int ln_ = LI(I_LOST_N);
    if (ln_ < LOST_CAP) p.lost_pos[(size_t)ln_ * p.cpad + ch] = LI(I_SOFT_COUNT);
    LI(I_LOST_N) = ln_ + 1;
    LI(I_DCD) = 0;
}
// mixer_center re-centred on mixer2 (oqpskdemodulator.cpp:660-667 / mskdemodulator.cpp:500-507), with
// CoarseFreqEstimate::bigchange (coarsefreqestimate.cpp:84-88): y[]=20 is applied by the estimator kernel on its next run.
// A dead lane leaves the baseband ring row alone.
__device__ __forceinline__ void recentre_mixer_center(const DemodParams &p, int ch, bool live, const Osc &m2, Osc &mc)
{
    const size_t cpad = p.cpad;
    osc_set_freq(mc, m2.freq, p.Fs);
    if (mc.freq < p.lockingbw / 2.0) osc_set_freq(mc, p.lockingbw / 2.0, p.Fs);
    if (mc.freq > (p.Fs / 2.0 - p.lockingbw / 2.0)) osc_set_freq(mc, p.Fs / 2.0 - p.lockingbw / 2.0, p.Fs);
    LI(I_EMPTYING) = 4;
    LI(I_ZERO_BB) = 1;
    double2 *rowz = p.bb + (size_t)ch * p.bb_len;                 // bbcycbuff[j]=0
    if (live) for (int j = 0; j < p.bb_len; j++) rowz[j] = make_double2(0.0, 0.0);
}
// OqpskDemodulator::FreqOffsetEstimateSlot (oqpskdemodulator.cpp:629-677) for the estimate est. Returns whether
// mixer_center was re-centred.
__device__ __forceinline__ bool oqpsk_freq_offset_slot(const DemodParams &p, int ch, bool live, double est, double mse, int &dcd,
                                                       Osc &m2, Osc &mc, int &countdown, int &countdown2, int &sig_true, int &sig_false)
{
    bool recentred = false;
    if ((mse < p.signalthreshold) && (!dcd)) {                        // :642-650
        if (countdown2 > 0) countdown2--;
        else osc_set_freq(m2, mc.freq + est, p.Fs);
    } else countdown2 = 5;
    if ((mse > p.signalthreshold) && (fabs(m2.freq - (mc.freq + est)) > 3.0))    // :653-657
        osc_set_freq(m2, mc.freq + est, p.Fs);
    if ((p.afc) && (mse < p.signalthreshold) && (fabs(m2.freq - mc.freq) > 3.0)) {   // :658-669
        if (countdown > 0) countdown--;
        else { recentre_mixer_center(p, ch, live, m2, mc); recentred = true; }
    } else countdown = 4;
    if (mse > p.signalthreshold) { sig_false++; if (p.wire_sigstat) { record_lost_signal(p, ch); dcd = 0; } } else sig_true++;   // :674-675
    return recentred;
}
// MskDemodulator::FreqOffsetEstimateSlot (mskdemodulator.cpp:490-519), the same way
__device__ __forceinline__ bool msk_freq_offset_slot(const DemodParams &p, int ch, bool live, double est, double mse, int &dcd,
                                                     Osc &m2, Osc &mc, int &countdown, int &sig_true, int &sig_false)
{
    bool recentred = false;
    if ((mse > p.signalthreshold) && (fabs(m2.freq - (mc.freq + est)) > 0.0))      // :494-497
        osc_set_freq(m2, mc.freq + est, p.Fs);
    if ((p.afc) && (dcd) && (fabs(m2.freq - mc.freq) > 2.0)) {                      // :498-509
        if (countdown > 0) countdown--;
        else { recentre_mixer_center(p, ch, live, m2, mc); recentred = true; }
    } else countdown = 4;
    if (mse > p.signalthreshold) { sig_false++; if (p.wire_sigstat) { record_lost_signal(p, ch); dcd = 0; } } else sig_true++;   // :516-517
    return recentred;
}

// ---- symbol-rate tails: everything after the carrier update of a strobe (bias rotate, delay, MSE, soft bits), which feeds
// nothing back inside a launch
// OQPSK (oqpskdemodulator.cpp:535-592). The ring slots a strobe consumes were written >= 400 symbols earlier: they are
// requested a strobe ahead of use (oqpsk_tail_prefetch).
struct OqpskTail {
    double marg_sum, marg_val, pm_sum, ma_sum, mse, lastmse;
    double2 sc0, sc1;                     // the two most recent constellation points
    int marg_pos, dt_pos, mse_pos;
    int soft_count, soft_pending, soft_overflow;
    double marg_old, pm_old, ma_old;
    double2 dt_old;
};
__device__ __forceinline__ OqpskTail load_oqpsk_tail(const DemodParams &p, int ch)
{
    const size_t cpad = p.cpad;
    return OqpskTail{LD(D_MARG_SUM), LD(D_MARG_VAL), LD(D_MSE_PM_SUM), LD(D_MSE_MA_SUM), LD(D_MSE), LD(D_LASTMSE),
                     make_double2(LD(D_SCAT0_RE), LD(D_SCAT0_IM)), make_double2(LD(D_SCAT1_RE), LD(D_SCAT1_IM)),
                     LI(I_MARG_POS), LI(I_DT_POS), LI(I_MSE_POS), LI(I_SOFT_COUNT), LI(I_SOFT_PENDING), LI(I_SOFT_OVERFLOW)};
}
__device__ __forceinline__ void store_oqpsk_tail(const DemodParams &p, int ch, const OqpskTail &t)
{
    const size_t cpad = p.cpad;
    LD(D_MARG_SUM) = t.marg_sum; LD(D_MARG_VAL) = t.marg_val;
    LD(D_MSE_PM_SUM) = t.pm_sum; LD(D_MSE_MA_SUM) = t.ma_sum; LD(D_MSE) = t.mse;
    LD(D_LASTMSE) = t.lastmse;
    LD(D_SCAT0_RE) = t.sc0.x; LD(D_SCAT0_IM) = t.sc0.y; LD(D_SCAT1_RE) = t.sc1.x; LD(D_SCAT1_IM) = t.sc1.y;
    LI(I_MARG_POS) = t.marg_pos; LI(I_DT_POS) = t.dt_pos; LI(I_MSE_POS) = t.mse_pos;
    LI(I_SOFT_COUNT) = t.soft_count; LI(I_SOFT_PENDING) = t.soft_pending; LI(I_SOFT_OVERFLOW) = t.soft_overflow;
}
__device__ __forceinline__ void oqpsk_tail_prefetch(const DemodParams &p, int ch, OqpskTail &t)
{
    t.marg_old = p.marg_ring[(size_t)t.marg_pos * p.cpad + ch];
    t.pm_old = p.mse_pm[(size_t)t.mse_pos * p.cpad + ch];
    t.ma_old = p.mse_ma[(size_t)t.mse_pos * p.cpad + ch];
    { int r = t.dt_pos + 1; if (r >= p.dt_len) r = 0; t.dt_old = p.dt_ring[(size_t)r * p.cpad + ch]; }
}
template <class Mean>
__device__ __forceinline__ void oqpsk_symbol_tail(const DemodParams &p, int ch, bool live, OqpskTail &t, const Mean &marg_mean,
                                                  const Mean &mse_mean, double2 pt_qpsk, double ct_ec)
{
    const double thr = p.signalthreshold;
    {   // marg->UpdateSigned(ct_ec)  MA(800)  (:535, DSP.cpp:418-426)
        ma_push_signed(t.marg_sum, t.marg_old, p.marg_ring[(size_t)t.marg_pos * p.cpad + ch], ct_ec);
        t.marg_pos++; if (t.marg_pos >= p.marg_len) t.marg_pos = 0;
        t.marg_val = marg_mean(t.marg_sum);
    }
    {   // dt.update(pt_qpsk): 400-symbol delay (:536, DSP.h:455-460)
        p.dt_ring[(size_t)t.dt_pos * p.cpad + ch] = pt_qpsk;
        t.dt_pos++; if (t.dt_pos >= p.dt_len) t.dt_pos = 0;
        pt_qpsk = t.dt_old;
    }
    pt_qpsk = c_mul(pt_qpsk, make_double2(cos(t.marg_val), sin(t.marg_val)));   // :537
    t.sc1 = t.sc0; t.sc0 = pt_qpsk;                                              // pointbuff (:546), decimated
    {   // MSEcalc::Update (DSP.cpp:451-463)
        const size_t e = (size_t)t.mse_pos * p.cpad + ch;
        const double ab = hypot(pt_qpsk.x, pt_qpsk.y);
        ma_push(t.pm_sum, t.pm_old, p.mse_pm[e], ab);
        double mu = mse_mean(t.pm_sum);
        if (mu < 0.000001) mu = 0.000001;
        const double r2 = sqrt(2.0);
        const double tre = (r2 * pt_qpsk.x) / mu, tim = (r2 * pt_qpsk.y) / mu;
        const double tda = (fabs(tre) - 1.0), tdb = (fabs(tim) - 1.0);
        const double v = (tda * tda) + (tdb * tdb);
        ma_push(t.ma_sum, t.ma_old, p.mse_ma[e], v);
        t.mse_pos++; if (t.mse_pos >= p.mse_len) t.mse_pos = 0;
        t.mse = mse_mean(t.ma_sum);
    }
    oqpsk_tail_prefetch(p, ch, t);                                    // operands of the next strobe pair
    if (live && t.mse < thr) {                                        // :565
        push_soft(p, ch, t.soft_count, t.soft_pending, t.soft_overflow, q_round(0.75 * pt_qpsk.y * 127.0 + 128.0));
        push_soft(p, ch, t.soft_count, t.soft_pending, t.soft_overflow, q_round(0.75 * pt_qpsk.x * 127.0 + 128.0));
        if (t.soft_pending >= 32) {                                   // :583-592
            if (!p.sql || t.mse < thr || t.lastmse < thr) t.soft_count += t.soft_pending;
            t.soft_pending = 0;
        }
    }
}

// DiffDecode::UpdateSoft (DSP.cpp:531-563)
__device__ __forceinline__ double diff_update_soft(double &last, double soft)
{
    double r;
    if (soft < 0 && last < 0) { r = last; last = soft; }
    else if (soft > 0 && last > 0) { r = -last; last = soft; }
    else { r = fabs(last); last = soft; }
    return r;
}

// MSK (mskdemodulator.cpp:429-476)
struct MskTail {
    double marg_sum, marg_val, ma_sum, mse, diff_last;
    double2 sc0, sc1;                     // the two most recent constellation points
    int marg_pos, dt_pos, mse_pos;
    int soft_count, soft_pending, soft_overflow;
};
__device__ __forceinline__ MskTail load_msk_tail(const DemodParams &p, int ch)
{
    const size_t cpad = p.cpad;
    return MskTail{LD(D_MARG_SUM), LD(D_MARG_VAL), LD(D_MSE_MA_SUM), LD(D_MSE), LD(D_DIFF_LAST),
                   make_double2(LD(D_SCAT0_RE), LD(D_SCAT0_IM)), make_double2(LD(D_SCAT1_RE), LD(D_SCAT1_IM)),
                   LI(I_MARG_POS), LI(I_DT_POS), LI(I_MSE_POS), LI(I_SOFT_COUNT), LI(I_SOFT_PENDING), LI(I_SOFT_OVERFLOW)};
}
__device__ __forceinline__ void store_msk_tail(const DemodParams &p, int ch, const MskTail &t)
{
    const size_t cpad = p.cpad;
    LD(D_MARG_SUM) = t.marg_sum; LD(D_MARG_VAL) = t.marg_val;
    LD(D_MSE_MA_SUM) = t.ma_sum; LD(D_MSE) = t.mse; LD(D_DIFF_LAST) = t.diff_last;
    LD(D_SCAT0_RE) = t.sc0.x; LD(D_SCAT0_IM) = t.sc0.y; LD(D_SCAT1_RE) = t.sc1.x; LD(D_SCAT1_IM) = t.sc1.y;
    LI(I_MARG_POS) = t.marg_pos; LI(I_DT_POS) = t.dt_pos; LI(I_MSE_POS) = t.mse_pos;
    LI(I_SOFT_COUNT) = t.soft_count; LI(I_SOFT_PENDING) = t.soft_pending; LI(I_SOFT_OVERFLOW) = t.soft_overflow;
}
template <class Mean>
__device__ __forceinline__ void msk_symbol_tail(const DemodParams &p, int ch, bool live, MskTail &t, const Mean &marg_mean,
                                                const Mean &mse_mean, double2 pt_msk, double ct_ec)
{
    {   // marg->UpdateSigned(ct_ec/2.0)  MA(SPS)  (:429)
        const size_t e = (size_t)t.marg_pos * p.cpad + ch;
        ma_push_signed(t.marg_sum, p.marg_ring[e], p.marg_ring[e], ct_ec / 2.0);
        t.marg_pos++; t.marg_pos %= p.marg_len;
        t.marg_val = marg_mean(t.marg_sum);
    }
    {   // dt.update(pt_msk) (:430)
        p.dt_ring[(size_t)t.dt_pos * p.cpad + ch] = pt_msk;
        t.dt_pos++; t.dt_pos %= p.dt_len;
        pt_msk = p.dt_ring[(size_t)t.dt_pos * p.cpad + ch];
    }
    pt_msk = c_mul(pt_msk, make_double2(cos(t.marg_val), sin(t.marg_val)));            // :431
    t.sc1 = t.sc0; t.sc0 = make_double2(pt_msk.x * 0.75, pt_msk.y * 0.75);           // pointbuff (:440)
    {   // :446-448
        const double tda = (fabs((pt_msk).x * 0.75) - 1.0), tdb = (fabs((pt_msk).y * 0.75) - 1.0);
        const double v = (tda * tda) + (tdb * tdb);
        ma_push(t.ma_sum, p.mse_ma[(size_t)t.mse_pos * p.cpad + ch], v);
        t.mse_pos++; t.mse_pos %= p.mse_len;
        t.mse = mse_mean(t.ma_sum);
    }
    const double imagin = diff_update_soft(t.diff_last, pt_msk.y);                   // :451
    if (live) push_soft(p, ch, t.soft_count, t.soft_pending, t.soft_overflow, q_round((imagin) * 127.0 + 128.0));
    double real = diff_update_soft(t.diff_last, pt_msk.x);                           // :459
    real = -real;
    if (live) push_soft(p, ch, t.soft_count, t.soft_pending, t.soft_overflow, q_round((real) * 127.0 + 128.0));
    if (t.soft_pending >= 12) { t.soft_count += t.soft_pending; t.soft_pending = 0; }     // :472-476
}

// Delay<double>(SPS/2) of the MSK timing loop (mskdemodulator.cpp delayt8): its delay k = ceil(SPS/2) and the interpolation
// weight exactly as DSP.h:357-374 computes it at ring position 0
inline void msk_half_symbol_delay(int sps, int &k, double &w)
{
    const double fd = (sps) / 2.0;
    const int size = (int)ceil(fd) + 1;
    double dptr = 0.0 - fd;
    while (floor(dptr) < 0) dptr += (double)size;
    w = dptr - floor(dptr);
    k = (int)ceil(fd);
}

// ---- plumbing of the pipelined kernels
// Named barriers: one producer warp arrives, one consumer warp syncs (64 threads).
__device__ __forceinline__ void nb_arrive(int id) { asm volatile("bar.arrive %0, 64;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void nb_sync(int id) { asm volatile("bar.sync %0, 64;" ::"r"(id) : "memory"); }
// Producer side of a hand-off: st.shared, membar.cta, bar.arrive; consumer side bar.sync, ld.shared. (Without the membar the
// OQPSK kernel is 1.2 % faster and every parity test still passes - bar.arrive is not documented to order the producer's
// stores, so it stays.)
__device__ __forceinline__ void handoff(int id) { __threadfence_block(); nb_arrive(id); }

// PCM input: each lane reads its own channel row 8 samples (16 bytes) at a time with plain vector loads, one block ahead
// of use (rows are 16-byte aligned and a multiple of 8 samples long: host-checked). Bulk-copy tiles cost 32 serialised copy
// instructions per 32 samples (one per lane) for 64 bytes each.
struct PcmReader {
    const int4 *row4;
    long long stride;
    bool live;
    int blk;                              // block of pk
    int4 pk, pk_next;                     // 8 consecutive PCM samples of this lane's channel, and the next 8

    __device__ __forceinline__ PcmReader(const int16_t *row, size_t stride_, bool live_, int i0)
        : row4(reinterpret_cast<const int4 *>(row)), stride((long long)stride_), live(live_), blk(i0 >> 3)
    { pk = block(blk); pk_next = block(blk + 1); }
    __device__ __forceinline__ int4 block(int b) const
    { return (live && (long long)b * 8 < stride) ? __ldg(row4 + b) : make_int4(0, 0, 0, 0); }
    // ((double)*ptr)/32768.0 (oqpskdemodulator.cpp:390, mskdemodulator.cpp:322); ii advances by one per call
    __device__ __forceinline__ double dval(int ii)
    {
        if ((ii >> 3) != blk) { blk = ii >> 3; pk = pk_next; pk_next = block(blk + 1); }
        const int k = ii & 7;
        const int w = (k < 2) ? pk.x : (k < 4) ? pk.y : (k < 6) ? pk.z : pk.w;
        int v = (k & 1) ? (w >> 16) : (int)(short)(w & 0xffff);
        if (!live) v = 0;
        return ((double)v) / 32768.0;
    }
};

} // namespace jb
