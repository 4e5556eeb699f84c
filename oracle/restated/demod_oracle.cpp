// TEST INFRASTRUCTURE ONLY (oracle): CPU restatement, never linked into the product.
#include "demod_oracle.h"
#include <algorithm>

namespace jor {

Trig::Trig()
{
    SinWT.resize(WTSIZE); CosWT.resize(WTSIZE);
    for (int i = 0; i < WTSIZE; i++) SinWT[i] = (sin(2 * M_PI * ((double)i) / WTSIZE));              // DSP.cpp:19
    for (int i = 0; i < WTSIZE; i++) CosWT[i] = (sin(M_PI_2 + 2 * M_PI * ((double)i) / WTSIZE));     // DSP.cpp:20
}
const Trig &trig() { static Trig t; return t; }

std::vector<double> rrc_design(double alpha, int firsize, double samplerate, double symbol_freq)
{
    if ((firsize % 2) == 0) firsize += 1;
    std::vector<double> P(firsize);
    double T = (samplerate) / (symbol_freq), fi;
    for (int i = 0; i < firsize; i++) {
        if (i == ((firsize - 1) / 2)) P[i] = (4.0 * alpha + M_PI - M_PI * alpha) / (M_PI * sqrt(T));
        else {
            fi = (((double)i) - ((double)(firsize - 1)) / 2.0);
            if (fabs(1.0 - pow(4.0 * alpha * fi / T, 2)) < 0.0000000001)
                P[i] = (alpha * ((M_PI - 2.0) * cos(M_PI / (4.0 * alpha)) + (M_PI + 2.0) * sin(M_PI / (4.0 * alpha))) / (M_PI * sqrt(2.0 * T)));
            else
                P[i] = (4.0 * alpha / (M_PI * sqrt(T)) * (cos((1.0 + alpha) * M_PI * fi / T) + T / (4.0 * alpha * fi) * sin((1.0 - alpha) * M_PI * fi / T)) / (1.0 - pow(4.0 * alpha * fi / T, 2)));
        }
    }
    return P;
}

void fft_pow2(cpx *x, int n, bool inv)
{
    static int cached_n = 0; static std::vector<cpx> tw; static std::vector<int> rev;
    if (cached_n != n) {
        cached_n = n; tw.resize(n / 2); rev.resize(n);
        for (int k = 0; k < n / 2; k++) { double a = -2.0 * M_PI * (double)k / (double)n; tw[k] = cpx(cos(a), sin(a)); }
        int bits = 0; while ((1 << bits) < n) bits++;
        for (int i = 0; i < n; i++) { int r = 0; for (int b = 0; b < bits; b++) if (i & (1 << b)) r |= 1 << (bits - 1 - b); rev[i] = r; }
    }
    for (int i = 0; i < n; i++) if (rev[i] > i) std::swap(x[i], x[rev[i]]);
    for (int len = 2; len <= n; len <<= 1) {
        int half = len >> 1, step = n / len;
        for (int i = 0; i < n; i += len)
            for (int k = 0; k < half; k++) {
                cpx w = tw[k * step]; if (inv) w = std::conj(w);
                cpx a = x[i + k], b = x[i + k + half] * w;
                x[i + k] = a + b; x[i + k + half] = a - b;
            }
    }
}

// ------------------------------------------------------------------ CoarseFreqEstimate
void CoarseFreqEstimate::setSettings(int power, double lbw, double fb_, double Fs_)
{
    lockingbw = lbw; fb = fb_; Fs = Fs_;
    nfft = (int)pow(2, power);
    hzperbin = Fs / ((double)nfft);
    out.assign(nfft, cpx(0, 0)); in.assign(nfft, cpx(0, 0)); y.assign(nfft, 0.0); z.assign(nfft, 0.0);
    startbin = (int)std::max(round(lockingbw / hzperbin), 1.0);
    stopbin = nfft - startbin;
    expectedpeakbin = (int)round(fb / (2.0 * hzperbin));
    emptyingcountdown = 1;                              // ctor value (coarsefreqestimate.cpp:24); setSettings leaves it
    freq_offset_est = 0;
    window.assign(nfft, 0.0); window[0] = 1;
    for (int i = 1; i <= startbin; i++) {
        double val = cos(M_PI_2 * ((double)i) / ((double)startbin)); val *= val;
        if ((nfft - i) < 0) break;
        if (i >= nfft) break;
        window[nfft - i] = val; window[i] = val;
    }
}
void CoarseFreqEstimate::bigchange() { emptyingcountdown = 4; for (int i = 0; i < nfft; i++) y[i] = 20; }

double CoarseFreqEstimate::ProcessBasebandData(const std::vector<cpx> &data)
{
    out = data; fft_pow2(out.data(), nfft, false);                                    // :93
    if (fb != 8400) for (int i = startbin; i <= stopbin; i++) out[i] = 0;             // :99
    else for (int i = 0; i < nfft; i++) out[i] *= window[i];                          // :100
    in = out; fft_pow2(in.data(), nfft, true);                                        // :102 (JFFT 1/N then wrapper xN = unnormalised)
    for (int i = 0; i < nfft; i++) in[i] = in[i] * in[i];                             // :103
    out = in; fft_pow2(out.data(), nfft, false);                                      // :104
    for (int i = 0; i < nfft / 2; i++) std::swap(out[i + nfft / 2], out[i]);          // :105
    for (int i = 0; i < nfft; i++) y[i] = y[i] * 0.9 + 0.1 * 10 * log10(fmax(std::abs(out[i]), 1));   // :108
    double zmax = 0; int zmaxloc = nfft / 2;
    for (int i = (int)round((-lockingbw / hzperbin) + ((double)(nfft / 2))); i < round((lockingbw / hzperbin) + ((double)(nfft / 2))); i++) {
        if ((i < 0) || (i >= nfft)) continue;
        double val = 0;
        for (int j = -1; j <= 1; j++) {
            if (((i - expectedpeakbin - j) < 0) || ((i + expectedpeakbin + j) >= nfft)) continue;
            val += (y[i - expectedpeakbin - j] + y[i + expectedpeakbin + j]);
        }
        z[i] = val;
        if (z[i] > zmax) { zmax = z[i]; zmaxloc = i; }
    }
    freq_offset_est = -((double)(zmaxloc - nfft / 2)) * hzperbin * 0.5;               // :131
    if (emptyingcountdown <= 0) return freq_offset_est;                               // :134-135
    emptyingcountdown--; return 0;
}

// ------------------------------------------------------------------ OQPSK
OqpskDemodOracle::OqpskDemodOracle(const DemodSettings &st) : s(st)
{
    // ctor :8-117 then setSettings :175-289 (only the surviving values are restated)
    dcd = false; mse = 100;
    if (s.freq_center > ((s.Fs / 2.0) - (s.lockingbw / 2.0))) s.freq_center = ((s.Fs / 2.0) - (s.lockingbw / 2.0));   // :183
    SamplesPerSymbol = 2.0 * s.Fs / s.fb;
    bbnfft = (int)pow(2, s.coarsefreqest_fft_power);
    bbcycbuff.assign(bbnfft, cpx(0, 0)); bbtmpbuff.assign(bbnfft, cpx(0, 0)); bbcycbuff_ptr = 0;
    cfe.setSettings(s.coarsefreqest_fft_power, 2.0 * s.lockingbw / 2.0, s.fb, s.Fs);           // :191
    mixer_center.SetFreq(s.freq_center, (int)s.Fs); mixer2.SetFreq(s.freq_center, (int)s.Fs);
    agc.init(4, s.Fs);                                                                          // :197
    ebno.init((int)(2 * 48000), true, s.Fs, s.fb);      // ctor :42 with the ctor's Fs=48000; setup_update(Fs,fb) :276
    marg.init(800); dt.setLength(400); msecalc.init(400);                                      // :44-45,53
    std::vector<double> taps = (s.fb == 8400) ? rrc_design(0.6, 55, s.Fs, s.fb / 2) : rrc_design(1.0, 55, s.Fs, s.fb / 2);   // :209-211
    fir_re.init(taps); fir_im.init(taps);
    double T = s.Fs / (s.fb / 2);                                                               // :221
    delays.setdelay(1); delayt41.setdelay(T / 4.0); delayt42.setdelay(T / 4.0); delayt8.setdelay(T / 8.0);
    if (s.fb == 8400) {                                                                         // :243-250 (the later assignment wins)
        st_iir_resonator.b[0] = 0.0012845857864470789; st_iir_resonator.b[1] = 0; st_iir_resonator.b[2] = -0.0012845857864470789;
        st_iir_resonator.a[0] = 1; st_iir_resonator.a[1] = -0.90681461999279889; st_iir_resonator.a[2] = 0.99743082842710584;
        ee = 0.65;
    } else {                                                                                    // :256-263
        st_iir_resonator.b[0] = 0.00032714218939589035; st_iir_resonator.b[1] = 0; st_iir_resonator.b[2] = 0.00032714218939589035;
        st_iir_resonator.a[0] = 1; st_iir_resonator.a[1] = -0.39005299948210803; st_iir_resonator.a[2] = 0.99934571562120822;
        ee = 0.4;
    }
    st_iir_resonator.init();
    ct_iir_loopfilter.b[0] = 0.0010275610653672064; ct_iir_loopfilter.b[1] = 0.0020551221307344128; ct_iir_loopfilter.b[2] = 0.0010275610653672064;   // :95-100
    ct_iir_loopfilter.a[0] = 1; ct_iir_loopfilter.a[1] = -1.9207386815577139; ct_iir_loopfilter.a[2] = 0.92509247310306331;
    ct_iir_loopfilter.init();
    st_osc.SetFreq(s.fb, (int)s.Fs); st_osc_ref.SetFreq(s.fb, (int)s.Fs);                       // :270-271
    {   // :280-283 (kernel of the 8400 pre-filter; built for every rate, used only at 8400) and ctor :115
        std::vector<double> pts = (s.fb == 8400) ? rrc_design(0.6, 2048, s.Fs, s.fb / 2) : rrc_design(1.0, 2048, s.Fs, s.fb / 2);
        QVector<double> qp((int)pts.size());
        for (size_t i = 0; i < pts.size(); i++) qp[(int)i] = pts[i];
        fir_pre.SetKernel(qp, 4096);
        mixer_fir_pre.SetFreq(8000, 48000);               // ctor freq_center=8000, Fs=48000; setSettings never touches it
    }
    coarseCounter = 0;
    sig2_last_init = false; sig2_last = 0; pt_d = 0; yui = 0; countdown2 = 5; countdown = 4;
    n_sig_true = n_sig_false = 0; nsamples = 0;
}

void OqpskDemodOracle::writeData(const int16_t *ptr, long len)
{
    if (!len) return;
    double lastmse = mse;                                                                       // :339
    std::vector<cpx> cval_prefiltered;                                                          // :343-381
    if (s.fb == 8400) {
        cval_prefiltered.resize(len);
        double savedphase = mixer_fir_pre.GetPhaseDeg();
        for (long i = 0; i < len; i++) {
            double dval = ((double)(ptr[i])) / 32768.0;
            cval_prefiltered[i] = mixer_fir_pre.WTCISValue() * dval;
            mixer_fir_pre.WTnextFrame();
        }
        fir_pre.update(cval_prefiltered.data(), (int)len);
        mixer_fir_pre.SetPhaseDeg(savedphase);
        for (long i = 0; i < len; i++) {
            cval_prefiltered[i] *= mixer_fir_pre.WTCISValue_conj();
            mixer_fir_pre.WTnextFrame();
        }
    }
    double mixer2_freq_sum = 0;                                                                 // :385
    for (long i = 0; i < len; i++) {
        double dval = ((double)(ptr[i])) / 32768.0;                                             // :390
        if ((coarseCounter >= s.Fs || !s.cpuReduce)) {                                          // :410-429
            bbcycbuff[bbcycbuff_ptr] = mixer_center.WTCISValue() * dval;
            bbcycbuff_ptr++; bbcycbuff_ptr %= bbnfft;
            if (bbcycbuff_ptr % (s.cpuReduce ? bbnfft : bbnfft / 4) == 0) {
                for (int j = 0; j < bbnfft; j++) { bbtmpbuff[j] = bbcycbuff[bbcycbuff_ptr]; bbcycbuff_ptr++; bbcycbuff_ptr %= bbnfft; }
                double est = cfe.ProcessBasebandData(bbtmpbuff);
                cfe_log.push_back(est); cfe_raw_log.push_back(cfe.freq_offset_est);   // emitted (gated) and raw estimate
                FreqOffsetEstimateSlot(est);
                coarseCounter = 0;
            }
        }
        coarseCounter++;
        cpx sig2;
        if (s.fb == 8400) {                                                                     // :436-448
            sig2 = mixer2.WTCISValue() * cval_prefiltered[i];
            mixer2_freq_sum += mixer2.GetFreqHz();
        } else {
            cpx cval = mixer2.WTCISValue() * dval;                                              // :453
            sig2 = cpx(fir_re.FIRUpdateAndProcess(cval.real()), fir_im.FIRUpdateAndProcess(cval.imag()));   // :456
        }
        double dabval = std::sqrt(sig2.real() * sig2.real() + sig2.imag() * sig2.imag());       // :461
        ebno.Update(dabval);                                                                    // :463
        sig2 *= agc.Update(dabval);                                                             // :466
        double abval = std::abs(sig2);                                                          // :469
        if (abval > 2.84) sig2 = (2.84 / abval) * sig2;                                         // :470
        double st_diff = delays.update(abval * abval) - (abval * abval);                        // :473
        double st_d1out = delayt41.update(st_diff);
        double st_d2out = delayt42.update(st_d1out);
        double st_eta = (st_d2out - st_diff) * st_d1out;
        st_eta = st_iir_resonator.update(st_eta);
        cpx st_m1 = cpx(st_eta, -delayt8.update(st_eta));
        cpx st_out = st_osc.WTCISValue() * st_m1;
        double st_angle_error = std::arg(st_out);                                               // :480
        st_osc.IncreseFreqHz(-st_angle_error * 0.00000001);
        st_osc.AdvanceFractionOfWave(-st_angle_error * 0.01 / 360.0);
        if (st_osc.GetFreqHz() < (st_osc_ref.GetFreqHz() - 0.1)) st_osc.SetFreq((st_osc_ref.GetFreqHz() - 0.1));
        if (st_osc.GetFreqHz() > (st_osc_ref.GetFreqHz() + 0.1)) st_osc.SetFreq((st_osc_ref.GetFreqHz() + 0.1));
        if (!sig2_last_init) { sig2_last = sig2; sig2_last_init = true; }                       // :487 static init
        if (st_osc.IfHavePassedPoint(ee)) {                                                     // :488
            double pt_last = st_osc.FractionOfSampleItPassesBy, pt_this = 1.0 - pt_last;
            cpx pt = pt_this * sig2 + pt_last * sig2_last;                                      // :494
            yui++; yui %= 2;
            if (!yui) pt_d = pt;
            else {
                cpx pt_qpsk = cpx(pt.real(), pt_d.imag());                                      // :503
                double ct_xt = tanh(pt.imag()) * pt.real();
                double ct_xt_d = tanh(pt_d.real()) * pt_d.imag();
                double ct_ec = ct_xt_d - ct_xt;
                if (ct_ec > M_PI) ct_ec = M_PI;
                if (ct_ec < -M_PI) ct_ec = -M_PI;
                if (s.fb > 8400) {                                                              // :518-525
                    ct_ec = ct_iir_loopfilter.update(ct_ec);
                    if (ct_ec > M_PI_2) ct_ec = M_PI_2;
                    if (ct_ec < -M_PI_2) ct_ec = -M_PI_2;
                    mixer2.IncresePhaseDeg(1.0 * ct_ec);
                    mixer2.IncreseFreqHz(0.01 * ct_ec);
                } else {                                                                        // :526-532
                    mixer2.IncresePhaseDeg(1.0 * ct_ec);
                    mixer2.IncreseFreqHz(0.5 * 0.01 * ct_iir_loopfilter.update(ct_ec));
                }
                marg.UpdateSigned(ct_ec);                                                       // :535
                dt.update(pt_qpsk);
                pt_qpsk *= cpx(cos(marg.Val), sin(marg.Val));
                mse = msecalc.Update(pt_qpsk);                                                  // :563
                if (mse < s.signalthreshold) {                                                  // :565
                    int ibit = jor::qRound(0.75 * pt_qpsk.imag() * 127.0 + 128.0);
                    if (ibit > 255) ibit = 255;
                    if (ibit < 0) ibit = 0;
                    RxDataBits.push_back((short)(unsigned char)ibit);
                    ibit = jor::qRound(0.75 * pt_qpsk.real() * 127.0 + 128.0);
                    if (ibit > 255) ibit = 255;
                    if (ibit < 0) ibit = 0;
                    RxDataBits.push_back((short)(unsigned char)ibit);
                    if (RxDataBits.size() >= 32) {                                              // :583-592
                        if (!s.sql || mse < s.signalthreshold || lastmse < s.signalthreshold)
                        {   soft_out.insert(soft_out.end(), RxDataBits.begin(), RxDataBits.end());
                            if (on_emit) on_emit(hook_ctx, RxDataBits.data(), (int)RxDataBits.size()); }
                        RxDataBits.clear();
                    }
                }
            }
        }
        sig2_last = sig2;                                                                       // :596
        mixer2.WTnextFrame(); mixer_center.WTnextFrame(); st_osc.WTnextFrame(); st_osc_ref.WTnextFrame();   // :600-603
        nsamples++;
    }
    mixer_fir_pre.SetFreq(mixer2_freq_sum / ((double)len));                                     // :608
}

void OqpskDemodOracle::FreqOffsetEstimateSlot(double est)
{
    if ((mse > s.signalthreshold) || (!dcd)) mixer_fir_pre.SetFreq(mixer_center.GetFreqHz() + est, (int)s.Fs);   // :634-638
    if ((mse < s.signalthreshold) && (!dcd)) {                                                  // :642-650
        if (countdown2 > 0) countdown2--;
        else mixer2.SetFreq(mixer_center.GetFreqHz() + est);
    } else countdown2 = 5;
    if ((mse > s.signalthreshold) && (fabs(mixer2.GetFreqHz() - (mixer_center.GetFreqHz() + est)) > 3.0))   // :653-657
        mixer2.SetFreq(mixer_center.GetFreqHz() + est);
    if ((s.afc) && (mse < s.signalthreshold) && (fabs(mixer2.GetFreqHz() - mixer_center.GetFreqHz()) > 3.0)) {   // :658-669
        if (countdown > 0) countdown--;
        else {
            mixer_center.SetFreq(mixer2.GetFreqHz());
            if (mixer_center.GetFreqHz() < s.lockingbw / 2.0) mixer_center.SetFreq(s.lockingbw / 2.0);
            if (mixer_center.GetFreqHz() > (s.Fs / 2.0 - s.lockingbw / 2.0)) mixer_center.SetFreq(s.Fs / 2.0 - s.lockingbw / 2.0);
            cfe.bigchange();
            for (int j = 0; j < bbnfft; j++) bbcycbuff[j] = 0;
        }
    } else countdown = 4;
    if (mse > s.signalthreshold) n_sig_false++; else n_sig_true++;                              // :674-675
    if (on_sigstat) on_sigstat(hook_ctx, !(mse > s.signalthreshold));
}

void OqpskDemodOracle::CenterFreqChangedSlot(double freq_center)
{
    if (s.fb != 8400) {                                                                         // :293-297
        if (freq_center < (0.5 * s.fb)) freq_center = 0.5 * s.fb;
        if (freq_center > (s.Fs / 2.0 - 0.5 * s.fb)) freq_center = s.Fs / 2.0 - 0.5 * s.fb;
    }
    mixer_center.SetFreq(freq_center, (int)s.Fs);                                               // :298
    if (s.afc) mixer2.SetFreq(mixer_center.GetFreqHz());                                        // :299
    if ((mixer2.GetFreqHz() - mixer_center.GetFreqHz()) > (s.lockingbw / 2.0)) mixer2.SetFreq(mixer_center.GetFreqHz() + (s.lockingbw / 2.0));    // :300-303
    if ((mixer2.GetFreqHz() - mixer_center.GetFreqHz()) < (-s.lockingbw / 2.0)) mixer2.SetFreq(mixer_center.GetFreqHz() - (s.lockingbw / 2.0));   // :304-307
    for (int j = 0; j < bbnfft; j++) bbcycbuff[j] = 0;                                          // :308
}

// ------------------------------------------------------------------ MSK
MskDemodOracle::MskDemodOracle(const DemodSettings &st) : s(st)
{
    dcd = false;
    if (s.freq_center > ((s.Fs / 2.0) - (s.lockingbw / 2.0))) s.freq_center = ((s.Fs / 2.0) - (s.lockingbw / 2.0));   // :145
    SamplesPerSymbol = int(s.Fs / s.fb);                                                        // :149
    bbnfft = (int)pow(2, s.coarsefreqest_fft_power);
    bbcycbuff.assign(bbnfft, cpx(0, 0)); bbtmpbuff.assign(bbnfft, cpx(0, 0)); bbcycbuff_ptr = 0;
    cfe.setSettings(s.coarsefreqest_fft_power, s.lockingbw, s.fb, s.Fs);                        // :154
    mixer_center.SetFreq(s.freq_center, (int)s.Fs); mixer2.SetFreq(s.freq_center, (int)s.Fs);
    st_osc.SetFreq(s.fb / 2, (int)s.Fs);                                                        // :159
    std::vector<double> taps(2 * SamplesPerSymbol);                                             // :164-170
    for (int i = 0; i < 2 * SamplesPerSymbol; i++) taps[i] = sin(M_PI * i / (2.0 * SamplesPerSymbol)) / (2.0 * SamplesPerSymbol);
    mf_re.init(taps); mf_im.init(taps);
    agc.init(1, s.Fs);                                                                          // :173
    ebno.init((int)(2.0 * s.Fs), false, s.Fs, s.fb);                                            // :176
    mse = 10.0;                                                                                 // :180
    msema.init(600);                                                                            // ctor :64 (not rebuilt by setSettings)
    if (s.fb >= 1200) {                                                                         // :189-250
        correctionfactor = 0.6;
        if (s.Fs == 48000) { st_iir_resonator.a[0] = 1; st_iir_resonator.a[1] = -1.993312819378528; st_iir_resonator.a[2] = 0.999476538254407;
            st_iir_resonator.b[0] = 2.617308727964618e-04; st_iir_resonator.b[1] = 0; st_iir_resonator.b[2] = -2.617308727964618e-04; ee = 0.025; }
        else { st_iir_resonator.a[0] = 1; st_iir_resonator.a[1] = -1.974342917561558; st_iir_resonator.a[2] = 0.998953350377616;
            st_iir_resonator.b[0] = 5.233248111921052e-04; st_iir_resonator.b[1] = 0; st_iir_resonator.b[2] = -5.233248111921052e-04; ee = 0.05; }
    } else {
        correctionfactor = 1.0;
        if (s.Fs == 48000) { st_iir_resonator.a[0] = 1; st_iir_resonator.a[1] = -1.998196509168551; st_iir_resonator.a[2] = 0.999738234875681;
            st_iir_resonator.b[0] = 1.308825621597620e-04; st_iir_resonator.b[1] = 0; st_iir_resonator.b[2] = -1.308825621597620e-04; ee = 0.025; }
        else { st_iir_resonator.a[0] = 1; st_iir_resonator.a[1] = -1.974342917561558; st_iir_resonator.a[2] = 0.998953350377616;
            st_iir_resonator.b[0] = 5.233248111921052e-04; st_iir_resonator.b[1] = 0; st_iir_resonator.b[2] = -5.233248111921052e-04; ee = 0.0125; }
    }
    st_iir_resonator.init();
    marg.init(SamplesPerSymbol); dt.setLength(SamplesPerSymbol / 2);                            // :254-256
    delayedsmpl.setLength(SamplesPerSymbol); delayt8.setdelay((SamplesPerSymbol) / 2.0);        // :258-260
    coarseCounter = 0; countdown = 4;
    n_sig_true = n_sig_false = 0; nsamples = 0;
}

void MskDemodOracle::writeData(const int16_t *ptr, long len)
{
    for (long i = 0; i < len; i++) {
        double dval = ((double)(ptr[i])) / 32768.0;                                             // :322
        if ((coarseCounter >= s.Fs || !s.cpuReduce)) {                                          // :350-367
            bbcycbuff[bbcycbuff_ptr] = mixer_center.WTCISValue() * dval;
            bbcycbuff_ptr++; bbcycbuff_ptr %= bbnfft;
            if (bbcycbuff_ptr % (s.cpuReduce ? bbnfft : bbnfft / 4) == 0) {
                for (int j = 0; j < bbnfft; j++) { bbtmpbuff[j] = bbcycbuff[bbcycbuff_ptr]; bbcycbuff_ptr++; bbcycbuff_ptr %= bbnfft; }
                double est = cfe.ProcessBasebandData(bbtmpbuff);
                cfe_log.push_back(est); cfe_raw_log.push_back(cfe.freq_offset_est);   // emitted (gated) and raw estimate
                FreqOffsetEstimateSlot(est);
                coarseCounter = 0;
            }
        }
        coarseCounter++;
        cpx cval = mixer2.WTCISValue() * (dval);                                                // :369
        cpx sig2 = cpx(mf_re.FIRUpdateAndProcess(cval.real()), mf_im.FIRUpdateAndProcess(cval.imag()));
        double dabval = std::sqrt(sig2.real() * sig2.real() + sig2.imag() * sig2.imag());       // :372
        ebno.Update(dabval);
        sig2 *= agc.Update(dabval);                                                             // :378
        double abval = std::sqrt(sig2.real() * sig2.real() + sig2.imag() * sig2.imag());        // :381
        if (abval > 2.84) sig2 = (2.84 / abval) * sig2;
        cpx pt_d = delayedsmpl.update_dont_touch(sig2);                                         // :384
        cpx pt_msk = cpx(sig2.real(), pt_d.imag());
        double st_eta = st_iir_resonator.update(std::abs(pt_msk));                              // :387
        cpx st_m1 = cpx(st_eta, -delayt8.update(st_eta));
        cpx st_out = st_osc.WTCISValue() * st_m1;
        double st_angle_error = std::arg(st_out);                                               // :392
        double weighting = fabs(tanh(st_angle_error));
        if (!dcd) st_osc.AdvanceFractionOfWave(-(1.0 - weighting) * st_angle_error * (0.05 / 360.0));     // :397-405
        else st_osc.AdvanceFractionOfWave(-(1.0 - weighting) * st_angle_error * (0.003 / 360.0));
        if (st_osc.IfHavePassedPoint(ee)) {                                                     // :408
            double ct_xt = tanh(sig2.imag()) * sig2.real();
            double ct_xt_d = tanh(pt_d.real()) * pt_d.imag();
            double ct_ec = ct_xt_d - ct_xt;
            if (ct_ec > M_PI) ct_ec = M_PI;
            if (ct_ec < -M_PI) ct_ec = -M_PI;
            if (ct_ec > M_PI_2) ct_ec = M_PI_2;
            if (ct_ec < -M_PI_2) ct_ec = -M_PI_2;
            double carrier_aggression = 12.0 * correctionfactor;                                // :422-426
            if (dcd) carrier_aggression = 8.0 * correctionfactor;
            mixer2.IncresePhaseDeg(carrier_aggression * 1.0 * ct_ec);
            mixer2.IncreseFreqHz(carrier_aggression * 0.01 * ct_ec);
            marg.UpdateSigned(ct_ec / 2.0);                                                     // :429-431
            dt.update(pt_msk);
            pt_msk *= cpx(cos(marg.Val), sin(marg.Val));
            double tda = (fabs((pt_msk).real() * 0.75) - 1.0);                                  // :446-448
            double tdb = (fabs((pt_msk).imag() * 0.75) - 1.0);
            mse = msema.Update((tda * tda) + (tdb * tdb));
            double imagin = diffdecode.UpdateSoft(pt_msk.imag());                               // :451-469
            int ibit = jor::qRound((imagin) * 127.0 + 128.0);
            if (ibit > 255) ibit = 255;
            if (ibit < 0) ibit = 0;
            RxDataBits.push_back((short)(unsigned char)ibit);
            double real = diffdecode.UpdateSoft(pt_msk.real());
            real = -real;
            ibit = jor::qRound((real) * 127.0 + 128.0);
            if (ibit > 255) ibit = 255;
            if (ibit < 0) ibit = 0;
            RxDataBits.push_back((short)(unsigned char)ibit);
            if (RxDataBits.size() >= 12) {                                                      // :472-476
                soft_out.insert(soft_out.end(), RxDataBits.begin(), RxDataBits.end());
                if (on_emit) on_emit(hook_ctx, RxDataBits.data(), (int)RxDataBits.size());
                RxDataBits.clear();
            }
        }
        mixer2.WTnextFrame(); mixer_center.WTnextFrame(); st_osc.WTnextFrame();                 // :480-483
        nsamples++;
    }
}

void MskDemodOracle::FreqOffsetEstimateSlot(double est)
{
    if ((mse > s.signalthreshold) && (fabs(mixer2.GetFreqHz() - (mixer_center.GetFreqHz() + est)) > 0.0))   // :494-497
        mixer2.SetFreq(mixer_center.GetFreqHz() + est);
    if ((s.afc) && (dcd) && (fabs(mixer2.GetFreqHz() - mixer_center.GetFreqHz()) > 2.0)) {       // :498-509
        if (countdown > 0) countdown--;
        else {
            mixer_center.SetFreq(mixer2.GetFreqHz());
            if (mixer_center.GetFreqHz() < s.lockingbw / 2.0) mixer_center.SetFreq(s.lockingbw / 2.0);
            if (mixer_center.GetFreqHz() > (s.Fs / 2.0 - s.lockingbw / 2.0)) mixer_center.SetFreq(s.Fs / 2.0 - s.lockingbw / 2.0);
            cfe.bigchange();
            for (int j = 0; j < bbnfft; j++) bbcycbuff[j] = 0;
        }
    } else countdown = 4;
    if (mse > s.signalthreshold) n_sig_false++; else n_sig_true++;                              // :516-517
    if (on_sigstat) on_sigstat(hook_ctx, !(mse > s.signalthreshold));
}

void MskDemodOracle::CenterFreqChangedSlot(double freq_center)
{
    if (freq_center < (0.75 * s.fb)) freq_center = 0.75 * s.fb;                                 // :267-268
    if (freq_center > (s.Fs / 2.0 - 0.75 * s.fb)) freq_center = s.Fs / 2.0 - 0.75 * s.fb;
    mixer_center.SetFreq(freq_center, (int)s.Fs);                                               // :269
    if (s.afc) mixer2.SetFreq(mixer_center.GetFreqHz());                                        // :270
    if ((mixer2.GetFreqHz() - mixer_center.GetFreqHz()) > (s.lockingbw / 2.0)) mixer2.SetFreq(mixer_center.GetFreqHz() + (s.lockingbw / 2.0));    // :271-274
    if ((mixer2.GetFreqHz() - mixer_center.GetFreqHz()) < (-s.lockingbw / 2.0)) mixer2.SetFreq(mixer_center.GetFreqHz() - (s.lockingbw / 2.0));   // :275-278
    for (int j = 0; j < bbnfft; j++) bbcycbuff[j] = 0;                                          // :279
}
} // namespace jor
