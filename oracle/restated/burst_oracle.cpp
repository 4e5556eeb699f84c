// TEST INFRASTRUCTURE ONLY (oracle): CPU restatement, never linked into the product.
#include "burst_oracle.h"
#include <algorithm>

namespace jor {

static QVector<std::complex<double>> hilbert_kernel(int N)      // QJHilbertFilter::setSize (DSP.cpp:759-789)
{
    N = (int)pow(2.0, (ceil(log2(N))));
    QVector<std::complex<double>> k;
    for (int i = 0; i < N; i++) {
        if (i == N / 2) { k.push_back(cpx(-1, 0)); continue; }
        if ((i % 2) == 0) { k.push_back(cpx(0, 0)); continue; }
        k.push_back(cpx(0, (2.0 / ((double)N)) / (std::tan(M_PI * (((double)i) / ((double)N) - 0.5)))));
    }
    return k;
}

BurstMskOracle::BurstMskOracle(double fb_, double Fs_, double fc_, double lbw_, double thr_)
{
    // ctor :11-100 then setSettings :150-323 (surviving values only); fb >= 1200 branch and the 600 bps branch
    afc = true; dcd = false;
    Fs = Fs_; lockingbw = lbw_; fb = fb_;
    if (fb > Fs) fb = Fs;
    freq_center = fc_;
    if (freq_center > ((Fs / 2.0) - (lockingbw / 2.0))) freq_center = ((Fs / 2.0) - (lockingbw / 2.0));
    signalthreshold = thr_;
    SamplesPerSymbol = int(Fs / fb);
    mixer_center.SetFreq(freq_center, (int)Fs); mixer2.SetFreq(freq_center, (int)Fs);
    const int sps = (int)SamplesPerSymbol;
    std::vector<double> taps(2 * sps);
    for (int i = 0; i < 2 * sps; i++) taps[i] = sin(M_PI * i / (2.0 * SamplesPerSymbol)) / (2.0 * SamplesPerSymbol);
    mf_re.init(taps); mf_im.init(taps);
    agc.init(1, Fs);
    ebno.init((int)(0.15 * Fs), false, Fs, fb);                    // MSKEbNoMeasure(0.15*Fs) :187
    hfir.SetKernel(hilbert_kernel(2048));                          // hfir.setSize(2048) :189
    mse = 10.0;
    a1.setdelay(SamplesPerSymbol / 2);
    symboltone_averotator = 1; rotator = 1; symboltone_rotator = 0;  // symboltone_rotator is not initialised before the first burst
    cntr = 0; startstop = -1;
    msema.init(75);                                                // ctor :78
    vol_gain = 0; rotator_freq = 0; carrier_rotation_est = 0;
    if (fb >= 1200) {                                              // :205-256
        bt_d1.setdelay(1.0 * SamplesPerSymbol);
        bt_ma1.setLength(qRound(126.0 * SamplesPerSymbol));
        mav1.init((int)(SamplesPerSymbol * 126));
        bt_ma_diff.setdelay(SamplesPerSymbol * 126);
        pdet.setSettings((int)(SamplesPerSymbol * 126.0 / 2.0), 0.1);
        tridentbuffer_sz = qRound((200.0) * SamplesPerSymbol);
        d1.setLength(((int)289 * SamplesPerSymbol) + 20);
        d2.setLength((int)(qRound(72 + 120.0) * SamplesPerSymbol));
        startstopstart = (int)(SamplesPerSymbol * (500));
        endRotation = (int)((120 + 37) * SamplesPerSymbol);
        st_iir_resonator.a[0] = 1; st_iir_resonator.a[1] = -1.993312819378528; st_iir_resonator.a[2] = 0.999476538254407;
        st_iir_resonator.b[0] = 2.617308727964618e-04; st_iir_resonator.b[1] = 0; st_iir_resonator.b[2] = -2.617308727964618e-04;
        ee = 0.025;
        startProcessing = 120;
    } else {                                                       // :257-311
        mav1.init((int)(SamplesPerSymbol * 150));
        bt_ma_diff.setdelay(SamplesPerSymbol * 150);
        bt_d1.setdelay(1.0 * SamplesPerSymbol);
        bt_ma1.setLength(qRound(150.0 * SamplesPerSymbol));
        pdet.setSettings((int)(SamplesPerSymbol * 150.0 / 2.0), 0.2);
        tridentbuffer_sz = qRound((224) * SamplesPerSymbol);
        d1.setLength(((int)397 * SamplesPerSymbol) + 20);
        d2.setLength(qRound((72 + 150.0) * SamplesPerSymbol));
        startstopstart = (int)(SamplesPerSymbol * (500));
        st_iir_resonator.a[0] = 1; st_iir_resonator.a[1] = -1.991228154418550; st_iir_resonator.a[2] = 0.997385427096603;
        st_iir_resonator.b[0] = 0.001307286451699; st_iir_resonator.b[1] = 0; st_iir_resonator.b[2] = -0.001307286451699;
        ee = 0.015;
        startProcessing = 150;
        endRotation = (int)((startProcessing + 56) * SamplesPerSymbol);
    }
    st_iir_resonator.init();
    agc2.init(SamplesPerSymbol * 128.0 / Fs, Fs);
    delayt8.setdelay((SamplesPerSymbol) / 2.0);
    tridentbuffer.assign(tridentbuffer_sz, 0.0); tridentbuffer_ptr = 0;
    st_osc.SetFreq(fb / 2.0, (int)Fs); st_osc_half.SetFreq(fb / 2.0, (int)Fs);
    delayedsmpl.setLength(sps);
    n_sig_true = n_sig_false = 0;
    nsamp = 0;
}

void BurstMskOracle::CenterFreqChangedSlot(double f)
{
    if (f < (0.75 * fb)) f = 0.75 * fb;
    if (f > (Fs / 2.0 - 0.75 * fb)) f = Fs / 2.0 - 0.75 * fb;
    mixer_center.SetFreq(f, (int)Fs);
    if (afc) mixer2.SetFreq(mixer_center.GetFreqHz());
    if ((mixer2.GetFreqHz() - mixer_center.GetFreqHz()) > (lockingbw / 2.0)) mixer2.SetFreq(mixer_center.GetFreqHz() + (lockingbw / 2.0));
    if ((mixer2.GetFreqHz() - mixer_center.GetFreqHz()) < (-lockingbw / 2.0)) mixer2.SetFreq(mixer_center.GetFreqHz() - (lockingbw / 2.0));
}

static void fft_real_kiss(const std::vector<double> &in, std::vector<cpx> &out)   // FFTrWrapper::transform (fftrwrapper.cpp:19-27)
{
    const int n = (int)in.size();
    out.resize(n);
    for (int i = 0; i < n; i++) out[i] = cpx(in[i], 0.0);
    fft_pow2(out.data(), n, false);
    for (int i = n / 2 + 1; i < n; i++) out[i] = 0;
}

void BurstMskOracle::writeData(const int16_t *ptr, long numofsamples)
{
    const cpx imag(0, 1);
    std::vector<cpx> hfirbuff(numofsamples);
    for (long i = 0; i < numofsamples; i++) hfirbuff[i] = cpx(((double)ptr[i]) / 32768.0, 0);      // :380-384
    hfir.update(hfirbuff.data(), (int)numofsamples);                                                // :386
    for (long i = 0; i < numofsamples; i++) {
        cpx cval = hfirbuff[i];
        agc.Update(std::abs(cval));                                                                 // :412
        cval *= agc.AGCVal;
        cpx cval_d = d1.update_dont_touch(cval);                                                    // :416
        double val_to_demod = d2.update_dont_touch(std::real(cval_d));                              // :419
        double fastarm = std::abs(bt_ma1.UpdateSigned(cval * std::conj(bt_d1.update(cval))));       // :422
        fastarm = mav1.UpdateSigned(fastarm);
        fastarm -= bt_ma_diff.update(fastarm);
        if (fastarm < 0) fastarm = 0;
        double bt_sig = fastarm * fastarm;
        if (bt_sig > 500) bt_sig = 500;
        if (pdet.update(bt_sig)) tridentbuffer_ptr = 0;                                             // :430-435
        if (tridentbuffer_ptr < tridentbuffer_sz) {                                                 // :437-442
            tridentbuffer[tridentbuffer_ptr] = std::real(cval_d);
            tridentbuffer_ptr++;
        } else if (tridentbuffer_ptr == tridentbuffer_sz) {                                         // :443-568
            tridentbuffer_ptr++;
            int size_base = 126, size_top = 74;
            if (fb < 1200) { size_base = 150; size_top = 74; }
            const int N = 4096 * 4 * 2;
            std::vector<double> in(N, 0.0);
            std::vector<cpx> out_base, out_top;
            const int nb = qRound(size_base * SamplesPerSymbol), nt = qRound(size_top * SamplesPerSymbol);
            for (int k = 0; k < nb && k < tridentbuffer_sz; k++) in[k] = tridentbuffer[k];
            fft_real_kiss(in, out_base);
            std::fill(in.begin(), in.end(), 0.0);
            for (int k = 0; k < nt && nb + k < tridentbuffer_sz; k++) in[k] = tridentbuffer[nb + k];
            fft_real_kiss(in, out_top);
            double hzperbin = Fs / ((double)N);
            int peakspacingbins = qRound((0.5 * fb) / hzperbin);
            int minvalbin = 0; double minval = 0;
            for (int k = 0; k < N / 2; k++) if (std::abs(out_base[k]) > minval) { minval = std::abs(out_base[k]); minvalbin = k; }
            double maxtop = 0, maxtophigh = 0; int maxtoppos = 0, maxtopposhigh = 0;
            for (int k = 0; k < N / 2; k++) {
                if (k > 50) {
                    if ((k < minvalbin - (peakspacingbins / 2)) && std::abs(out_top[k]) > maxtop) { maxtop = std::abs(out_top[k]); maxtoppos = k; }
                    if ((k > minvalbin + (peakspacingbins / 2)) && std::abs(out_top[k]) > maxtophigh) { maxtophigh = std::abs(out_top[k]); maxtopposhigh = k; }
                }
            }
            int distfrompeak = std::abs(maxtoppos - minvalbin);
            bool accept = minval > 500.0 && std::abs(distfrompeak - peakspacingbins) < std::abs(peakspacingbins / 20) && !(dcd) && !(cntr > 0 && cntr < (500 * SamplesPerSymbol));
            trident_log.push_back(minvalbin); trident_log.push_back(minval); trident_log.push_back(maxtoppos); trident_log.push_back(maxtopposhigh); trident_log.push_back(accept ? 1.0 : 0.0);
            fill_log.push_back((double)(nsamp + i));
            segment_log.insert(segment_log.end(), tridentbuffer.begin(), tridentbuffer.end());
            if (accept) {
                vol_gain = 1.4142 * (500.0 / (minval / 3));
                double carrierphase = std::arg(out_base[minvalbin]) - (M_PI / 4.0);
                mixer2.SetPhaseDeg((180.0 / M_PI) * carrierphase);
                mixer2.SetFreq(((maxtopposhigh + maxtoppos) / 2) * hzperbin);
                CenterFreqChangedSlot(((maxtopposhigh + maxtoppos) / 2) * hzperbin);
                startstop = startstopstart; cntr = 0; n_sig_true++;
                RxDataBits.clear(); RxDataBits.push_back(-1);
                mse = 0; msema.Zero();
                symboltone_averotator = 1; symboltone_rotator = 1; rotator = 1; rotator_freq = 0; carrier_rotation_est = 0;
                st_iir_resonator.init();
                st_osc.SetPhaseDeg(0); st_osc_half.SetPhaseDeg(0);
            }
        }
        if (startstop > 0) {                                                                        // :571-586
            if (cntr >= (startProcessing * SamplesPerSymbol)) startstop--;
            if (cntr < 1000000) cntr++;
            if (mse < signalthreshold) startstop = startstopstart;
        }
        if (startstop == 0) { startstop--; n_sig_false++; cntr = 0; mse = 1; }                      // :588-596
        if (startstop > 0 || mse < signalthreshold) {                                               // :599
            cval = mixer2.WTCISValue() * (val_to_demod) * vol_gain;
            cpx sig2 = cpx(mf_re.FIRUpdateAndProcess(cval.real()), mf_im.FIRUpdateAndProcess(cval.imag()));
            if (cntr > (startProcessing * SamplesPerSymbol) && cntr < endRotation) {                // :606-626
                cpx symboltone_pt = sig2 * symboltone_rotator * imag;
                double er = std::tanh(symboltone_pt.imag()) * (symboltone_pt.real());
                symboltone_rotator = symboltone_rotator * std::exp(imag * er * 0.5);
                symboltone_averotator = symboltone_averotator * 0.999 + 0.001 * symboltone_rotator;
                symboltone_pt = cpx((symboltone_pt.real()), a1.update(symboltone_pt.real()));
                double progress = (double)cntr - (SamplesPerSymbol * (startProcessing));
                double goal = endRotation - (SamplesPerSymbol * startProcessing);
                progress = progress / goal;
                double st_err = std::arg((st_osc_half.WTCISValue()) * std::conj(symboltone_pt));
                st_err *= 0.5 * (1.0 - progress * progress);
                st_osc_half.AdvanceFractionOfWave(-(1.0 / (2.0 * M_PI)) * st_err * 0.05);
                st_osc.SetPhaseDeg(st_osc_half.GetPhaseDeg() + (360.0 * (1.0 - ee)));
            }
            sig2 *= symboltone_averotator;                                                          // :628-630
            rotator = rotator * std::exp(imag * rotator_freq);
            sig2 *= rotator;
            ebno.Update(std::abs(sig2));                                                            // :634
            if (cntr == endRotation + (200 * SamplesPerSymbol)) ebno_log.push_back(ebno.EbNo);      // :637-640
            sig2 *= agc2.Update(std::abs(sig2));                                                    // :643
            double abval = std::abs(sig2);
            if (abval > 2.84) sig2 = (2.84 / abval) * sig2;
            cpx pt_d = delayedsmpl.update_dont_touch(sig2);                                         // :650
            cpx pt_msk = cpx(sig2.real(), pt_d.imag());
            double st_eta = std::abs(pt_msk);
            st_eta = st_iir_resonator.update(st_eta);
            cpx st_m1 = cpx(st_eta, -delayt8.update(st_eta));
            cpx st_out = st_osc.WTCISValue() * st_m1;
            double st_angle_error = std::arg(st_out);
            if (cntr > endRotation) st_osc.AdvanceFractionOfWave(-st_angle_error * 0.002 / 360.0); // :661-665
            if (st_osc.IfHavePassedPoint(ee)) {                                                     // :668
                double ct_xt = tanh(sig2.imag()) * sig2.real();
                double ct_xt_d = tanh(pt_d.real()) * pt_d.imag();
                double ct_ec = ct_xt_d - ct_xt;
                if (ct_ec > M_PI) ct_ec = M_PI;
                if (ct_ec < -M_PI) ct_ec = -M_PI;
                if (ct_ec > M_PI_2) ct_ec = M_PI_2;
                if (ct_ec < -M_PI_2) ct_ec = -M_PI_2;
                if (cntr > (startProcessing * SamplesPerSymbol)) {                                  // :680-687
                    rotator = rotator * std::exp(imag * ct_ec * 0.25);
                    if (cntr > endRotation) rotator_freq = rotator_freq + ct_ec * 0.0001;
                }
                if (cntr > (startProcessing * SamplesPerSymbol)) {                                  // :706-711
                    double tda = (fabs((pt_msk * 0.75).real()) - 1.0);
                    double tdb = (fabs((pt_msk * 0.75).imag()) - 1.0);
                    mse = msema.Update((tda * tda) + (tdb * tdb));
                }
                double imagin = diffdecode.UpdateSoft(pt_msk.imag());                               // :714-739
                int ibit = qRound((imagin) * 127.0 + 128.0);
                if (ibit > 255) ibit = 255;
                if (ibit < 0) ibit = 0;
                RxDataBits.push_back((short)(unsigned char)ibit);
                double real = diffdecode.UpdateSoft(pt_msk.real());
                real = -real;
                ibit = qRound((real) * 127.0 + 128.0);
                if (ibit > 255) ibit = 255;
                if (ibit < 0) ibit = 0;
                RxDataBits.push_back((short)(unsigned char)ibit);
                if (RxDataBits.size() >= 12) { soft_out.insert(soft_out.end(), RxDataBits.begin(), RxDataBits.end()); RxDataBits.clear(); }
            }
            st_osc.WTnextFrame(); st_osc_half.WTnextFrame(); mixer2.WTnextFrame(); mixer_center.WTnextFrame();   // :744-748
        }
    }
    nsamp += numofsamples;
}
} // namespace jor

// =========================================================================== burst OQPSK
namespace jor {

BurstOqpskOracle::BurstOqpskOracle(double fb_, double Fs_, double fc_, double lbw_, double thr_)
{
    // ctor :4-133 then setSettings :202-277 (surviving values)
    sql = false;
    Fs = Fs_; lockingbw = lbw_; fb = fb_; freq_center = fc_;
    if (freq_center > ((Fs / 2.0) - (lockingbw / 2.0))) freq_center = ((Fs / 2.0) - (lockingbw / 2.0));
    signalthreshold = thr_;
    SamplesPerSymbol = 2.0 * Fs / fb;
    mixer2.SetFreq(freq_center, (int)Fs);
    agc.init(1, Fs);
    agc2.init(SamplesPerSymbol * 64.0 / Fs, Fs);
    hfir.SetKernel(hilbert_kernel(2048));
    bt_d1.setdelay(1.0 * SamplesPerSymbol);
    bt_ma1.setLength(qRound(128.0 * SamplesPerSymbol));
    mav1.init((int)(SamplesPerSymbol * 128));
    bt_ma_diff.setdelay(SamplesPerSymbol * 128);
    d1.setLength((int)(SamplesPerSymbol * 128.0 * 2.5 - 190));
    tridentbuffer_sz = qRound((256.0 + 16.0 + 16.0) * SamplesPerSymbol);
    tridentbuffer.assign(tridentbuffer_sz, 0.0); tridentbuffer_ptr = 0;
    d2.setLength(tridentbuffer_sz);
    pdet.setSettings((int)(SamplesPerSymbol * 128.0 / 2.0), 0.2);
    a1.setdelay(SamplesPerSymbol / 2.0);
    ee = 0.4; symboltone_averotator = 1; carrier_rotation_est = 0;
    ebno.init((int)(SamplesPerSymbol * (256.0)), true, Fs, fb);
    rotator = 1;
    startstopstart = (int)(SamplesPerSymbol * (1050));
    insertpreamble = false;
    // ctor-only members
    mse = 100;
    std::vector<double> taps = rrc_design(1, 55, 48000, 10500 / 2.0);                      // ctor :38-46 (Fs, fb ctor values)
    fir_re.init(taps); fir_im.init(taps);
    const double sps0 = 2.0 * 48000 / 10500;
    delays.setdelay(1); delayt41.setdelay(sps0 / 4.0); delayt42.setdelay(sps0 / 4.0); delayt8.setdelay(sps0 / 8.0);
    st_iir_resonator.b[0] = 0.0048847995518126464; st_iir_resonator.b[1] = 0; st_iir_resonator.b[2] = -0.0048847995518126464;   // 75 Hz (:69-75)
    st_iir_resonator.a[0] = 1; st_iir_resonator.a[1] = -0.3882746897971619; st_iir_resonator.a[2] = 0.99023040089637471;
    st_iir_resonator.init();
    st_osc.SetFreq(10500, 48000); st_osc_ref.SetFreq(10500, 48000); st_osc_quarter.SetFreq(10500 / 4.0, 48000);
    msema.init(128);
    pt_d = 0; yui = 0; sig2_last = 0; symboltone_rotator = 1; startstop = -1; vol_gain = 1; cntr = 0;
    rotator_freq = 0;
    n_sig_true = n_sig_false = 0;
    nsamp = 0;
}

void BurstOqpskOracle::writeData(const int16_t *ptr, long numofsamples)
{
    const cpx imag(0, 1);
    double lastmse = mse;                                                                          // :317
    std::vector<cpx> hfirbuff(numofsamples);
    for (long i = 0; i < numofsamples; i++) hfirbuff[i] = cpx(((double)ptr[i]) / 32768.0, 0);    // :337-341
    hfir.update(hfirbuff.data(), (int)numofsamples);                                               // :344
    for (long i = 0; i < numofsamples; i++) {
        cpx cval = hfirbuff[i];
        agc.Update(std::abs(cval));                                                                // :370-371
        cval *= agc.AGCVal;
        cpx cval_d = d1.update_dont_touch(cval);                                                   // :374
        double val_to_demod = (d2.update_dont_touch(std::real(cval_d)));                           // :377
        double fastarm = std::abs(bt_ma1.UpdateSigned(cval * std::conj(bt_d1.update(cval))));      // :380-385
        fastarm = mav1.UpdateSigned(fastarm);
        fastarm -= bt_ma_diff.update(fastarm);
        if (fastarm < 0) fastarm = 0;
        double bt_sig = fastarm * fastarm;
        if (bt_sig > 500) bt_sig = 500;
        if (pdet.update(bt_sig)) tridentbuffer_ptr = 0;                                            // :388-391
        if (tridentbuffer_ptr < tridentbuffer_sz) { tridentbuffer[tridentbuffer_ptr] = std::real(cval_d); tridentbuffer_ptr++; }
        else if (tridentbuffer_ptr == tridentbuffer_sz) {                                          // :398-506
            tridentbuffer_ptr++;
            const int N = 4096 * 4 * 2;
            const int nseg = qRound(128.0 * SamplesPerSymbol);
            std::vector<double> in(N, 0.0);
            std::vector<cpx> out_base, out_top;
            for (int k = 0; k < nseg && k < tridentbuffer_sz; k++) in[k] = tridentbuffer[k];
            fft_real_kiss(in, out_base);
            std::fill(in.begin(), in.end(), 0.0);
            for (int k = 0; k < nseg && nseg + k < tridentbuffer_sz; k++) in[k] = tridentbuffer[nseg + k];
            fft_real_kiss(in, out_top);
            std::vector<double> out_abs_diff(N / 2);
            for (int k = 0; k < N / 2; k++) out_abs_diff[k] = (std::abs(out_top[k]) - std::abs(out_base[k]));
            double hzperbin = Fs / ((double)N);
            double binpeakspacing = (0.25 * fb) / hzperbin;
            int bps = qRound(binpeakspacing);
            int firstbin = bps, lstbin = N / 2 - bps;
            double maxval = out_abs_diff[firstbin - bps] + out_abs_diff[firstbin + bps] - out_abs_diff[firstbin];
            double maxvalbin = firstbin;
            for (int k = firstbin; k < lstbin; k++) {
                double testval = out_abs_diff[k - bps] + out_abs_diff[k + bps] - out_abs_diff[k];
                if (testval > maxval) { maxval = testval; maxvalbin = k; }
            }
            double minval = std::abs(out_base[0]); double minvalbin = 0;
            for (int k = 0; k < N / 2; k++) if ((std::abs(out_base[k])) > minval) { minval = std::abs(out_base[k]); minvalbin = k; }
            bool accept = (maxval > 500.0) && (fabs((((double)(maxvalbin - minvalbin))) * hzperbin) < 20.0);
            trident_log.push_back(minvalbin); trident_log.push_back(minval); trident_log.push_back(maxvalbin); trident_log.push_back(maxval); trident_log.push_back(accept ? 1.0 : 0.0);
            fill_log.push_back((double)(nsamp + i));
            segment_log.insert(segment_log.end(), tridentbuffer.begin(), tridentbuffer.end());
            if (accept) {
                double carrierphase = std::arg(out_base[(int)minvalbin]) - (M_PI / 4.0);
                mixer2.SetFreq(hzperbin * minvalbin);
                mixer2.SetPhaseDeg((180.0 / M_PI) * carrierphase);
                vol_gain = 1.4142 * 500.0 / minval;
                st_osc.SetFreq(st_osc_ref.GetFreqHz());
                st_osc.SetPhaseDeg(0); st_osc_ref.SetPhaseDeg(0);
                st_iir_resonator.init();
                startstop = startstopstart; cntr = 0; rotator = 1; insertpreamble = true; rotator_freq = 0;
                symboltone_averotator = 1; carrier_rotation_est = 0;
                n_sig_true++;
                mse = 0; msema.Zero();
            }
        }
        cpx cval_dd = mixer2.WTCISValue() * (vol_gain * val_to_demod);                             // :509
        cpx sig2 = cpx(fir_re.FIRUpdateAndProcess(cval_dd.real()), fir_im.FIRUpdateAndProcess(cval_dd.imag()));
        if (startstop > 0) {                                                                       // :515-524
            startstop--;
            if (cntr < 1000000) cntr++;
            if (mse < 0.75) startstop = startstopstart;
        }
        if (startstop == 0) { startstop--; n_sig_false++; }                                        // :525-529
        if ((cntr > ((256 - 10) * SamplesPerSymbol)) && insertpreamble) { RxDataBits.push_back(-1); insertpreamble = false; }   // :531-535
        if ((cntr > SamplesPerSymbol * (128 + 10)) && (cntr < ((256 - 10) * SamplesPerSymbol))) {  // :538-558
            double progress = (((double)cntr) - (SamplesPerSymbol * (128 + 10))) / (((256 - 10) * SamplesPerSymbol) - (SamplesPerSymbol * (128 + 10)));
            cpx symboltone_pt = sig2 * symboltone_rotator * imag;
            double er = std::tanh(symboltone_pt.imag()) * (symboltone_pt.real());
            symboltone_rotator = symboltone_rotator * std::exp(imag * er * 0.01);
            symboltone_averotator = symboltone_averotator * 0.95 + 0.05 * symboltone_rotator;
            symboltone_pt = cpx((symboltone_pt.real()), a1.update(symboltone_pt.real()));
            carrier_rotation_est = std::arg(symboltone_averotator);
            double st_err = std::arg((st_osc_quarter.WTCISValue()) * std::conj(symboltone_pt));
            st_err *= 1.5 * (1.0 - progress * progress);
            st_osc_quarter.AdvanceFractionOfWave(-(1.0 / (2.0 * M_PI)) * st_err * 0.1);
            st_osc.SetPhaseDeg((st_osc_quarter.GetPhaseDeg()) * 4.0 + (360.0 * ee));
        }
        sig2 *= symboltone_averotator;                                                             // :562-565
        rotator = rotator * std::exp(imag * rotator_freq);
        sig2 *= rotator;
        double sig2abs = std::abs(sig2);
        ebno.Update(sig2abs);                                                                      // :570
        if (fabs(cntr - ((128.0 + 128.0 + 128.0) * SamplesPerSymbol)) < 0.5) ebno_log.push_back(ebno.EbNo);   // :573
        sig2 *= agc2.Update(sig2abs);                                                              // :576
        double abval = std::abs(sig2);
        if (abval > 2.84) sig2 = (2.84 / abval) * sig2;
        double st_diff = delays.update(abval * abval) - (abval * abval);                           // :583-591
        double st_d1out = delayt41.update(st_diff);
        double st_d2out = delayt42.update(st_d1out);
        double st_eta = (st_d2out - st_diff) * st_d1out;
        st_iir_resonator.update(st_eta);
        if (cntr > SamplesPerSymbol * (128 + 128)) st_eta = st_iir_resonator.y;
        cpx st_m1 = cpx(st_eta, -delayt8.update(st_eta));
        cpx st_out = st_osc.WTCISValue() * st_m1;
        double st_angle_error = std::arg(st_out);
        if (cntr > SamplesPerSymbol * (128 + 64)) {                                                // :597-601
            st_osc.IncreseFreqHz(-st_angle_error * 0.00000001);
            st_osc.AdvanceFractionOfWave(-st_angle_error * 0.01 / 360.0);
        }
        if (st_osc.GetFreqHz() < (st_osc_ref.GetFreqHz() - 0.1)) st_osc.SetFreq((st_osc_ref.GetFreqHz() - 0.1));
        if (st_osc.GetFreqHz() > (st_osc_ref.GetFreqHz() + 0.1)) st_osc.SetFreq((st_osc_ref.GetFreqHz() + 0.1));
        if (st_osc.IfHavePassedPoint(ee)) {                                                        // :606
            double pt_last = st_osc.FractionOfSampleItPassesBy, pt_this = 1.0 - pt_last;
            cpx pt = pt_this * sig2 + pt_last * sig2_last;
            double twospeed = -4.0 * ((std::fmod((st_osc_quarter.GetPhaseDeg()) * 2.0 + (360.0 * ee * 0.5), 360.0) / 360.0) - (0.34046 + 0.4111 * ee));
            bool even = true;
            if (twospeed < 0) even = false;
            yui++; yui %= 2;
            if (cntr < ((128 + 128) * SamplesPerSymbol)) {
                if ((even && yui == 1) || (!even && yui == 0)) { yui++; yui %= 2; }
            }
            if (!yui) pt_d = pt;
            else {
                cpx pt_qpsk = cpx(pt.real(), pt_d.imag());
                double ct_xt = tanh(pt.imag()) * pt.real();
                double ct_xt_d = tanh(pt_d.real()) * pt_d.imag();
                double ct_ec = ct_xt_d - ct_xt;
                if (ct_ec > M_PI) ct_ec = M_PI;
                if (ct_ec < -M_PI) ct_ec = -M_PI;
                if (ct_ec > M_PI_2) ct_ec = M_PI_2;
                if (ct_ec < -M_PI_2) ct_ec = -M_PI_2;
                if (cntr > ((128 + 10) * SamplesPerSymbol)) {                                      // :641-645
                    rotator = rotator * std::exp(imag * ct_ec * 0.1);
                    if (cntr > ((128 + 10) * SamplesPerSymbol)) rotator_freq = rotator_freq + ct_ec * 0.0001;
                }
                if (cntr > ((128 + 10) * SamplesPerSymbol)) {                                      // :684-689
                    double tda = (fabs(pt_qpsk.real()) - 1.0), tdb = (fabs(pt_qpsk.imag()) - 1.0);
                    mse = msema.Update((tda * tda) + (tdb * tdb));
                }
                if (startstop > 0) {                                                               // :692-722
                    int ibit = qRound(0.75 * pt_qpsk.imag() * 127.0 + 128.0);
                    if (ibit > 255) ibit = 255;
                    if (ibit < 0) ibit = 0;
                    RxDataBits.push_back((short)(unsigned char)ibit);
                    ibit = qRound(0.75 * pt_qpsk.real() * 127.0 + 128.0);
                    if (ibit > 255) ibit = 255;
                    if (ibit < 0) ibit = 0;
                    RxDataBits.push_back((short)(unsigned char)ibit);
                    if (RxDataBits.size() >= 32) {
                        if (!sql || mse < signalthreshold || lastmse < signalthreshold) soft_out.insert(soft_out.end(), RxDataBits.begin(), RxDataBits.end());
                        RxDataBits.clear();
                    }
                }
            }
        }
        sig2_last = sig2;                                                                          // :727
        mixer2.WTnextFrame(); st_osc.WTnextFrame(); st_osc_ref.WTnextFrame(); st_osc_quarter.WTnextFrame();
    }
    nsamp += numofsamples;
}
} // namespace jor
