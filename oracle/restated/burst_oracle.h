// TEST INFRASTRUCTURE ONLY (oracle): CPU restatement of the reference's burst MSK demodulator
// (JAERO/burstmskdemodulator.cpp) and the primitives only it uses. Never linked into the product.
#ifndef JAERO_BURST_ORACLE_H
#define JAERO_BURST_ORACLE_H
#include "dsp_oracle.h"
#include "jfft.h"

namespace jor {

// TMovingAverage<cpx> (DSP.h:145-199)
struct CMovingAverage
{
    std::vector<cpx> buf; cpx sum, Val; int ptr;
    void setLength(int n) { buf.assign(n, cpx(0, 0)); sum = 0; Val = 0; ptr = 0; }
    cpx UpdateSigned(cpx s)
    { sum = sum - buf[ptr]; sum = sum + (s); buf[ptr] = (s); ptr++; ptr %= (int)buf.size(); Val = sum / ((double)buf.size()); return Val; }
};

// PeakDetector (DSP.h:491-576)
struct PeakDetector
{
    DelayThing<double> d1, d2, d3; double lastdy, threshold, maxval; int cntdown, maxcntdown, maxpos, maxposcntdown;
    void setSettings(int length, double th)
    { d1.setLength(length * 2); d2.setLength(length); lastdy = 0; maxcntdown = 2 * length; cntdown = maxcntdown; threshold = th; maxposcntdown = -1; d3.setLength(2 * length); maxval = 0; maxpos = 0; }
    int findmaxpos(DelayThing<double> &d, double &mv)          // DelayThing::findmaxpos (DSP.h:467-481)
    {
        int mp = 0, sz = (int)d.buffer.size();
        mv = d.buffer[d.ptr];
        for (int i = 0; i < sz; i++) { if (d.buffer[d.ptr] > mv) { mv = d.buffer[d.ptr]; mp = i; } d.ptr++; d.ptr %= sz; }
        return mp;
    }
    bool update(double &val)
    {
        double val2 = d3.update_dont_touch(val);
        double dy = val - d1.update_dont_touch(val);
        d2.update(val);
        if ((!cntdown) && (val > threshold) && ((lastdy >= 0 && dy < 0))) {
            cntdown = maxcntdown; maxval = 0; maxpos = findmaxpos(d3, maxval); maxposcntdown = maxpos;
        }
        if (cntdown > 0) cntdown--;
        lastdy = dy;
        val = val2;
        if (!maxposcntdown) { maxposcntdown--; return true; }
        if (maxposcntdown > 0) maxposcntdown--;
        return false;
    }
};

struct BurstMskOracle                                    // burstmskdemodulator.cpp
{
    double Fs, fb, lockingbw, freq_center, signalthreshold, SamplesPerSymbol, ee;
    bool afc, dcd;
    WaveTable mixer_center, mixer2, st_osc, st_osc_half;
    FIR mf_re, mf_im; AGC agc, agc2; EbNoMeasure ebno; MovingAverage msema, mav1;
    JFastFir hfir;
    Delay<cpx> bt_d1; Delay<double> bt_ma_diff, a1, delayt8; CMovingAverage bt_ma1; PeakDetector pdet;
    DelayThing<cpx> d1, delayedsmpl; DelayThing<double> d2;
    std::vector<double> tridentbuffer; int tridentbuffer_ptr, tridentbuffer_sz;
    IIR st_iir_resonator; DiffDecode diffdecode;
    double mse, vol_gain, rotator_freq, carrier_rotation_est;
    cpx symboltone_averotator, symboltone_rotator, rotator;
    int cntr, startstop, startstopstart, endRotation, startProcessing;
    std::vector<short> RxDataBits;
    // observables
    std::vector<short> soft_out; std::vector<double> ebno_log; long n_sig_true, n_sig_false;
    std::vector<double> trident_log;                   // per trident test: minvalbin, minval, maxtoppos, maxtopposhigh, accepted
    std::vector<double> fill_log;                      // per trident test: stream index of the input sample that completed the fill
    std::vector<double> segment_log;                   // per trident test: the tridentbuffer_sz samples of the completed fill
    long nsamp;                                        // input samples consumed so far
    BurstMskOracle(double fb, double Fs, double freq_center, double lockingbw, double signalthreshold);
    void writeData(const int16_t *pcm, long n);        // :371-754
    void CenterFreqChangedSlot(double f);              // :326-343
};
} // namespace jor

namespace jor {
struct BurstOqpskOracle                                  // burstoqpskdemodulator.cpp
{
    double Fs, fb, lockingbw, freq_center, signalthreshold, SamplesPerSymbol, ee;
    bool sql;
    WaveTable mixer2, st_osc, st_osc_ref, st_osc_quarter;
    FIR fir_re, fir_im; AGC agc, agc2; EbNoMeasure ebno; MovingAverage msema, mav1;
    JFastFir hfir;
    Delay<cpx> bt_d1; Delay<double> bt_ma_diff, a1, delays, delayt41, delayt42, delayt8; CMovingAverage bt_ma1; PeakDetector pdet;
    DelayThing<cpx> d1; DelayThing<double> d2;
    std::vector<double> tridentbuffer; int tridentbuffer_ptr, tridentbuffer_sz;
    IIR st_iir_resonator;
    double mse, vol_gain, rotator_freq, carrier_rotation_est;
    cpx symboltone_averotator, symboltone_rotator, rotator, pt_d, sig2_last;
    int cntr, startstop, startstopstart, yui; bool insertpreamble;
    std::vector<short> RxDataBits;
    std::vector<short> soft_out; std::vector<double> ebno_log; long n_sig_true, n_sig_false;
    std::vector<double> trident_log;                   // per trident test: minvalbin, minval, maxvalbin, maxval, accepted
    std::vector<double> fill_log;                      // per trident test: stream index of the input sample that completed the fill
    std::vector<double> segment_log;                   // per trident test: the tridentbuffer_sz samples of the completed fill
    long nsamp;                                        // input samples consumed so far
    BurstOqpskOracle(double fb, double Fs, double freq_center, double lockingbw, double signalthreshold);
    void writeData(const int16_t *pcm, long n);        // writeDataSlot :315-737 (mono)
};
} // namespace jor
#endif
