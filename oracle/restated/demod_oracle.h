// TEST INFRASTRUCTURE ONLY (oracle): CPU restatement of the reference's continuous demodulators
// and coarse frequency estimator. Never linked into the product.
#ifndef JAERO_DEMOD_ORACLE_H
#define JAERO_DEMOD_ORACLE_H
#include "dsp_oracle.h"
#include "jfft.h"      // restated JFastFir (oracle/jfft_restated.cpp) for the 8400 bps pre-filter

namespace jor {

struct DemodSettings                                   // oqpskdemodulator.h:20-39 / mskdemodulator.h:24-45
{
    int coarsefreqest_fft_power; double freq_center, lockingbw, fb, Fs, signalthreshold;
    bool afc, sql, cpuReduce;
};

// CoarseFreqEstimate: coarsefreqestimate.cpp:39-76 (setSettings), :84-88 (bigchange), :90-137 (ProcessBasebandData)
struct CoarseFreqEstimate
{
    int nfft, startbin, stopbin, expectedpeakbin, emptyingcountdown; double Fs, fb, lockingbw, hzperbin, freq_offset_est;
    std::vector<cpx> out, in; std::vector<double> window, y, z;
    void setSettings(int power, double lockingbw, double fb, double Fs);
    void bigchange();
    double ProcessBasebandData(const std::vector<cpx> &data);   // returns the value the reference would emit
};

struct OqpskDemodOracle                                // oqpskdemodulator.cpp
{
    DemodSettings s; bool dcd; double mse, ee, SamplesPerSymbol;
    WaveTable mixer_center, mixer2, st_osc, st_osc_ref;
    FIR fir_re, fir_im; AGC agc; EbNoMeasure ebno; MovingAverage marg; DelayThing<cpx> dt; MSEcalc msecalc;
    Delay<double> delays, delayt41, delayt42, delayt8; IIR st_iir_resonator, ct_iir_loopfilter;
    CoarseFreqEstimate cfe; std::vector<cpx> bbcycbuff, bbtmpbuff; int bbcycbuff_ptr, bbnfft, coarseCounter;
    // function-local statics of the reference, made per-instance (oqpskdemodulator.cpp:487,496,498,641,652)
    bool sig2_last_init; cpx sig2_last, pt_d; int yui, countdown2, countdown;
    std::vector<short> RxDataBits;
    JFastFir fir_pre; WaveTable mixer_fir_pre;         // 8400 bps pre-filter (:112-115,280-283)
    // observables
    std::vector<short> soft_out; std::vector<double> cfe_log, cfe_raw_log; long n_sig_true, n_sig_false; long nsamples;
    // optional direct connections, as JAERO/mainwindow.cpp:198-237,432,508 makes them: processDemodulatedSoftBits(vector) and
    // SignalStatus(bool) are delivered synchronously, inside writeData
    void (*on_emit)(void *ctx, const short *bits, int n) = nullptr; void (*on_sigstat)(void *ctx, bool ok) = nullptr; void *hook_ctx = nullptr;
    explicit OqpskDemodOracle(const DemodSettings &);
    void writeData(const int16_t *pcm, long n);        // :334-627
    void FreqOffsetEstimateSlot(double est);           // :629-677
    void CenterFreqChangedSlot(double freq_center);    // :291-310
    void DCDstatSlot(bool d) { dcd = d; }
    void setAFC(bool v) { s.afc = v; }                 // :149-163
    void setSQL(bool v) { s.sql = v; }
    void setCPUReduce(bool v) { s.cpuReduce = v; }
};

struct MskDemodOracle                                  // mskdemodulator.cpp
{
    DemodSettings s; bool dcd; double mse, ee, correctionfactor; int SamplesPerSymbol;
    WaveTable mixer_center, mixer2, st_osc;
    FIR mf_re, mf_im; AGC agc; EbNoMeasure ebno; MovingAverage marg, msema; DelayThing<cpx> dt, delayedsmpl;
    Delay<double> delayt8; IIR st_iir_resonator; DiffDecode diffdecode;
    CoarseFreqEstimate cfe; std::vector<cpx> bbcycbuff, bbtmpbuff; int bbcycbuff_ptr, bbnfft, coarseCounter;
    int countdown;                                     // static at mskdemodulator.cpp:493
    std::vector<short> RxDataBits;
    std::vector<short> soft_out; std::vector<double> cfe_log, cfe_raw_log; long n_sig_true, n_sig_false; long nsamples;
    void (*on_emit)(void *ctx, const short *bits, int n) = nullptr; void (*on_sigstat)(void *ctx, bool ok) = nullptr; void *hook_ctx = nullptr;
    explicit MskDemodOracle(const DemodSettings &);
    void writeData(const int16_t *pcm, long n);        // :313-488
    void FreqOffsetEstimateSlot(double est);           // :490-519
    void CenterFreqChangedSlot(double freq_center);    // :265-282
    void DCDstatSlot(bool d) { dcd = d; }
    void setAFC(bool v) { s.afc = v; }                 // :105-122
    void setSQL(bool v) { s.sql = v; }
    void setCPUReduce(bool v) { s.cpuReduce = v; }
};
} // namespace jor
#endif
