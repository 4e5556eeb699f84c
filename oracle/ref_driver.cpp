// TEST INFRASTRUCTURE ONLY (oracle/_ref).
// extern "C" harness around the reference's own hot-path sources, which are
// compiled VERBATIM from /root/reference/JAERO by oracle/Makefile (never copied
// into this repo) against oracle/shim (Qt stand-ins, restated JFFT/libcorrect).
// This file supplies what moc would have generated (signal bodies) and routes the
// two signal->slot connections the hot path relies on:
//   demod::BBOverlapedBuffer -> CoarseFreqEstimate::ProcessBasebandData   (oqpskdemodulator.cpp:57)
//   CoarseFreqEstimate::FreqOffsetEstimate -> demod::FreqOffsetEstimateSlot (oqpskdemodulator.cpp:58)
// Function-local statics in the reference (oqpskdemodulator.cpp:487-498,641,652)
// are shared between instances: use ONE OQPSK instance per process.
#include <map>
#include <vector>
#include <complex>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <new>
#include "qt_shim.h"
#define private public
#define protected public
#include "DSP.h"
#include "coarsefreqestimate.h"
#include "mskdemodulator.h"
#include "oqpskdemodulator.h"
#include "burstmskdemodulator.h"
#include "burstoqpskdemodulator.h"
#include "fftwrapper.h"
#include "fftrwrapper.h"
#include "jconvolutionalcodec.h"
#undef private
#undef protected

// the reference leaves several members uninitialised (cpuReduce, EbNo ...,
// SURVEY.md App. A.8): zero-fill every heap object so runs are deterministic.
void *operator new(std::size_t n) { void *p = calloc(1, n ? n : 1); if (!p) throw std::bad_alloc(); return p; }
void *operator new[](std::size_t n) { void *p = calloc(1, n ? n : 1); if (!p) throw std::bad_alloc(); return p; }
void operator delete(void *p) noexcept { free(p); }
void operator delete[](void *p) noexcept { free(p); }
void operator delete(void *p, std::size_t) noexcept { free(p); }
void operator delete[](void *p, std::size_t) noexcept { free(p); }

struct RefHandle
{
    int kind;                       // 0 = OQPSK, 1 = MSK, 2 = burst MSK, 3 = burst OQPSK
    OqpskDemodulator *oq;
    MskDemodulator *msk;
    BurstMskDemodulator *bmsk;
    BurstOqpskDemodulator *boq;
    std::vector<double> ebno_log;   // EbNoMeasurmentSignal values (burst modes emit one per burst)
    std::vector<short> soft;        // concatenated processDemodulatedSoftBits payloads
    std::vector<int> emit_sizes;    // size of each emit
    std::vector<double> cfe_log;    // every FreqOffsetEstimate value, in order
    long n_signal_true, n_signal_false;
    double last_mse_signal, last_ebno_signal;
};
static std::map<const void *, RefHandle *> g_handles;
static RefHandle *find(const void *p) { auto it = g_handles.find(p); return it == g_handles.end() ? 0 : it->second; }

// ---------------- signal bodies (moc substitute) ----------------
#define NOP_SIGNALS(C) \
    void C::ScatterPoints(const QVector<cpx_type> &) {} \
    void C::OrgOverlapedBuffer(const QVector<double> &) {} \
    void C::PeakVolume(double) {} \
    void C::SampleRateChanged(double) {} \
    void C::BitRateChanged(double, bool) {} \
    void C::Plottables(double, double, double) {} \
    void C::WarningTextSignal(const QString &) {}
NOP_SIGNALS(OqpskDemodulator)
NOP_SIGNALS(MskDemodulator)
NOP_SIGNALS(BurstMskDemodulator)
NOP_SIGNALS(BurstOqpskDemodulator)
void BurstMskDemodulator::SymbolPhase(double) {}
void BurstMskDemodulator::RxData(QByteArray &) {}
void BurstMskDemodulator::BBOverlapedBuffer(const QVector<cpx_type> &) {}
void BurstOqpskDemodulator::BBOverlapedBuffer(const QVector<cpx_type> &) {}
void BurstOqpskDemodulator::writeDataSignal(const char *, qint64) {}
void MskDemodulator::SymbolPhase(double) {}
void MskDemodulator::RxData(const QByteArray &) {}

void OqpskDemodulator::BBOverlapedBuffer(const QVector<cpx_type> &b) { coarsefreqestimate->ProcessBasebandData(b); }
void MskDemodulator::BBOverlapedBuffer(const QVector<cpx_type> &b) { coarsefreqestimate->ProcessBasebandData(b); }
void CoarseFreqEstimate::FreqOffsetEstimate(double f)
{
    RefHandle *h = find(parent());
    if (!h) return;                     // stand-alone estimator (jref_cfe_*): result read from the member
    h->cfe_log.push_back(f);
    if (h->kind == 0) h->oq->FreqOffsetEstimateSlot(f); else h->msk->FreqOffsetEstimateSlot(f);
}
#define OBS_SIGNALS(C) \
    void C::MSESignal(double m) { RefHandle *h = find(this); if (h) h->last_mse_signal = m; } \
    void C::EbNoMeasurmentSignal(double e) { RefHandle *h = find(this); if (h) { h->last_ebno_signal = e; h->ebno_log.push_back(e); } } \
    void C::SignalStatus(bool s) { RefHandle *h = find(this); if (h) { if (s) h->n_signal_true++; else h->n_signal_false++; } } \
    void C::processDemodulatedSoftBits(const QVector<short> &v) \
    { RefHandle *h = find(this); if (!h) return; h->emit_sizes.push_back(v.size()); for (int i = 0; i < v.size(); i++) h->soft.push_back(v[i]); }
OBS_SIGNALS(OqpskDemodulator)
OBS_SIGNALS(MskDemodulator)
OBS_SIGNALS(BurstMskDemodulator)
OBS_SIGNALS(BurstOqpskDemodulator)

extern "C" {

// ---------------- continuous OQPSK (oqpskdemodulator.cpp) ----------------
void *jref_oqpsk_new(double fb, double Fs, double freq_center, double lockingbw, int fft_power,
                     double signalthreshold, int afc, int sql, int cpureduce)
{
    RefHandle *h = new RefHandle();
    h->kind = 0;
    h->oq = new OqpskDemodulator(0);
    g_handles[h->oq] = h;
    h->oq->setCPUReduce(cpureduce != 0);
    OqpskDemodulator::Settings s;
    s.fb = fb; s.Fs = Fs; s.freq_center = freq_center; s.lockingbw = lockingbw;
    s.coarsefreqest_fft_power = fft_power; s.signalthreshold = signalthreshold;
    h->oq->setSettings(s);
    h->oq->setAFC(afc != 0);
    h->oq->setSQL(sql != 0);
    h->oq->start();
    return h;
}
void *jref_msk_new(double fb, double Fs, double freq_center, double lockingbw, int fft_power,
                   double signalthreshold, int afc, int sql, int cpureduce)
{
    RefHandle *h = new RefHandle();
    h->kind = 1;
    h->msk = new MskDemodulator(0);
    g_handles[h->msk] = h;
    h->msk->setCPUReduce(cpureduce != 0);
    MskDemodulator::Settings s;
    s.fb = fb; s.Fs = Fs; s.freq_center = freq_center; s.lockingbw = lockingbw;
    s.coarsefreqest_fft_power = fft_power; s.signalthreshold = signalthreshold;
    h->msk->setSettings(s);
    h->msk->setAFC(afc != 0);
    h->msk->setSQL(sql != 0);
    h->msk->start();
    return h;
}
// burst demodulators (burstmskdemodulator.cpp / burstoqpskdemodulator.cpp), settings as mainwindow.cpp:876-899
void *jref_burst_msk_new(double fb, double Fs, double freq_center, double lockingbw, double signalthreshold)
{
    RefHandle *h = new RefHandle();
    h->kind = 2;
    h->bmsk = new BurstMskDemodulator(0);
    g_handles[h->bmsk] = h;
    BurstMskDemodulator::Settings s;
    s.fb = fb; s.Fs = Fs; s.freq_center = freq_center; s.lockingbw = lockingbw; s.signalthreshold = signalthreshold;
    h->bmsk->setSettings(s);
    h->bmsk->start();
    return h;
}
void *jref_burst_oqpsk_new(double fb, double Fs, double freq_center, double lockingbw, double signalthreshold)
{
    RefHandle *h = new RefHandle();
    h->kind = 3;
    h->boq = new BurstOqpskDemodulator(0);
    g_handles[h->boq] = h;
    BurstOqpskDemodulator::Settings s;
    s.fb = fb; s.Fs = Fs; s.freq_center = freq_center; s.lockingbw = lockingbw; s.signalthreshold = signalthreshold;
    h->boq->setSettings(s);
    h->boq->start();
    return h;
}
void jref_write(void *hv, const int16_t *pcm, long n)
{
    RefHandle *h = (RefHandle *)hv;
    if (h->kind == 0) h->oq->writeData((const char *)pcm, (qint64)n * 2);
    else if (h->kind == 1) h->msk->writeData((const char *)pcm, (qint64)n * 2);
    else if (h->kind == 2) h->bmsk->writeData((const char *)pcm, (qint64)n * 2);
    else h->boq->writeData((const char *)pcm, (qint64)n * 2);
}
void jref_set_dcd(void *hv, int dcd)
{
    RefHandle *h = (RefHandle *)hv;
    if (h->kind == 0) h->oq->DCDstatSlot(dcd != 0);
    else if (h->kind == 1) h->msk->DCDstatSlot(dcd != 0);
    else if (h->kind == 2) h->bmsk->DCDstatSlot(dcd != 0);
}
// the run-time controls, through the reference's own slots (oqpskdemodulator.cpp:149-167,291-310, mskdemodulator.cpp:105-122,265-282)
void jref_set_center_freq(void *hv, double hz)
{ RefHandle *h = (RefHandle *)hv; if (h->kind == 0) h->oq->CenterFreqChangedSlot(hz); else if (h->kind == 1) h->msk->CenterFreqChangedSlot(hz); }
void jref_set_afc(void *hv, int v)
{ RefHandle *h = (RefHandle *)hv; if (h->kind == 0) h->oq->setAFC(v != 0); else if (h->kind == 1) h->msk->setAFC(v != 0); }
void jref_set_sql(void *hv, int v)
{ RefHandle *h = (RefHandle *)hv; if (h->kind == 0) h->oq->setSQL(v != 0); else if (h->kind == 1) h->msk->setSQL(v != 0); }
void jref_set_cpu_reduce(void *hv, int v)
{ RefHandle *h = (RefHandle *)hv; if (h->kind == 0) h->oq->setCPUReduce(v != 0); else if (h->kind == 1) h->msk->setCPUReduce(v != 0); }
long jref_ebno_log_take(void *hv, double *out, long cap)
{
    RefHandle *h = (RefHandle *)hv;
    long n = (long)h->ebno_log.size(); if (n > cap) n = cap;
    memcpy(out, h->ebno_log.data(), n * sizeof(double));
    h->ebno_log.clear();
    return n;
}
long jref_soft_count(void *hv) { return (long)((RefHandle *)hv)->soft.size(); }
long jref_soft_take(void *hv, short *out, long cap)
{
    RefHandle *h = (RefHandle *)hv;
    long n = (long)h->soft.size(); if (n > cap) n = cap;
    memcpy(out, h->soft.data(), n * sizeof(short));
    h->soft.erase(h->soft.begin(), h->soft.begin() + n);
    return n;
}
long jref_emit_count(void *hv) { return (long)((RefHandle *)hv)->emit_sizes.size(); }
long jref_cfe_log_take(void *hv, double *out, long cap)
{
    RefHandle *h = (RefHandle *)hv;
    long n = (long)h->cfe_log.size(); if (n > cap) n = cap;
    memcpy(out, h->cfe_log.data(), n * sizeof(double));
    h->cfe_log.erase(h->cfe_log.begin(), h->cfe_log.begin() + n);
    return n;
}
// loop-state snapshot; layout shared with jaero_status in include/jaero_b200.h
//  0 mixer2 freq Hz   1 mixer2 WTptr   2 mixer_center freq Hz  3 st_osc freq Hz  4 st_osc WTptr
//  5 AGC value        6 mse            7 EbNo                  8 marg (bias MA)  9 last coarse est
// 10 signal-true cnt 11 signal-false cnt 12 mixer_center WTptr 13 st_osc_ref WTptr (OQPSK)
int jref_state(void *hv, double *o)
{
    RefHandle *h = (RefHandle *)hv;
    if (h->kind == 0) {
        OqpskDemodulator *d = h->oq;
        o[0] = d->mixer2.freq; o[1] = d->mixer2.WTptr; o[2] = d->mixer_center.freq;
        o[3] = d->st_osc.freq; o[4] = d->st_osc.WTptr; o[5] = d->agc->AGCVal; o[6] = d->mse;
        o[7] = d->ebnomeasure->EbNo; o[8] = d->marg->Val; o[9] = d->coarsefreqestimate->freq_offset_est;
        o[10] = (double)h->n_signal_true; o[11] = (double)h->n_signal_false;
        o[12] = d->mixer_center.WTptr; o[13] = d->st_osc_ref.WTptr;
    } else if (h->kind == 1) {
        MskDemodulator *d = h->msk;
        o[0] = d->mixer2.freq; o[1] = d->mixer2.WTptr; o[2] = d->mixer_center.freq;
        o[3] = d->st_osc.freq; o[4] = d->st_osc.WTptr; o[5] = d->agc->AGCVal; o[6] = d->mse;
        o[7] = d->ebnomeasure->EbNo; o[8] = d->marg->Val; o[9] = d->coarsefreqestimate->freq_offset_est;
        o[10] = (double)h->n_signal_true; o[11] = (double)h->n_signal_false;
        o[12] = d->mixer_center.WTptr; o[13] = 0;
    } else if (h->kind == 2) {
        // burst layout: 8 = vol_gain, 9 = rotator_freq, 12 = cntr, 13 = startstop
        BurstMskDemodulator *d = h->bmsk;
        o[0] = d->mixer2.freq; o[1] = d->mixer2.WTptr; o[2] = d->mixer_center.freq;
        o[3] = d->st_osc.freq; o[4] = d->st_osc.WTptr; o[5] = d->agc->AGCVal; o[6] = d->mse;
        o[7] = d->ebnomeasure->EbNo; o[8] = d->vol_gain; o[9] = d->rotator_freq;
        o[10] = (double)h->n_signal_true; o[11] = (double)h->n_signal_false;
        o[12] = (double)d->cntr; o[13] = (double)d->startstop;
    } else {
        BurstOqpskDemodulator *d = h->boq;
        o[0] = d->mixer2.freq; o[1] = d->mixer2.WTptr; o[2] = d->mixer2.freq;
        o[3] = d->st_osc.freq; o[4] = d->st_osc.WTptr; o[5] = d->agc->AGCVal; o[6] = d->mse;
        o[7] = d->ebnomeasure->EbNo; o[8] = d->vol_gain; o[9] = d->rotator_freq;
        o[10] = (double)h->n_signal_true; o[11] = (double)h->n_signal_false;
        o[12] = (double)d->cntr; o[13] = (double)d->startstop;
    }
    return 14;
}
void jref_free(void *hv)
{
    RefHandle *h = (RefHandle *)hv;
    if (h->kind == 0) { g_handles.erase(h->oq); delete h->oq; } else if (h->kind == 1) { g_handles.erase(h->msk); delete h->msk; }
    else if (h->kind == 2) { g_handles.erase(h->bmsk); delete h->bmsk; } else { g_handles.erase(h->boq); delete h->boq; }
    delete h;
}

// ---------------- DSP primitives (DSP.h / DSP.cpp) ----------------
int jref_rrc_design(double alpha, int firsize, double Fs, double symbol_freq, double *out, int cap)
{
    RootRaisedCosine r; r.design(alpha, firsize, Fs, symbol_freq);
    int n = r.Points.size(); if (n > cap) n = cap;
    for (int i = 0; i < n; i++) out[i] = r.Points[i];
    return r.Points.size();
}
void jref_trig_tables(double *sinwt, double *coswt)
{
    for (int i = 0; i < WTSIZE; i++) { sinwt[i] = tringlookup.SinWT[i]; coswt[i] = tringlookup.CosWT[i]; }
}
void jref_fir(const double *taps, int ntaps, const double *x, double *y, long n)
{
    FIR f(ntaps);
    for (int i = 0; i < ntaps; i++) f.FIRSetPoint(i, taps[i]);
    for (long i = 0; i < n; i++) y[i] = f.FIRUpdateAndProcess(x[i]);
}
int jref_qround(double d) { return qRound(d); }
// n_lanes WaveTables, each running its own script: lane l's k-th operation is op[l*n_ops + k] with argument arg[l*n_ops + k]
// (the JAERO_OSC_* codes of include/jaero_b200.h: 0 SetFreq(a), 1 WTnextFrame(), 2 the index of WTCISValue() one frame ahead on a
// copy, 3 IncresePhaseDeg(a), 4 SetPhaseDeg(a), 5 AdvanceFractionOfWave(a), 6 IfHavePassedPoint(a), 7 SetFreq(a, samplerate)).
// Every lane starts with WTptr = last_WTptr = WTstep = freq = 0 at `samplerate`. After each operation
// log[(l*n_ops + k)*9 + f] holds f = 0 WTptr, 1 last_WTptr, 2 WTstep, 3 freq, 4 the index WTCISValue() read (tint),
// 5 what IfHavePassedPoint returned (0 for the other ops), 6 FractionOfSampleItPassesBy, 7-8 WTCISValue() (re, im).
void jref_wavetable_script(int n_lanes, int n_ops, const int32_t *op, const double *arg, double samplerate, double *log)
{
    for (int l = 0; l < n_lanes; l++) {
        WaveTable w;
        w.samplerate = samplerate; w.freq = 0; w.WTstep = 0; w.WTptr = 0; w.last_WTptr = 0; w.FractionOfSampleItPassesBy = 0;
        for (int k = 0; k < n_ops; k++) {
            const size_t e = (size_t)l * n_ops + k;
            const double a = arg[e];
            bool flag = false;
            cpx_type v;
            int tint;
            switch (op[e]) {
            case 0: w.SetFreq(a); break;
            case 1: w.WTnextFrame(); break;
            case 3: w.IncresePhaseDeg(a); break;
            case 4: w.SetPhaseDeg(a); break;
            case 5: w.AdvanceFractionOfWave(a); break;
            case 6: flag = w.IfHavePassedPoint(a); break;
            case 7: w.SetFreq(a, (int)samplerate); break;
            }
            if (op[e] == 2) { WaveTable c = w; c.WTnextFrame(); v = c.WTCISValue(); tint = c.tint; }
            else { v = w.WTCISValue(); tint = w.tint; }
            double *g = log + e * 9;
            g[0] = w.WTptr; g[1] = w.last_WTptr; g[2] = w.WTstep; g[3] = w.freq; g[4] = tint; g[5] = flag ? 1.0 : 0.0;
            g[6] = w.FractionOfSampleItPassesBy; g[7] = v.real(); g[8] = v.imag();
        }
    }
}

// ---------------- FFT wrappers (fftwrapper.cpp, fftrwrapper.cpp) ----------------
void jref_fft(int nfft, int inverse, const double *in_ri, double *out_ri)
{
    FFTWrapper<double> f(nfft, inverse != 0);
    QVector<cpx_type> a(nfft), b(nfft);
    for (int i = 0; i < nfft; i++) a[i] = cpx_type(in_ri[2 * i], in_ri[2 * i + 1]);
    f.transform(a, b);
    for (int i = 0; i < nfft; i++) { out_ri[2 * i] = b[i].real(); out_ri[2 * i + 1] = b[i].imag(); }
}
void jref_fftr_forward(int nfft, const double *in, double *out_ri)
{
    FFTrWrapper<double> f(nfft);
    QVector<double> a(nfft); QVector<cpx_type> b(nfft);
    for (int i = 0; i < nfft; i++) a[i] = in[i];
    f.transform(a, b);
    for (int i = 0; i < nfft; i++) { out_ri[2 * i] = b[i].real(); out_ri[2 * i + 1] = b[i].imag(); }
}
void jref_fftr_inverse(int nfft, const double *in_ri, double *out)
{
    FFTrWrapper<double> f(nfft);
    QVector<cpx_type> a(nfft); QVector<double> b(nfft);
    for (int i = 0; i < nfft; i++) a[i] = cpx_type(in_ri[2 * i], in_ri[2 * i + 1]);
    f.transform(a, b);
    for (int i = 0; i < nfft; i++) out[i] = b[i];
}
// JFastFir configured exactly as tests/jfastfir_tests.cpp:34-37
void jref_jfastfir_rrc(double alpha, int firsize, double Fs, double symbol_freq, int nfft, double *inout_ri, long n)
{
    JFastFir fir; RootRaisedCosine rrc;
    rrc.design(alpha, firsize, Fs, symbol_freq);
    fir.SetKernel(rrc.Points, nfft);
    QVector<cpx_type> v((int)n);
    for (long i = 0; i < n; i++) v[(int)i] = cpx_type(inout_ri[2 * i], inout_ri[2 * i + 1]);
    fir.update(v);
    for (long i = 0; i < n; i++) { inout_ri[2 * i] = v[(int)i].real(); inout_ri[2 * i + 1] = v[(int)i].imag(); }
}

// ---------------- CoarseFreqEstimate stand-alone (coarsefreqestimate.cpp:90-137) ----------------
void *jref_cfe_new(int fft_power, double lockingbw, double fb, double Fs)
{
    CoarseFreqEstimate *c = new CoarseFreqEstimate(0);
    c->setSettings(fft_power, lockingbw, fb, Fs);
    return c;
}
double jref_cfe_process(void *cv, const double *data_ri, double *y_out)
{
    CoarseFreqEstimate *c = (CoarseFreqEstimate *)cv;
    int n = (int)c->nfft;
    QVector<cpx_type> d(n);
    for (int i = 0; i < n; i++) d[i] = cpx_type(data_ri[2 * i], data_ri[2 * i + 1]);
    c->ProcessBasebandData(d);
    if (y_out) for (int i = 0; i < n; i++) y_out[i] = c->y[i];
    return c->freq_offset_est;
}
void jref_cfe_bigchange(void *cv) { ((CoarseFreqEstimate *)cv)->bigchange(); }
void jref_cfe_free(void *cv) { delete (CoarseFreqEstimate *)cv; }

// ---------------- Viterbi wrapper (jconvolutionalcodec.cpp) ----------------
void *jref_codec_new(int paddinglength)
{
    JConvolutionalCodec *c = new JConvolutionalCodec(0);
    QVector<quint16> polys; polys.push_back(109); polys.push_back(79);
    c->SetCode(2, 7, polys, paddinglength);          // as aerol.cpp:936-940
    return c;
}
int jref_codec_decode_continuous(void *cv, const uint8_t *soft, int n, int *bits_out)
{
    JConvolutionalCodec *c = (JConvolutionalCodec *)cv;
    QByteArray in((const char *)soft, n);
    QVector<int> &r = c->Decode_Continuous(in);
    for (int i = 0; i < r.size(); i++) bits_out[i] = r[i];
    return r.size();
}
int jref_codec_decode_soft(void *cv, const uint8_t *soft, int n, int *bits_out)
{
    JConvolutionalCodec *c = (JConvolutionalCodec *)cv;
    QByteArray in((const char *)soft, n);
    QVector<int> &r = c->Decode_soft(in, n);
    for (int i = 0; i < r.size(); i++) bits_out[i] = r[i];
    return r.size();
}
void jref_codec_free(void *cv) { delete (JConvolutionalCodec *)cv; }

} // extern "C"
