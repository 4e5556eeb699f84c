// Device-side data layout of the continuous demodulators (K1a OQPSK, K1b MSK) and the coarse
// frequency estimator (K2). Product code, sm_90a only.
//
// One GPU thread owns one channel for the serial part of the loop; everything a channel keeps
// between samples lives in HBM as structure-of-arrays with the CHANNEL index minor
// (element [k][ch]), so that a warp of 32 channels touches 32 consecutive doubles whenever the
// ring position k is common to all channels — which it is for every sample-rate ring (AGC, EbNo,
// FIR, delay lines), because all channels of a batch advance in lock-step. Symbol-rate rings
// (marg, dt, MSE) have per-channel positions and are simply gathered.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace jb {

static const int LOST_CAP = 64;           // SignalStatus(false) events a channel can record between two drains of its soft ring
static const int MAX_TAPS = 160;          // MSK 600 bps @48 kHz: 2*SPS = 160 (mskdemodulator.cpp:164)

// ---- per-channel scalar state, doubles: D[idx][channel]
enum DIdx {
    // WaveTable x4: WTptr, WTstep, freq, last_WTptr  (DSP.h:64,75-79)
    D_M2_PTR, D_M2_STEP, D_M2_FREQ, D_M2_LAST,
    D_MC_PTR, D_MC_STEP, D_MC_FREQ, D_MC_LAST,
    D_ST_PTR, D_ST_STEP, D_ST_FREQ, D_ST_LAST,
    D_SR_PTR, D_SR_STEP, D_SR_FREQ, D_SR_LAST,          // st_osc_ref (OQPSK only)
    D_AGC_SUM, D_AGC_VAL,
    D_EB_SUM1, D_EB_SUM2, D_EB_EBNO,                    // E, E2 running sums, smoothed EbNo
    D_DLY_S0,                                           // delays(1):   x[n-1]
    D_DLY41_0, D_DLY41_1, D_DLY41_2,                    // delayt41:    x[n-1..n-3]
    D_DLY42_0, D_DLY42_1, D_DLY42_2,
    D_DLY8_0, D_DLY8_1, D_DLY8_2,                       // delayt8 (OQPSK fractional)
    D_RES_X1, D_RES_X2, D_RES_Y1, D_RES_Y2,             // st_iir_resonator history (x[n-1],x[n-2],y[n-1],y[n-2])
    D_LF_X1, D_LF_X2, D_LF_Y1, D_LF_Y2,                 // ct_iir_loopfilter history
    D_SIG2L_RE, D_SIG2L_IM,                             // sig2_last (static, oqpskdemodulator.cpp:487)
    D_PTD_RE, D_PTD_IM,                                 // pt_d      (static, :498)
    D_MARG_SUM, D_MARG_VAL,
    D_MSE_PM_SUM, D_MSE_MA_SUM, D_MSE,
    D_DIFF_LAST,                                        // DiffDecode::lastsoftstate (MSK)
    D_CFE_EST,                                          // last CoarseFreqEstimate::freq_offset_est
    D_LASTMSE,                                          // `lastmse` captured at the start of writeData (:339)
    D_SCAT0_RE, D_SCAT0_IM, D_SCAT1_RE, D_SCAT1_IM,     // the two most recent constellation points (ScatterPoints, decimated)
    D_COUNT
};
// ---- per-channel scalar state, ints: I[idx][channel]
enum IIdx {
    I_YUI, I_COUNTDOWN, I_COUNTDOWN2, I_DCD, I_SIG2L_INIT,
    I_MARG_POS, I_DT_POS, I_MSE_POS,
    I_SOFT_COUNT, I_SOFT_PENDING, I_SOFT_OVERFLOW,
    I_SIG_TRUE, I_SIG_FALSE, I_EMPTYING,                // SignalStatus counters, CoarseFreqEstimate::emptyingcountdown
    I_ZERO_BB,                                          // request: clear the baseband ring (oqpskdemodulator.cpp:667)
    I_LOST_N,                                           // SignalStatus(false) events recorded since the soft ring was last drained
    I_PEAK,                                             // max |int16 input sample| since the last status read (PeakVolume)
    I_COUNT
};

struct DemodParams {
    int kind, n_channels, cpad;       // cpad = n_channels rounded up to 32 (row pitch of every [k][ch] array)
    double Fs, fb, lockingbw, signalthreshold, ee;
    int afc, sql, cpu_reduce, report_ebno;
    int ntaps;                        // 55 (OQPSK) / 2*SPS (MSK)
    int agc_len, ebno_len, bbnfft;
    int bb_len;                       // entries per row of the coarse-estimator ring (= bbnfft)
    int marg_len, dt_len, mse_len;    // 800/401/400 (OQPSK) ; SPS / SPS/2+1 / 600 (MSK)
    int sps;                          // MSK: int(Fs/fb)
    double correctionfactor;          // MSK
    double res_a1, res_a2, res_b0, res_b1, res_b2;   // st_iir_resonator (a0 = 1)
    double lf_a1, lf_a2, lf_b0, lf_b1, lf_b2;        // ct_iir_loopfilter
    double w41v[4], w8v[4];           // Delay<> interpolation weight at each ring position (DSP.h:357-374 computes it from buffptr)
    int k41, k8;                      // ceil(fd) for T/4 and T/8; ring sizes are k+1
    int soft_cap;                     // per-channel soft-bit ring capacity (shorts)
    // device pointers
    double *D; int *I;
    double *agc_ring, *ebno_e1, *ebno_e2;
    double *fir_re, *fir_im;          // [(ntaps+1)][cpad]
    double2 *bb;                      // [ch][bb_len]   (channel-major: rows feed the FFT directly)
    double *marg_ring, *mse_pm, *mse_ma;
    double2 *dt_ring;
    double2 *dsmpl_ring;              // MSK delayedsmpl [(sps+1)][cpad]
    double *dly8_ring;                // MSK delayt8 (integer delay SPS/2) [(sps/2+1)][cpad]
    int16_t *soft;                    // [ch][soft_cap]
    long long *soft_total;            // [cpad] soft values drained from the ring so far (jaero_status.softbits)
    // connect(demodulator, SignalStatus(bool), aerol, SignalStatusSlot(bool)) (JAERO/mainwindow.cpp:432,508): when wired, a
    // SignalStatus(false) at the end of FreqOffsetEstimateSlot is AeroL::LostSignal (aerol.h:921-931), which answers with
    // DataCarrierDetect(false) at once: the kernel clears the channel's DCD and records the soft-bit position of the event for
    // the device frame layer (lost_pos[k][ch] = soft values emitted before event k).
    int wire_sigstat; int *lost_pos;  // [LOST_CAP][cpad]
    const int *chan_of;               // [cpad] channel seated at (cta, lane) of the pipelined 10500 bps kernel (null: identity)
    const double *sin_t, *cos_t;      // the reference's 19999-entry tables (DSP.cpp:19-20), built on the host
    double *cfe_est_out;              // [ch] value CoarseFreqEstimate would emit this epoch
    const double2 *xpre;              // 8400 bps: K6 output of the current call [ch][xstride] (null otherwise)
    size_t xstride;
    double *m2_freq_sum;              // 8400 bps: running mixer2_freq_sum of the current call [cpad]
    // matched-filter taps of THIS batch (FIR::FIRSetPoint, DSP.cpp:283-286). They travel in the kernel parameter block
    // (constant bank, uniform loads), so batches of different modes can be alive on one GPU at the same time.
    double taps[MAX_TAPS];
};

// Uniform (lock-step) positions the host tracks and passes per launch.
struct SegmentArgs {
    long long sample0;                // samples consumed before this launch (drives every sample-rate ring)
    int i0, i1;                       // sample indices of this launch inside the pcm buffer
    int skip_a_first;                 // the first sample's ring write / trigger test was already done
    int stop_after_a;                 // the last sample only does its ring write (coarse estimate follows)
    int apply_cfe;                    // run FreqOffsetEstimateSlot(cfe_est_out[ch]) before anything else
    int bb_pos, coarse_counter;       // bbcycbuff_ptr, coarseCounter at entry
    int new_write;                    // first launch of a writeData call: latch lastmse
};

int oqpsk_segment_launch(const DemodParams &p, const SegmentArgs &a, const int16_t *d_pcm, size_t stride, cudaStream_t s);
int oqpsk_pipe_launch(const DemodParams &p, const SegmentArgs &a, const int16_t *d_pcm, size_t stride, cudaStream_t s);
int msk_pipe_launch(const DemodParams &p, const SegmentArgs &a, const int16_t *d_pcm, size_t stride, cudaStream_t s);

// test support (jaero_probe_math / jaero_probe_osc): the device arithmetic primitives of demod_device.cuh on caller operands, each
// compiled in the unit whose flags the product builds it with. op is a JAERO_MATH_* / JAERO_OSC_* code of include/jaero_b200.h.
int probe_math_launch(int op, size_t n, const double *a, const double *b, double *out, cudaStream_t s);       // demod_kernels.cu
int probe_math_cfe_launch(int op, size_t n, const double *a, const double *b, double *out, cudaStream_t s);   // cfe.cu
int probe_osc_launch(int n_lanes, int n_ops, const int32_t *op, const double *arg, double samplerate, double *log, cudaStream_t s);

// K2: coarse frequency estimate for every channel of a batch (coarsefreqestimate.cpp:90-137)
struct CfePlan {
    int nfft, n1, n2, startbin, stopbin, expectedpeakbin, lo, hi, is8400;
    double hzperbin;
    double2 *tw;        // W_nfft^k, k < nfft
    double2 *work_a, *work_b;   // [group][nfft]
    double *y;          // [ch][nfft]  smoothed log spectrum (fft-shifted order, as the reference keeps it)
    double *window;     // 8400 only
    int clusters;       // >0: nfft 16384 runs in the cluster-resident kernel with this many co-resident clusters
    int group;          // channels per pass group (sized so the work buffers stay L2-resident)
};
int cfe_run(const CfePlan &plan, const DemodParams &p, int oldest, cudaStream_t s, long long *launches);
int cfe_cluster_run(const CfePlan &plan, const DemodParams &p, int oldest, int n_clusters, cudaStream_t s, long long *launches);
int cfe_cluster_capacity();

} // namespace jb
