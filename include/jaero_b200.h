/* jaero_b200 — C ABI of the H100-native JAERO demodulator / Viterbi hot path.
 *
 * Drop-in boundary (SURVEY.md §8b). Every entry point below replaces a piece of the reference's
 * per-instance C++/Qt interface with a *batched* call over many independent channels; a single
 * reference object is a batch of one. Plain pointers and sizes only — no Qt, no torch, no CUDA
 * types. All functions return 0 on success or a negative JAERO_E_* code; jaero_last_error()
 * gives the message for the calling thread. There is NO CPU fallback: if no CUDA device is
 * usable the create calls fail with JAERO_E_CUDA.
 *
 *   reference interface (file:line)                               this header
 *   -------------------------------------------------------------  ---------------------------
 *   OqpskDemodulator::Settings  JAERO/oqpskdemodulator.h:20-39      jaero_settings
 *   MskDemodulator::Settings    JAERO/mskdemodulator.h:24-45        jaero_settings
 *   ctor + setSettings + setAFC/setSQL/setCPUReduce + start()
 *     JAERO/oqpskdemodulator.cpp:8-117,149-163,175-289,312-315      jaero_batch_create
 *     JAERO/mskdemodulator.cpp:9-84,105-118,135-263,296-299
 *   qint64 writeData(const char*, qint64)
 *     JAERO/oqpskdemodulator.cpp:334-627, mskdemodulator.cpp:313-488 jaero_batch_write[_device]
 *   signal processDemodulatedSoftBits(const QVector<short>&)
 *     JAERO/oqpskdemodulator.h:67, mskdemodulator.h:152             jaero_batch_read_softbits
 *   slot DCDstatSlot(bool)  oqpskdemodulator.cpp:679-684            jaero_batch_set_dcd
 *   slot CenterFreqChangedSlot(double) oqpskdemodulator.cpp:291-310 jaero_batch_set_center_freq
 *   signals MSESignal / EbNoMeasurmentSignal / SignalStatus / Plottables,
 *     getCurrentFreq()  oqpskdemodulator.cpp:322-325,670-675         jaero_batch_get_status
 *   CoarseFreqEstimate::ProcessBasebandData + FreqOffsetEstimateSlot
 *     JAERO/coarsefreqestimate.cpp:90-137, oqpskdemodulator.cpp:629-677   (inside jaero_batch_write)
 *   AeroLInterleaver::deinterleave_ba  JAERO/aerol.cpp:603-625       jaero_viterbi_decode_continuous(cols>0)
 *   JConvolutionalCodec::SetCode / Decode_Continuous / Decode_soft
 *     JAERO/jconvolutionalcodec.cpp:20-29,151-201,98-125            jaero_viterbi_*
 *   destructor                                                      jaero_batch_destroy / jaero_viterbi_destroy
 */
#ifndef JAERO_B200_H
#define JAERO_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define JAERO_OK 0
#define JAERO_E_ARG (-1)      /* bad argument */
#define JAERO_E_CUDA (-2)     /* CUDA runtime error / no device (no CPU fallback exists) */
#define JAERO_E_STATE (-3)    /* call not valid in this state */
#define JAERO_E_OVERFLOW (-4) /* a soft-bit ring overflowed because the caller did not drain it */

#define JAERO_KIND_OQPSK 0 /* continuous 8400/10500 bps OQPSK, JAERO/oqpskdemodulator.cpp */
#define JAERO_KIND_MSK 1   /* continuous 600/1200 bps MSK,     JAERO/mskdemodulator.cpp */

/* Same fields, defaults and units as the reference's Settings structs. */
typedef struct jaero_settings {
    int kind;                    /* JAERO_KIND_* */
    int coarsefreqest_fft_power; /* 14 (OQPSK) / 13 (MSK) */
    double freq_center;          /* Hz; used for every channel unless per-channel values are given */
    double lockingbw;            /* Hz */
    double fb;                   /* bits/s: 600, 1200, 8400, 10500 */
    double Fs;                   /* Hz, 48000 */
    double signalthreshold;      /* 0.65 (OQPSK) / 0.5 (MSK) */
    int afc;                     /* setAFC */
    int sql;                     /* setSQL */
    int cpu_reduce;              /* setCPUReduce */
    int report_ebno;             /* 1: keep the two 2 s EbNo moving averages (observable only) */
} jaero_settings;

/* Per-channel telemetry: what the reference emits as MSESignal, EbNoMeasurmentSignal,
 * SignalStatus, Plottables(freq_est, freq_center, bw) plus the loop state used by parity tests. */
typedef struct jaero_status {
    double mixer2_freq;   /* Hz  (Plottables freq_est) */
    double mixer2_wtptr;  /* NCO table pointer [0,19999) */
    double center_freq;   /* Hz  (getCurrentFreq) */
    double st_freq;       /* symbol-timing oscillator Hz */
    double st_wtptr;
    double agc;           /* AGC::AGCVal */
    double mse;           /* MSESignal */
    double ebno;          /* EbNoMeasurmentSignal (0 if report_ebno==0) */
    double marg;          /* residual-bias moving average */
    double cfe_est;       /* last coarse frequency estimate (Hz offset) */
    double n_sig_true;    /* SignalStatus(true) count */
    double n_sig_false;   /* SignalStatus(false) count */
    double center_wtptr;
    double st_ref_wtptr;
    int64_t samples;      /* samples consumed so far */
    int64_t softbits;     /* soft values emitted so far (drained + still in the ring; burst markers included) */
    int32_t dcd;
    int32_t reserved;
    double peak_volume;   /* PeakVolume (oqpskdemodulator.cpp:393-405): max |input sample| / 32768 since the previous status read */
    double scatter[4];    /* ScatterPoints, decimated: the two most recent constellation points (re, im, re, im) as pointbuff holds them */
} jaero_status;

typedef struct jaero_batch jaero_batch;
typedef struct jaero_viterbi jaero_viterbi;

const char *jaero_last_error(void);
int jaero_device_count(void);

/* n_channels independent demodulators of one mode on one GPU. freq_center_per_channel may be NULL. */
int jaero_batch_create(const jaero_settings *settings, int n_channels,
                       const double *freq_center_per_channel, int device_ordinal, jaero_batch **out);
void jaero_batch_destroy(jaero_batch *b);
int jaero_batch_channels(const jaero_batch *b);

/* writeData for every channel: pcm[ch*channel_stride + i], i < n_samples, little-endian int16 mono,
 * HOST memory (the call stages it to the GPU). Asynchronous with respect to the host unless
 * followed by a read/status call; ordering between calls is preserved. */
int jaero_batch_write(jaero_batch *b, const int16_t *pcm, size_t n_samples, size_t channel_stride);
/* Same, pcm already resident in this GPU's memory (device pointer). */
int jaero_batch_write_device(jaero_batch *b, const int16_t *d_pcm, size_t n_samples, size_t channel_stride);
/* Block until everything queued so far has executed. */
int jaero_batch_sync(jaero_batch *b);

/* Drain the soft bits emitted since the last read (the concatenated payloads of the reference's
 * processDemodulatedSoftBits emits: multiples of 32 (OQPSK) / 12 (MSK) values 0..255).
 * out[ch*cap + k]; counts[ch] = number written for that channel. HOST pointers. */
int jaero_batch_read_softbits(jaero_batch *b, int16_t *out, size_t cap_per_channel, int32_t *counts);
/* Device-resident view of the same rings for on-GPU consumers (d_soft[ch*ring_cap + k], d_counts[ch]);
 * valid until the next write. jaero_batch_reset_softbits() marks them consumed. */
int jaero_batch_softbits_device(jaero_batch *b, const int16_t **d_soft, const int32_t **d_counts, size_t *ring_cap);
int jaero_batch_reset_softbits(jaero_batch *b);

int jaero_batch_set_dcd(jaero_batch *b, int channel, int dcd);            /* channel<0: all */
int jaero_batch_set_center_freq(jaero_batch *b, int channel, double hz);  /* CenterFreqChangedSlot */
/* setAFC / setSQL / setCPUReduce of the reference classes: every channel of the batch, effective from the next write */
int jaero_batch_set_afc(jaero_batch *b, int state);
int jaero_batch_set_sql(jaero_batch *b, int state);
int jaero_batch_set_cpu_reduce(jaero_batch *b, int state);
/* Seating of the channels inside the 10500 bps kernel. Channels never interact, so results do not depend on it; throughput does:
 * the library seats channels with the same symbol-timing phase next to each other (automatically, every 128 estimator epochs
 * after the first two checks; this call does it now when slot_of is NULL, or installs the given permutation slot_of[channel] = seat). */
int jaero_batch_regroup(jaero_batch *b, const int32_t *slot_of);
/* connect(demodulator, SIGNAL(SignalStatus(bool)), aerol, SLOT(SignalStatusSlot(bool))) (JAERO/mainwindow.cpp:432,508): with it, a
 * SignalStatus(false) clears the channel's DCD in the kernel and is handed to the device frame layer (jaero_pchannel_process_batch /
 * jaero_cchannel_process_batch) as a LostSignal at its soft-bit position. Off by default (host-driven DCD via jaero_batch_set_dcd). */
int jaero_batch_wire_signal_status(jaero_batch *b, int enabled);
int jaero_batch_get_status(jaero_batch *b, int channel, jaero_status *out);
int jaero_batch_get_status_all(jaero_batch *b, jaero_status *out /* [n_channels] */);
/* kernel launches issued by this batch so far (for bench.py's gpu_launches) */
int64_t jaero_batch_launch_count(const jaero_batch *b);
/* Run on a caller-owned CUDA stream (a cudaStream_t passed as void*; NULL = back to the batch's own stream),
 * so the caller's events / other work order against the demodulator kernels. */
int jaero_batch_set_stream(jaero_batch *b, void *cuda_stream);
/* Measurement aid: when enabled, every segment-kernel launch and every coarse-estimator run is bracketed by CUDA
 * events on the launch stream; get_profile() synchronises and returns the accumulated device milliseconds and
 * launch counts since the last call: out[0]=segment ms, out[1]=segment launches, out[2]=estimator ms,
 * out[3]=estimator runs, out[4]=samples per channel covered by the segment launches. */
int jaero_batch_set_profiling(jaero_batch *b, int enabled);
int jaero_batch_get_profile(jaero_batch *b, double out[5]);
/* Coarse-estimator path of the batch: the number of co-resident 8-CTA clusters the nfft 2^14 estimator runs on, or 0 when it
 * runs as the four-step kernels through global memory (nfft up to 2^13, or no cluster fits the device). */
int jaero_batch_cfe_clusters(const jaero_batch *b);

/* ---- test support (not part of the drop-in surface) ----
 * One coarse-estimator epoch of a batch on a ring the caller supplies, with the batch's own plan, ring, smoothed spectrum y and
 * per-channel estimator state, so a test can compare the estimator kernels with an independent reference of
 * CoarseFreqEstimate::ProcessBasebandData (JAERO/coarsefreqestimate.cpp:84-137).
 * geometry: out = {nfft, ring length bb_len, fold search start lo, end hi (exclusive), expectedpeakbin, clusters of the write path}. */
int jaero_batch_cfe_geometry(const jaero_batch *b, int32_t out[6]);
/* Waits for the batch to be idle, copies ring[ch*bb_len + k] (complex, interleaved re/im) into the batch's baseband ring, applies
 * CoarseFreqEstimate::bigchange() to the channels with bigchange[ch] != 0 (NULL: none) as the demodulator kernels do, runs one
 * epoch linearised from ring index `oldest` and synchronises. impl: 0 the path jaero_batch_write takes, 1 the four-pass kernels,
 * 2 the cluster kernel (JAERO_E_STATE where it cannot run); max_clusters > 0 caps the clusters the cluster kernel is launched with,
 * and max_group > 0 the channels per pass group of the four-pass kernels (0: the batch's own, at most 1024).
 * y_out [n_channels][nfft] (the cluster kernel stores only bins lo-expectedpeakbin-1 .. hi+expectedpeakbin+1), raw_est [n_channels]
 * (freq_offset_est) and emitted_est [n_channels] (the gated value FreqOffsetEstimate carries) may each be NULL. Afterwards the
 * batch is in the state an estimator epoch of jaero_batch_write leaves it in, with the caller's ring as its baseband ring. */
int jaero_batch_probe_cfe(jaero_batch *b, const double *ring, int oldest, const int32_t *bigchange, int impl, int max_clusters,
                          int max_group, double *y_out, double *raw_est, double *emitted_est);
/* The streaming overlap-save FFT convolution of the 8400 bps pre-filter and the burst Hilbert filter (JFastFir: per channel,
 * y[n] = sum_k taps[k] x[n-L-k] for n >= 2L and 0 before, L = nfft - K + 1) on caller data, through the production host path and
 * block kernel, so a test can compare it with an independent reference. taps [K] complex, x and y [n_channels][n] complex
 * (interleaved re/im). writes[0 .. n_writes) is the sequence of write calls the samples arrive in; each must be > 0 and they
 * must add up to n. (K, nfft) must be a pair the library has a block kernel for: (2049, 4096) or (2048, 8192). Allocates and
 * frees its own buffers and stream on `device`. */
int jaero_probe_fastfir(int device, int nfft, const double *taps, int K, int n_channels, const double *x, size_t n,
                        const int32_t *writes, int n_writes, double *y);
/* The demodulators' device arithmetic primitives (jaero_b200/csrc/demod_device.cuh, cfe.cu) on caller operands, compiled with the
 * flags the product builds them with, so a test can compare them with exact and long-double references:
 * out[i] = op(a[i], b[i]) for i < n; integer results are returned as doubles. b is read only by the two-operand ops (NULL
 * otherwise). Allocates and frees its own buffers and stream on `device`. */
#define JAERO_MATH_DIV_EXACT 0     /* div_exact(a, b, 1.0 / b): the moving-average means (demod_kernels.cu, -fmad=false) */
#define JAERO_MATH_DIV_FAST 1      /* div_fast(a, b) as demod_kernels.cu compiles it */
#define JAERO_MATH_ATAN2_FAST 2    /* atan2_fast(y = a, x = b) */
#define JAERO_MATH_HYPOT_FAST 3    /* hypot_fast(a, b) */
#define JAERO_MATH_LOG10_GE1 4     /* log10_ge1(a), a >= 1, as cfe.cu compiles it */
#define JAERO_MATH_OSC_INDEX 5     /* osc_index(a): the WaveTable entry WTCISValue reads */
#define JAERO_MATH_Q_ROUND 6       /* q_round(a): qRound */
#define JAERO_MATH_FMOD360 7       /* fmod360(a): fmod(a, 360) */
#define JAERO_MATH_DIV_FAST_CFE 8  /* div_fast(a, b) as cfe.cu compiles it */
int jaero_probe_math(int device, int op, size_t n, const double *a, const double *b, double *out);
/* n_lanes independent WaveTable oscillators, each running its own script of n_ops operations through the device Osc helpers:
 * lane l's k-th operation is op[l*n_ops + k] applied with argument arg[l*n_ops + k]. Every lane starts at ptr = last = step =
 * freq = 0 and a passing fraction of 0, with sample rate `samplerate` (an integer for JAERO_OSC_SET_FREQ_SR). After each operation log[(l*n_ops + k)*7 + f] holds
 * f = 0 ptr, 1 last ptr, 2 step, 3 freq, 4 the table index (osc_index of ptr; for JAERO_OSC_NEXT_INDEX the index after the next
 * frame), 5 the flag JAERO_OSC_HAVE_PASSED_POINT returned (0 for the other ops), 6 the latest passing fraction. */
#define JAERO_OSC_SET_FREQ 0          /* osc_set_freq(arg): SetFreq(arg) */
#define JAERO_OSC_NEXT_FRAME 1        /* osc_next_frame: WTnextFrame() */
#define JAERO_OSC_NEXT_INDEX 2        /* osc_next_index: the index WTnextFrame() + WTCISValue() would read; the state is kept */
#define JAERO_OSC_INCREASE_PHASE_DEG 3 /* osc_increase_phase_deg(arg): IncresePhaseDeg(arg) */
#define JAERO_OSC_SET_PHASE_DEG 4     /* osc_set_phase_deg(arg): SetPhaseDeg(arg) */
#define JAERO_OSC_ADVANCE_FRACTION 5  /* osc_advance_fraction_of_wave(arg): AdvanceFractionOfWave(arg) */
#define JAERO_OSC_HAVE_PASSED_POINT 6 /* osc_have_passed_point(arg): IfHavePassedPoint(arg) */
#define JAERO_OSC_SET_FREQ_SR 7       /* osc_set_freq_wrap(arg, (int)samplerate): SetFreq(arg, samplerate), which also wraps ptr */
int jaero_probe_osc(int device, int n_lanes, int n_ops, const int32_t *op, const double *arg, double samplerate, double *log);

/* ---- K=7 r=1/2 soft Viterbi (polys 109,79), one independent decoder per channel ---- */
int jaero_viterbi_create(int n_channels, int paddinglength, int device_ordinal, jaero_viterbi **out);
void jaero_viterbi_destroy(jaero_viterbi *v);
/* Decode_Continuous for every channel: soft[ch*n_soft + k] (0..255, 128 = erasure), n_soft even.
 * interleaver_cols > 0: soft is the *interleaved* 64 x cols block and the de-interleave gather
 * (AeroLInterleaver::deinterleave_ba) is fused in front; 0: soft is already in code order.
 * bits_out[ch*(n_soft/2) + k] in {0,1}. The 62-value overlap is carried per channel. HOST pointers.
 * n_valid[ch] (may be NULL) = number of bits Decode_Continuous returns for that channel: n_soft/2,
 * except on a channel's first call after create/reset, where QVector::mid() truncates the result to
 * n_soft/2 - (paddinglength/2 + 1) (jconvolutionalcodec.cpp:194) — AeroL's frame alignment relies on it. */
int jaero_viterbi_decode_continuous(jaero_viterbi *v, const uint8_t *soft, size_t n_soft,
                                    int interleaver_cols, uint8_t *bits_out, int32_t *n_valid);
int jaero_viterbi_decode_continuous_device(jaero_viterbi *v, const uint8_t *d_soft, size_t n_soft,
                                           int interleaver_cols, uint8_t *d_bits_out, int32_t *d_n_valid);
/* Decode_soft (one-shot, no overlap / padding): n_soft/2 bits out per channel. */
int jaero_viterbi_decode_block(jaero_viterbi *v, const uint8_t *soft, size_t n_soft, uint8_t *bits_out);
int jaero_viterbi_reset(jaero_viterbi *v);   /* SetCode(): clears the overlap of every channel */
int jaero_viterbi_sync(jaero_viterbi *v);
int64_t jaero_viterbi_launch_count(const jaero_viterbi *v);

/* ---- P-channel frame layer (600 / 1200 / 10500 bps, continuous): soft bits -> CRC-checked signal units ----
 * Replaces AeroL::processDemodulatedSoftBits -> AeroL::Decode(bits,true) (JAERO/aerol.cpp:2077-2090,1124-2039,
 * non-burst branch), AeroL::updateDCD (:1109-1122) and the DataCarrierDetect -> DCDstatSlot feedback
 * (JAERO/mainwindow.cpp:234-237). */
typedef struct jaero_pchannel jaero_pchannel;
int jaero_pchannel_create(int n_channels, double fb, int device_ordinal, jaero_pchannel **out);
void jaero_pchannel_destroy(jaero_pchannel *p);
/* Consume everything the batch's demodulators emitted since the last call (device-resident, no host hop),
 * run framing + de-interleave + Viterbi + descramble + CRC, and write each channel's DCD back into the batch.
 * Known deviation (DESIGN.md §8): a frame's CRC-driven DCD countdown updates land at the end of the call that completed it,
 * after any UW sync later in that call, and a DCD they raise does not stop the 10.5 kbps UW search within that call. The DCD
 * written back to the demodulators follows the same rule. */
int jaero_pchannel_process_batch(jaero_pchannel *p, jaero_batch *b);
/* Same for soft bits supplied by the host: soft[ch*cap + k], counts[ch] (drop-in for processDemodulatedSoftBits). */
int jaero_pchannel_process_softbits(jaero_pchannel *p, const int16_t *soft, size_t cap_per_channel, const int32_t *counts);
/* AeroL::updateDCD: call once per second of signal (the reference's 1 s QTimer). b may be NULL. */
int jaero_pchannel_tick(jaero_pchannel *p, jaero_batch *b);
/* AeroL::SignalStatusSlot(false) -> AeroL::LostSignal() (JAERO/aerol.h:917-931): cntr = 1e9, DCD countdown = 0, DCD = false and
 * DataCarrierDetect(false) to the demodulator (b may be NULL: frame layer only). channel -1 = every channel. */
int jaero_pchannel_lost_signal(jaero_pchannel *p, jaero_batch *b, int channel);
/* writeData with the AeroL attached the way JAERO/mainwindow.cpp:198-237,432,508 wires the objects (HOST pcm): the stream is cut
 * in front of every coarse-estimator trigger sample and the frame layer runs at each cut, so FreqOffsetEstimateSlot reads the DCD
 * that results from exactly the soft bits emitted before that sample, and a SignalStatus(false) reaches LostSignal before any
 * later soft bit. Exact for OQPSK (DCD is only read in that slot); for MSK the timing-loop gain (mskdemodulator.cpp:387-405)
 * switches at the next cut, at most one estimator epoch (bbnfft/4 samples) after the reference's emit-granular switch.
 * Turns jaero_batch_wire_signal_status on for the batch. */
int jaero_pchannel_write_batch(jaero_pchannel *p, jaero_batch *b, const int16_t *pcm, size_t n_samples, size_t channel_stride);
/* Limits of one process call: a channel may hand over up to one full soft-bit ring (max(4096, 2*fb+64) values, i.e. 2 s of
 * signal at 10500 bps, 3.4 / 6.8 s at 1200 / 600 bps); more than that, or more signal units than jaero_pchannel_su_capacity()
 * left unread, raises the overflow flag: the next read_sus returns JAERO_E_OVERFLOW and the affected frames are incomplete. */
int jaero_pchannel_su_capacity(const jaero_pchannel *p);   /* SUs a channel can hold between two reads */
/* Drain decoded signal units: out[(ch*cap + k)*16 + 0..11] = SU bytes, [12] = CRC ok, [13] = index in frame,
 * [14..15] = frame number (LE). counts[ch] = SUs written. HOST pointers. */
int jaero_pchannel_read_sus(jaero_pchannel *p, uint8_t *out, size_t cap_per_channel, int32_t *counts);
/* Drop the queued signal units without copying them (device-side consumers / benchmarks). Asynchronous. */
int jaero_pchannel_discard_sus(jaero_pchannel *p);
/* dcd[ch], su_total[ch], su_ok[ch] (any may be NULL) */
int jaero_pchannel_get_stats(jaero_pchannel *p, int32_t *dcd, int64_t *su_total, int64_t *su_ok);
int64_t jaero_pchannel_launch_count(const jaero_pchannel *p);

/* ---- burst MSK demodulator (600 / 1200 bps R/T-channel bursts) ----
 * Replaces BurstMskDemodulator (JAERO/burstmskdemodulator.h:49-215): ctor + setSettings (burstmskdemodulator.cpp:11-323),
 * writeData (:371-754), DCDstatSlot (:757), and its processDemodulatedSoftBits / SignalStatus / EbNoMeasurmentSignal
 * signals. Soft-bit streams carry the reference's -1 "start of burst" marker. */
typedef struct jaero_burst jaero_burst;
typedef struct jaero_burst_status {
    double mixer2_freq, mixer2_wtptr, center_freq, st_freq, st_wtptr, agc, mse, ebno, vol_gain, rotator_freq;
    double n_sig_true, n_sig_false;   /* SignalStatus(true/false) emits */
    double cntr, startstop;
    double last_burst_ebno;           /* value of the most recent EbNoMeasurmentSignal */
    double n_ebno_emits;
} jaero_burst_status;
/* settings->kind is ignored; fb 600 or 1200, Fs 48000; freq_center / lockingbw / signalthreshold as BurstMskDemodulator::Settings */
int jaero_burst_msk_create(const jaero_settings *settings, int n_channels, int device_ordinal, jaero_burst **out);
/* Burst OQPSK demodulator (10500 bps C-channel / T-channel bursts): replaces BurstOqpskDemodulator
 * (JAERO/burstoqpskdemodulator.h), ctor + setSettings (burstoqpskdemodulator.cpp:4-277), writeData (:315-737) and its
 * processDemodulatedSoftBits / SignalStatus / EbNoMeasurmentSignal signals. fb 10500, Fs 48000; settings->sql as setSQL(). */
int jaero_burst_oqpsk_create(const jaero_settings *settings, int n_channels, int device_ordinal, jaero_burst **out);
void jaero_burst_destroy(jaero_burst *b);
int jaero_burst_write(jaero_burst *b, const int16_t *pcm, size_t n_samples, size_t channel_stride);          /* HOST pcm */
int jaero_burst_write_device(jaero_burst *b, const int16_t *d_pcm, size_t n_samples, size_t channel_stride);
int jaero_burst_read_softbits(jaero_burst *b, int16_t *out, size_t cap_per_channel, int32_t *counts);
int jaero_burst_set_dcd(jaero_burst *b, int channel, int dcd);
int jaero_burst_set_afc(jaero_burst *b, int state);                       /* setAFC (the constructors start with AFC on) */
int jaero_burst_set_sql(jaero_burst *b, int state);
int jaero_burst_get_status_all(jaero_burst *b, jaero_burst_status *out);
int jaero_burst_sync(jaero_burst *b);
int64_t jaero_burst_launch_count(const jaero_burst *b);
/* ---- test support (not part of the drop-in surface): the trident FFTs and peak searches of a burst batch on caller segments.
 * geometry: out = {tri_sz (samples of a fill), base_len, top_len (samples of the base / top section), nfft of the transforms}. */
int jaero_burst_trident_geometry(const jaero_burst *b, int32_t out[4]);
/* Writes segments[e][0 .. tri_sz) into trident slot ev_slot[e] of channel ev_channel[e] (each pair at most once, channel in
 * [0, n_channels), slot in [0, 8)), records the events in the event table as the front kernel would, and runs the trident
 * kernels in rounds of 128 events, as jaero_burst_write does. spectra_out [n_events][2][nfft] complex (NULL: not copied)
 * receives the base spectrum, then the top spectrum, of each event. With spectra_in (same layout) non-NULL the FFTs are
 * skipped and only the peak search of the batch's kind runs on the caller's spectra; segments may then be NULL.
 * result [n_events][5]: burst MSK {minvalbin, minval, maxtoppos, maxtopposhigh, arg(base[minvalbin])}, burst OQPSK
 * {minvalbin, |base[minvalbin]|, maxvalbin, maxval, arg(base[minvalbin])}.
 * The probe overwrites the batch's trident buffers and event table: afterwards the batch may only be destroyed. */
int jaero_burst_probe_trident(jaero_burst *b, int n_events, const int32_t *ev_channel, const int32_t *ev_slot, const double *segments,
                              const double *spectra_in, double *spectra_out, double *result);

/* ---- R/T burst channel layer (SURVEY.md section 8(f)2) ----
 * Replaces the burst branch of AeroL::Decode (JAERO/aerol.cpp:1124-1350, :1985-2031: unique-word detection with the
 * start-of-burst timing gates, sync / time-out handling), AeroL::updateDCD (:1109-1122) and RTChannelDeleaveFECScram
 * (JAERO/aerol.h:554-895: trial de-interleave + Decode_soft at every candidate packet length, descrambling, CRC-16
 * decisions, byte packing). Input: the soft-bit stream a burst demodulator emits (values 0..255, -1 = start of burst).
 * Output records are JAERO_RT_RECORD bytes: int32 type (1 = R packet, 2 = T packet), int32 number of SUs (T), int32
 * payload length, int32 index of the packet's first bit, then the payload (R: 19 bytes; T: 6-byte header + 12 per SU). */
#define JAERO_RT_RECORD 400
typedef struct jaero_rt jaero_rt;
int jaero_rt_create(double fb, int n_channels, int device_ordinal, jaero_rt **out);     /* fb 600 / 1200 (MSK) or 10500 (OQPSK) */
void jaero_rt_destroy(jaero_rt *r);
/* host soft bits: soft[ch * cap + i], counts[ch] values per channel (AeroL::processDemodulatedSoftBits) */
int jaero_rt_process_softbits(jaero_rt *r, const int16_t *soft, size_t cap_per_channel, const int32_t *counts);
/* Opt-in vector semantics: AeroL::Decode returns in the middle of a soft-bit vector when the burst time-out fires
 * (JAERO/aerol.cpp:2018-2027) and the rest of that vector is lost. With it on, jaero_rt_process_burst drops the rest of the
 * demodulator's emit (12 / 32 values, +1 with the start marker) and jaero_rt_process_softbits treats each call as one vector.
 * Off (default): nothing is dropped. */
int jaero_rt_set_vector_mode(jaero_rt *r, int enabled);
/* consume (and drain) the soft bits a burst demodulator batch has produced, entirely on the device */
int jaero_rt_process_burst(jaero_rt *r, jaero_burst *b);
int jaero_rt_tick(jaero_rt *r);                                                          /* the 1 s updateDCD timer */
int jaero_rt_read_packets(jaero_rt *r, uint8_t *out, int cap_packets_per_channel, int32_t *counts);
int jaero_rt_get_stats(jaero_rt *r, int32_t *n_trial_decodes, int32_t *n_bad_packets, int32_t *dcd);   /* any may be NULL */
int64_t jaero_rt_launch_count(const jaero_rt *r);

/* ---- C-channel (8400 bps) frame layer (SURVEY.md section 8(f)3) ----
 * Replaces AeroL::DecodeC (JAERO/aerol.cpp:2187-2500): dual unique-word detector with I/Q ambiguity correction
 * (:848-896), 16 x (64 x 4) de-interleave, PuncturedCode::depunture_soft_block(...,4) (:2505-2518), Decode_Continuous,
 * delay line, scrambler, the three sub-band signal units per frame with CRC-16 + DCD countdown, the 25 x 12-byte voice
 * payload (what Voicesignal carries to the vocoder). Output records are JAERO_C_RECORD bytes: 3 x {12 SU bytes, crc_ok,
 * 3 pad}, 300 voice bytes, int32 frame number. */
#define JAERO_C_RECORD 352
typedef struct jaero_cchannel jaero_cchannel;
int jaero_cchannel_create(int n_channels, int device_ordinal, jaero_cchannel **out);
void jaero_cchannel_destroy(jaero_cchannel *c);
int jaero_cchannel_process_batch(jaero_cchannel *c, jaero_batch *b);      /* consume (and drain) an 8400 bps batch's soft bits on the device; DCD fed back */
int jaero_cchannel_process_softbits(jaero_cchannel *c, const int16_t *soft, size_t cap_per_channel, const int32_t *counts);
int jaero_cchannel_tick(jaero_cchannel *c, jaero_batch *b);               /* the 1 s updateDCD timer; b may be NULL */
int jaero_cchannel_lost_signal(jaero_cchannel *c, jaero_batch *b, int channel);   /* AeroL::LostSignal, as jaero_pchannel_lost_signal */
int jaero_cchannel_write_batch(jaero_cchannel *c, jaero_batch *b, const int16_t *pcm, size_t n_samples, size_t channel_stride);   /* as jaero_pchannel_write_batch */
int jaero_cchannel_read_frames(jaero_cchannel *c, uint8_t *out, int cap_frames_per_channel, int32_t *counts);
int jaero_cchannel_get_stats(jaero_cchannel *c, int32_t *dcd, int64_t *su_total, int64_t *su_ok);   /* any may be NULL */
int64_t jaero_cchannel_launch_count(const jaero_cchannel *c);

/* ---- ingest router (SURVEY.md section 8(f)4, host side) ----
 * The reference's many-channel feed is one ZMQ PUB topic per channel, each message three frames
 * [topic][uint32 sample rate][int16 PCM] (JAERO/zmq_audioreceiver.cpp:37-87; the subscription is the first 5 bytes of the
 * topic, :46) delivered to dataReceived(audio, sampleRate). The router takes the frames as the transport delivers them (no
 * libzmq dependency), files the PCM under the matching channel and feeds whole batches to jaero_batch_write. */
typedef struct jaero_ingest jaero_ingest;
int jaero_ingest_create(int n_channels, const char *const *topics, uint32_t sample_rate, size_t capacity_samples, jaero_ingest **out);
void jaero_ingest_destroy(jaero_ingest *g);
/* returns the channel index (>= 0) or a negative error. JAERO_E_OVERFLOW: the channel's buffer cannot take the whole message;
 * NOTHING of it was filed - flush the batch (jaero_ingest_flush) and hand the same message over again. */
int jaero_ingest_message(jaero_ingest *g, const void *topic, size_t topic_len, const void *rate, size_t rate_len, const void *pcm, size_t pcm_bytes);
size_t jaero_ingest_available(const jaero_ingest *g);                  /* samples every channel has */
int jaero_ingest_flush(jaero_ingest *g, jaero_batch *b, size_t n_samples);

/* ---- wideband IQ digital down-converter (DDC) ----
 * Turns one complex IQ stream from a software radio (interleaved cu8 as an RTL-SDR delivers it, or cs16) into one real int16 PCM
 * stream per channel at output rate Fs_out = input_rate / decimation, the audio input of the demodulators (Fs 48000). The PCM
 * stays in device memory for jaero_batch_write_device / jaero_burst_write_device. Per channel c, with input x[n] counted from
 * create (x[n<0] = 0; cu8: (v - 127.5) / 128, cs16: v / 32768), T_c = round(offset_hz[c] / input_rate * 2^32) mod 2^32 and
 * S_c = round(audio_hz[c] / Fs_out * 2^32) mod 2^32:
 *   z[n] = x[n] exp(-2 pi i ((n T_c) mod 2^32) / 2^32);  u[j] = sum_k h1[k] z[j D1 - k];  v[m] = sum_k h2[k] u[m D2 - k]
 *   pcm[m] = clamp(rint(gain * 32768 * Re{v[m] exp(2 pi i ((m S_c) mod 2^32) / 2^32)}), -32768, 32767)  (rint: half to even)
 * Output m exists once input m * decimation has arrived: N inputs give floor((N - 1) / decimation) + 1 outputs per channel, and
 * the output does not depend on how the stream is cut into writes. After a retune, a stage-1 sample u[j] uses the offset in force
 * when input j * D1 arrives and an output m the audio frequency in force when input m * decimation arrives.
 * Filters (jaero_ddc_plan): real low-pass stages, h1 decimating by D1 and h2 by D2 (D1 * D2 = decimation; D2 = 1, h2 = {1} is a
 * single stage), whose composite response passes |f| <= bandwidth/2 around the offset within +-0.1 dB of its 0 Hz gain and
 * attenuates every tone with |f| >= bandwidth/2 + transition, up to +-input_rate/2 and aliases included, by at least 70 dB.
 *
 * Rational rates (jaero_ddc_plan_rational, jaero_ddc_create_rational): for a radio whose rate is not a multiple of 48 kHz, the
 * output rate is Fs_out = input_rate * L / M for coprime L (interpolation, 1 to 256) and M (decimation). Stage 1 is as above with
 * D1 dividing M; stage 2 is a polyphase resampler, M2 = M / D1:
 *   w[i] = u[i / L] if L divides i, else 0   (u[j < 0] = 0);   v[m] = sum_k h2[k] w[m M2 - k]   (h2 sums to L: unit passband gain)
 * and pcm[m] as above, with Fs_out = input_rate * L / M in S_c. Output m exists once input floor(m M / L) has arrived: N inputs
 * give ceil(N L / M) outputs per channel, and everything output m reads has arrived by then. An output m uses the audio
 * frequency in force when input floor(m M / L) arrives; the offset rule is unchanged. The output does not depend on how the
 * stream is cut into writes. The filter specification is the one above, the images of the x L zero-stuffing included. With
 * L = 1 every formula reduces to the one above term by term, and jaero_ddc_plan / jaero_ddc_create are exactly those calls.
 * Every other jaero_ddc_* call works on either kind of handle. */
#define JAERO_IQ_CU8 0   /* interleaved unsigned 8-bit I, Q */
#define JAERO_IQ_CS16 1  /* interleaved signed 16-bit I, Q */
typedef struct jaero_ddc jaero_ddc;
/* Host only, no device needed: the stages create would use, stages = {D1, K1, D2, K2} (K = number of taps); h1 [K1] and h2 [K2]
 * receive the taps unless NULL (pass NULL to query the lengths first). */
int jaero_ddc_plan(double input_rate, int decimation, double bandwidth, double transition, int32_t stages[4], double *h1, double *h2);
/* Rejects a channel whose |offset_hz| exceeds input_rate/2 - bandwidth/2 or whose audio passband
 * [audio_hz - bandwidth/2, audio_hz + bandwidth/2] leaves (0, Fs_out/2). */
int jaero_ddc_create(double input_rate, int decimation, int n_channels, const double *offset_hz, const double *audio_hz,
                     double bandwidth, double transition, double gain, int device_ordinal, jaero_ddc **out);
/* The same at output rate input_rate * interpolation / decimation: stages = {L, D1, K1, M2, K2}, h2 the K2-tap prototype at
 * L * input_rate / D1 (summing to L). Rejects L outside 1..256, a ratio with a common factor (reduce it), and a ratio for which no
 * split meets the filter specification within the tap limits. */
int jaero_ddc_plan_rational(double input_rate, int interpolation, int decimation, double bandwidth, double transition, int32_t stages[5],
                            double *h1, double *h2);
int jaero_ddc_create_rational(double input_rate, int interpolation, int decimation, int n_channels, const double *offset_hz,
                              const double *audio_hz, double bandwidth, double transition, double gain, int device_ordinal, jaero_ddc **out);
void jaero_ddc_destroy(jaero_ddc *d);
/* n_iq complex samples, format JAERO_IQ_*. HOST iq (copied before the call returns) */
int jaero_ddc_write(jaero_ddc *d, const void *iq, size_t n_iq, int format);
/* Same, iq resident in this GPU's memory (aligned to one sample) */
int jaero_ddc_write_device(jaero_ddc *d, const void *d_iq, size_t n_iq, int format);
/* The PCM the last write produced: d_pcm[ch * stride + i], i < n, device memory, rows 16-byte aligned (stride a multiple of 8).
 * Valid until the next write and ordered on the DDC's stream: put the consuming batch on the same stream (jaero_batch_set_stream,
 * jaero_ddc_set_stream). */
int jaero_ddc_output(jaero_ddc *d, const int16_t **d_pcm, size_t *n, size_t *stride);
/* Host copy of the same: out[ch * cap_per_channel + i]; *n = outputs per channel. Synchronises. */
int jaero_ddc_read_pcm(jaero_ddc *d, int16_t *out, size_t cap_per_channel, size_t *n);
/* Run on a caller-owned CUDA stream (cudaStream_t as void*; NULL = back to the DDC's own stream) */
int jaero_ddc_set_stream(jaero_ddc *d, void *cuda_stream);
/* Retune between writes (channel -1: every channel); same limits as create. Ordered on the DDC's stream: writes issued before
 * the call use the old value, later writes the new one; the host does not wait. */
int jaero_ddc_set_offset(jaero_ddc *d, int channel, double hz);
int jaero_ddc_set_audio_freq(jaero_ddc *d, int channel, double hz);
/* input samples written so far; clipped [n_channels] output samples clamped to the int16 range (either may be NULL) */
int jaero_ddc_get_stats(jaero_ddc *d, int64_t *inputs, int64_t *clipped);
int64_t jaero_ddc_launch_count(const jaero_ddc *d);

/* ---- PCM rate converter ----
 * Brings int16 PCM recorded at another audio rate (44100 Hz, say) to the demodulators' rate (Fs 48000) on the device, so that no
 * CPU resampler sits in front of jaero_batch_write_device / jaero_burst_write_device.
 *   Input: n_channels independent int16 PCM streams at input_rate, channel-major with a row stride as jaero_batch_write takes
 *   them; channel c's samples are x_c[n], counted from create, with x_c[n<0] = 0.
 *   Rates: whole hertz. L / M = output_rate / input_rate, reduced to lowest terms here; rejected when L = M = 1, L > 1024 or
 *   M > 1024. (8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 88200, 96000 and 192000 Hz into 48000, 24000 or 12000 Hz
 *   all fit; 11025 -> 48000 Hz is L = 640.)
 *   Filter: one real Kaiser low-pass prototype h of K taps at L * input_rate, summing to L (unit gain at DC). It passes
 *   [0, passband_hz] within +-0.1 dB and attenuates [min(input_rate, output_rate)/2, L * input_rate/2] by at least 70 dB (designed
 *   for 76 dB), one stopband for the aliases of the decimation and the images of the x L zero-stuffing. Rejected when
 *   passband_hz >= min(input_rate, output_rate)/2 or when the design needs more than 2^17 taps.
 *   Output, per channel c:
 *     w_c[i] = x_c[i / L] if L divides i, else 0;   v_c[m] = sum_k h[k] w_c[m M - k]
 *     pcm_c[m] = clamp(rint(v_c[m]), -32768, 32767)  (rint: half to even); clamped samples are counted per channel.
 *   Output m exists once input floor(m M / L) has arrived: N inputs give ceil(N L / M) outputs per channel. The output does not
 *   depend on how the stream is cut into writes. A write of 0 samples queues nothing and its output is empty. Sample positions
 *   are 64-bit. */
typedef struct jaero_resample jaero_resample;
/* Host only, no device needed: stages = {L, M, K}; h [K] receives the prototype unless NULL (pass NULL to query K first). */
int jaero_resample_plan(double input_rate, double output_rate, double passband_hz, int32_t stages[3], double *h);
/* n_channels streams at input_rate -> output_rate. Fails with JAERO_E_CUDA without a device. */
int jaero_resample_create(double input_rate, double output_rate, int n_channels, double passband_hz, int device_ordinal, jaero_resample **out);
void jaero_resample_destroy(jaero_resample *s);
/* n_samples per channel, pcm[ch * channel_stride + i], channel_stride >= n_samples. HOST pcm (copied before the call returns) */
int jaero_resample_write(jaero_resample *s, const int16_t *pcm, size_t n_samples, size_t channel_stride);
/* Same, pcm resident in this GPU's memory */
int jaero_resample_write_device(jaero_resample *s, const int16_t *d_pcm, size_t n_samples, size_t channel_stride);
/* The PCM the last write produced: d_pcm[ch * stride + i], i < n, device memory, rows 16-byte aligned (stride a multiple of 8).
 * Valid until the next write and ordered on the resampler's stream: put the consuming batch on the same stream. */
int jaero_resample_output(jaero_resample *s, const int16_t **d_pcm, size_t *n, size_t *stride);
/* Host copy of the same: out[ch * cap_per_channel + i]; *n = outputs per channel. Synchronises. */
int jaero_resample_read_pcm(jaero_resample *s, int16_t *out, size_t cap_per_channel, size_t *n);
/* Run on a caller-owned CUDA stream (cudaStream_t as void*; NULL = back to the resampler's own stream) */
int jaero_resample_set_stream(jaero_resample *s, void *cuda_stream);
/* input samples per channel written so far; clipped [n_channels] output samples clamped to the int16 range (either may be NULL) */
int jaero_resample_get_stats(jaero_resample *s, int64_t *inputs, int64_t *clipped);
int64_t jaero_resample_launch_count(const jaero_resample *s);

/* ---- wideband carrier scanner ----
 * Finds the carriers in the IQ stream the down-converter takes, so that its channels can be planned from the stream itself.
 * The scanner averages the stream's power spectrum on the device; jaero_scan_find_carriers (host only) finds and measures the
 * carriers in it. Spectrum contract:
 *   Input: x[n] converted as the DDC converts it (cu8: (v - 127.5) / 128, cs16: v / 32768), counted from create or the last reset.
 *   Frames: frame f is x[f * hop + n], n < nfft; it counts once its last sample has arrived. Window: periodic Hann,
 *   w[n] = 0.5 - 0.5 cos(2 pi n / nfft). With X_f[k] = sum_n w[n] x[f hop + n] exp(-2 pi i k n / nfft) and F frames:
 *     mean[i] = (1/F) sum_f |X_f[k]|^2 / sum_n w[n]^2,   max_hold[i] = max_f |X_f[k]|^2 / sum_n w[n]^2
 *   in fftshift order: index i is bin k = (i + nfft/2) mod nfft, at (i - nfft/2) * input_rate / nfft Hz from the tuner centre.
 *   Units: complex white noise of variance s^2 gives mean ~ s^2 in every bin; a carrier's mean-square power is
 *   (1/nfft) * sum over its bins of (mean - floor). A bursty carrier shows its burst level in max_hold and is diluted by its duty
 *   cycle in mean.
 *   The per-frame powers are added into the running sum in frame order, so mean and max_hold are bit-identical however the
 *   stream is cut into writes. With no frame yet, both are 0. */
#define JAERO_MODE_UNKNOWN 0
#define JAERO_MODE_MSK600 1
#define JAERO_MODE_MSK1200 2
#define JAERO_MODE_OQPSK8400 3
#define JAERO_MODE_OQPSK10500 4
#define JAERO_CARRIER_AT_DC 1     /* |center_hz| < dc_guard_hz: an RTL-SDR's DC spike may be all there is */
#define JAERO_CARRIER_AT_EDGE 2   /* the run touches the first or last bin: the carrier may extend past the band */
typedef struct jaero_scan jaero_scan;
/* nfft a power of two from 2^10 to 2^16, 1 <= hop <= nfft, input_rate > 0. Fails with JAERO_E_CUDA without a device. */
int jaero_scan_create(double input_rate, int nfft, int hop, int device_ordinal, jaero_scan **out);
void jaero_scan_destroy(jaero_scan *s);
/* n_iq complex samples, format JAERO_IQ_CU8 / JAERO_IQ_CS16. HOST iq (copied before the call returns). A failed write leaves the
 * average unchanged. */
int jaero_scan_write(jaero_scan *s, const void *iq, size_t n_iq, int format);
/* Same, iq resident in this GPU's memory (aligned to one sample) */
int jaero_scan_write_device(jaero_scan *s, const void *d_iq, size_t n_iq, int format);
/* Run on a caller-owned CUDA stream (cudaStream_t as void*; NULL = back to the scanner's own stream) */
int jaero_scan_set_stream(jaero_scan *s, void *cuda_stream);
/* Start a new average: the frame count, the sample origin, mean and max_hold restart */
int jaero_scan_reset(jaero_scan *s);
/* mean [nfft] and max_hold [nfft] (either may be NULL), *frames = frames averaged (may be NULL). Synchronises. */
int jaero_scan_read(jaero_scan *s, double *mean, double *max_hold, int64_t *frames);
int64_t jaero_scan_launch_count(const jaero_scan *s);

/* Carrier finding, host only (no device), on any spectrum laid out as jaero_scan_read returns it (nfft as for create, values
 * finite and >= 0). params NULL: the defaults {3 dB, 100 kHz, 0.25, 200 Hz, 0 Hz}.
 *   floor: W = the odd integer nearest floor_window_hz / bin_hz (2 floor(x/2) + 1), clamped to [3, nfft]; floor[i] is the order
 *     statistic of index floor((W - 1) * floor_quantile) of psd[s .. s+W-1], s = clamp(i - (W-1)/2, 0, nfft - W). A low
 *     quantile keeps the floor right where much of a window is occupied.
 *   runs: bin i is occupied when psd[i] >= floor[i] * 10^(threshold_db/10); carriers are the maximal runs of occupied bins with
 *     (bins * bin_hz) >= min_width_hz.
 *   per run, e = psd - floor: lo_hz / hi_hz the first / last bin's frequency; peak_hz the strongest bin (largest psd, the first
 *     on ties); center_hz the centroid of e (peak_hz if sum e <= 0); power = sum e / nfft; snr_db = 10 log10(sum e / sum floor);
 *     peak_db = 10 log10(max psd / floor); floor = the floor at the peak bin; width_hz the half-power width of e around the peak:
 *     with `top` the mean e of the run's bins whose e is at least half the run's largest e, from the peak outwards to the first
 *     bin whose e is below top / 2, each crossing interpolated linearly between that bin and the one before it (the band's
 *     first / last bin when there is none). The mean over the top, not the single largest bin, sets the level because the
 *     largest of many noisy bins lies well above the true peak of an averaged spectrum. mode: the JAERO_MODE_* whose nominal half-power
 *     width is nearest to width_hz on a log scale, UNKNOWN when the ratio to it is outside [0.8, 1.25].
 * Carriers come out in ascending frequency, at most cap of them; *n_found is the total even when cap is smaller. */
typedef struct jaero_scan_params {
    double threshold_db;      /* > 0 */
    double floor_window_hz;   /* > 0 */
    double floor_quantile;    /* [0, 1] */
    double min_width_hz;      /* >= 0 */
    double dc_guard_hz;       /* >= 0 */
} jaero_scan_params;
typedef struct jaero_carrier {
    double center_hz, peak_hz, lo_hz, hi_hz, width_hz, power, snr_db, peak_db, floor;
    int32_t mode;             /* JAERO_MODE_* hint */
    int32_t flags;            /* JAERO_CARRIER_* */
} jaero_carrier;
int jaero_scan_find_carriers(const double *psd, int nfft, double input_rate, const jaero_scan_params *params,
                             jaero_carrier *out, int cap, int *n_found);

/* ---- mode identifier ----
 * Tells each PCM channel's JAERO bit rate and carrier frequency from the spectral lines of its square. Squaring an MSK or OQPSK
 * carrier at fc leaves two discrete lines at 2 fc +- fb / 2: their distance is the bit rate and their midpoint twice the carrier
 * (the physics of the reference's CoarseFreqEstimate, searched here at every JAERO rate over the whole band). The identifier
 * averages the squared signal's power spectrum on the device; jaero_ident_classify (host only) finds the line pair in it.
 * Spectrum contract, per channel c of n_channels int16 PCM streams at Fs (channel-major with a row stride, as jaero_batch_write
 * takes them, so down-converter, rate-converter or recording output feeds it directly):
 *   x_c[n] = pcm_c[n] / 32768, counted from create or the last reset. N = nfft, hop = N / 2; frame f is x_c[f hop + n], n < N,
 *   and counts once its last sample has arrived. w[n] = 0.5 - 0.5 cos(2 pi n / N) (periodic Hann). Per frame:
 *     X[k] = sum_n w[n] x_c[f hop + n] exp(-2 pi i k n / N)
 *     A[k] = 2 X[k] for 0 < k < N/2, else 0                  (the analytic signal, without its DC and Nyquist bins)
 *     a[n] = (1/N) sum_k A[k] exp(+2 pi i k n / N)
 *     Y[k] = sum_n a[n]^2 exp(-2 pi i k n / N)
 *   sq_mean_c[i] = (1/F) sum_f |Y_f[k]|^2 / (sum_n w[n]^2)^2 over the F frames so far, in fftshift order: index i is bin
 *   k = (i + N/2) mod N, at (i - N/2) Fs / N Hz of the squared signal, twice the PCM frequency modulo Fs. A unit cosine at a bin
 *   centre gives 1 at its 2f bin. Frames are added in frame order, so sq_mean is bit-identical however the stream is cut into
 *   writes and whatever the batch's channel count and order. With no frame yet it is 0.
 * Limits: Fs whole hertz in [8000, 192000]; nfft a power of two from 2^10 to 2^14; anything else is JAERO_E_ARG. */
typedef struct jaero_ident jaero_ident;
/* Fails with JAERO_E_CUDA without a device. */
int jaero_ident_create(double Fs, int n_channels, int nfft, int device_ordinal, jaero_ident **out);
void jaero_ident_destroy(jaero_ident *d);
/* n_samples per channel, pcm[ch * channel_stride + i], channel_stride >= n_samples. HOST pcm (copied before the call returns).
 * A failed write leaves the average unchanged. */
int jaero_ident_write(jaero_ident *d, const int16_t *pcm, size_t n_samples, size_t channel_stride);
/* Same, pcm resident in this GPU's memory (aligned to one sample), e.g. jaero_ddc_output's on the same stream */
int jaero_ident_write_device(jaero_ident *d, const int16_t *d_pcm, size_t n_samples, size_t channel_stride);
/* Run on a caller-owned CUDA stream (cudaStream_t as void*; NULL = back to the identifier's own stream) */
int jaero_ident_set_stream(jaero_ident *d, void *cuda_stream);
/* Start a new average: the frame count, the sample origin and sq_mean restart */
int jaero_ident_reset(jaero_ident *d);
/* sq_mean [n_channels][nfft] (may be NULL), *frames = frames averaged per channel (may be NULL). Synchronises. */
int jaero_ident_read(jaero_ident *d, double *sq_mean, int64_t *frames);
int64_t jaero_ident_launch_count(const jaero_ident *d);

/* Classification, host only (no device), of one channel's sq_mean (nfft and Fs as for create, values finite and >= 0).
 * params NULL: the defaults {5 dB, 400 Hz, 0.5}. 5 dB lies between the
 * largest score of noise (about 3 dB over 4 s) and the weakest right rate at Eb/N0 4 dB (600 bps, about 6.5 dB).
 *   floor: jaero_scan_find_carriers' sliding order statistic with floor_window_hz and floor_quantile, bin_hz = Fs / nfft.
 *   Q[i] = sq_mean[i] / floor[i], 0 where floor[i] is 0.
 *   For each mode m in (MSK600, MSK1200, OQPSK8400, OQPSK10500), fb_m = 600, 1200, 8400, 10500, D_m = round(fb_m nfft / Fs)
 *   (half away from zero): score_m = max over i of min(Q[i], max over e in (-1, 0, +1) of Q[(i + D_m + e) mod nfft]), the first i
 *   on ties, and for it the first e with the largest Q; j = i + D_m + e. score_db[m] = 10 log10(score_m) (-HUGE_VAL for 0).
 *   best = the mode with the largest score (the first on ties); margin_db = score_db[best] - the largest other score_db.
 *   Each line of best's pair (bins i and j mod nfft) is refined by a log-parabolic fit through its bin and its two neighbours
 *   (indices mod nfft): delta = (l- - l+) / (2 (l- - 2 l0 + l+)) with l = ln sq_mean, clamped to [-0.5, 0.5]; 0 when any of the
 *   three values is <= 0 or the denominator is 0. With p = i + delta_i and q = j + delta_j (j unwrapped), bin_hz = Fs / nfft:
 *     line_hz[0] = (i + delta_i - nfft/2) bin_hz,  line_hz[1] = ((j mod nfft) + delta_j - nfft/2) bin_hz   (squared signal)
 *     fb_hz = (q - p) bin_hz,  carrier_hz = ((mid mod Fs) + Fs) mod Fs / 2 with mid = ((p + q) / 2 - nfft/2) bin_hz, in [0, Fs/2)
 *   mode = best if score_db[best] >= threshold_db, else JAERO_MODE_UNKNOWN. frames is 0 here: the classifier sees only the
 *   spectrum; jaero_ident_read reports the frames behind it. */
typedef struct jaero_ident_params {
    double threshold_db;      /* finite */
    double floor_window_hz;   /* > 0 */
    double floor_quantile;    /* [0, 1] */
} jaero_ident_params;
typedef struct jaero_ident_result {
    double carrier_hz;        /* PCM frequency of the carrier, [0, Fs/2) */
    double fb_hz;             /* measured distance between the lines */
    double line_hz[2];        /* the lines, Hz of the squared signal */
    double score_db[4];       /* per mode, JAERO_MODE_* - 1 */
    double margin_db;
    int64_t frames;
    int32_t mode;             /* JAERO_MODE_* */
} jaero_ident_result;
int jaero_ident_classify(const double *sq_mean, int nfft, double Fs, const jaero_ident_params *params, jaero_ident_result *out);

/* ---- ISU / SSU reassembly and ACARS block parsing (SURVEY.md section 8(f)4, host side) ----
 * One handle per channel. Replaces RISUData::update (JAERO/aerol.cpp:27-112), ISUData::update (:151-214),
 * ParserISU::parse (:340-487) and ACARSDefragmenter (:221-329), fed the way AeroL::Decode feeds them (:1357-1399 R
 * packets, :1497-1513 T packets, :1900-1925 P-channel signal units). Pure host code, no device. The aircraft-database
 * look-up of ParserISU::acarslookupresult (:493-520) is not part of this library; only its removal of the leading dots of
 * the registration is applied. Input signal units must be CRC-valid (the device layers report crc_ok per unit). */
#define JAERO_REASM_ACARS 0      /* record kinds */
#define JAERO_REASM_ERROR 1      /* text = the reference's Errorsignal string */
#define JAERO_REASM_COMPLETE 1   /* push return bits: an ISU completed */
#define JAERO_REASM_MISSING 2    /* a subsequent signal unit had no open sequence */
#define JAERO_REASM_PARSED 4     /* the completed ISU was accepted by the parser */
#define JAERO_ACARS_NONACARS 1   /* flags: user data is not an ACARS block, text = its bytes in hex */
#define JAERO_ACARS_DOWNLINK 2
#define JAERO_ACARS_VALID 4
#define JAERO_ACARS_HASTEXT 8
#define JAERO_ACARS_MORE 16
typedef struct jaero_acars_record {
    int32_t kind;
    uint32_t aes_id;                 /* ISUItem: AESID, GESID, QNO, REFNO, SEQNO, NOOCTLESTINLASTSSU */
    uint8_t ges_id, qno, refno, seqno, last_octets;
    uint8_t mode, tak, block_id;     /* ACARSItem: MODE, TAK, BI */
    uint8_t label[2], label_len;     /* LABEL */
    uint8_t reg[7], reg_len;         /* PLANEREG */
    uint8_t flags;                   /* JAERO_ACARS_* */
    uint32_t userdata_len;           /* bytes of ISU user data the record was parsed from */
    uint32_t text_len;               /* bytes of message text (or error text) */
} jaero_acars_record;
typedef struct jaero_reasm jaero_reasm;
int jaero_reasm_create(jaero_reasm **out);
void jaero_reasm_destroy(jaero_reasm *h);
int jaero_reasm_reset(jaero_reasm *h);                                      /* AeroL::setSettings (:992-993) */
int jaero_reasm_short_frame(jaero_reasm *h);                                /* the short-frame reset (:1997) */
/* one P- or T-channel signal unit (first 10 of its 12 bytes are used); returns JAERO_REASM_* bits or a negative error */
int jaero_reasm_push_su(jaero_reasm *h, const uint8_t *su, int downlink);
/* one R-channel packet (first 17 of its 19 bytes are used) */
int jaero_reasm_push_r(jaero_reasm *h, const uint8_t *info, int downlink);
/* one T-channel packet as jaero_rt_read_packets returns it: 6-byte header + n_sus x 12 bytes */
int jaero_reasm_push_t_packet(jaero_reasm *h, const uint8_t *info, int n_sus);
int jaero_reasm_pending(const jaero_reasm *h);
/* pops the oldest record; returns the text length, -1 when there is none, -2 when cap < rec->text_len (nothing popped) */
long jaero_reasm_pop(jaero_reasm *h, jaero_acars_record *rec, char *text, size_t cap);
int jaero_reasm_get_stats(const jaero_reasm *h, uint64_t *isus, uint64_t *messages, uint64_t *errors, uint64_t *missing);   /* any may be NULL */

#ifdef __cplusplus
}
#endif
#endif
