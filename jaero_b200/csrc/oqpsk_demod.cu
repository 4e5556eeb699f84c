// K1a — fused continuous OQPSK demodulator segment kernel (8400* / 10500 bps), one thread per channel.
//   (* the 8400 bps FFT pre-filter, oqpskdemodulator.cpp:343-381, is not part of this kernel yet)
//
// Replaces OqpskDemodulator::writeData (JAERO/oqpskdemodulator.cpp:334-627) and
// OqpskDemodulator::FreqOffsetEstimateSlot (:629-677) for a whole batch of channels:
// int16 -> coarse-estimator ring write -> NCO mix (table NCO, DSP.cpp:79-85) -> 55-tap RRC FIR x2
// (DSP.cpp:292-304) -> EbNo (DSP.cpp:729-744) -> AGC (DSP.cpp:370-379) -> clip -> symbol-timing chain
// (delays, resonator, T/8 quadrature, arg, PLL nudges :473-484) -> strobe interpolation (:488-494)
// -> carrier loop (:512-532) -> bias rotate / 400-symbol delay (:535-537) -> MSE gate (:563-565)
// -> soft bits (:569-592).
//
// The per-sample recursion is serial per channel (the carrier loop feeds the NCO ahead of the
// FIR), so the parallel axis is the channel: lane = channel, all sample-rate ring positions are
// warp-uniform, every HBM ring access is a coalesced 256 B row. FIR delay lines live in shared
// memory ([tap][lane], conflict-free), everything else in registers.
#include "demod_stages.cuh"

namespace jb {

static const int OQ_THREADS = 32;
static const int OQ_PROW = 80;            // bytes per channel row of a PCM tile in shared memory (64 B payload + pad)
// shared memory map (bytes): FIR windows (OQ_SM_FIR) | ring tiles x6 | PCM tiles x2 | mbarriers | pre-filtered tiles x2
static const int OQ_SM_PCM = OQ_THREADS * OQ_PROW;                     // one PCM tile
static const int OQ_XROW = 32 * 16 + 16;    // bytes per channel row of a pre-filtered-sample tile (32 double2 + pad)
static const int OQ_SM_X = OQ_THREADS * OQ_XROW;
static const int OQ_SM_TOTAL = OQ_SM_FIR + 6 * OQ_SM_RING + 2 * OQ_SM_PCM + 64;
static const int OQ_SM_TOTAL_PRE = OQ_SM_TOTAL + 2 * OQ_SM_X;

// PRE = true: the 8400 bps variant (oqpskdemodulator.cpp:436-448): no FIR in the loop, the sample entering the loop is
// mixer2.CIS * cval_prefiltered[i] (K6 output, staged like the PCM rows), and mixer2's frequency is summed per sample.
template <bool PRE>
__global__ void __launch_bounds__(OQ_THREADS)
oqpsk_segment_kernel(const __grid_constant__ DemodParams p, const SegmentArgs a, const int16_t *__restrict__ pcm, size_t stride,
                     const double2 *__restrict__ xpre, size_t xstride, double *__restrict__ m2_freq_sum)
{
    extern __shared__ __align__(128) unsigned char oq_smem_raw[];
    double *s_re = reinterpret_cast<double *>(oq_smem_raw);   // [OQ_FIRROWS][32]
    double *s_im = s_re + OQ_FIRROWS * OQ_THREADS;
    double *t_agc = reinterpret_cast<double *>(oq_smem_raw + OQ_SM_FIR);          // [2][T][32]
    double *t_e1 = t_agc + 2 * OQ_T * OQ_THREADS;
    double *t_e2 = t_e1 + 2 * OQ_T * OQ_THREADS;
    unsigned char *t_pcm = oq_smem_raw + OQ_SM_FIR + 6 * OQ_SM_RING;              // [2][32][OQ_PROW]
    unsigned long long *bars = reinterpret_cast<unsigned long long *>(t_pcm + 2 * OQ_SM_PCM);   // ring[2], pcm[2], x[2]
    unsigned char *t_x = oq_smem_raw + OQ_SM_TOTAL;                               // [2][32][OQ_XROW] (PRE only)
    const int lane = threadIdx.x;
    const int ch_raw = blockIdx.x * OQ_THREADS + lane;
    const bool live = ch_raw < p.n_channels;
    const int ch = ch_raw;                                    // dead lanes run on their (allocated) pad column with zero input
    const int nlive = min(OQ_THREADS, p.n_channels - (int)blockIdx.x * OQ_THREADS);
    const size_t cpad = p.cpad;
    if (lane == 0) { for (int k = 0; k < 6; k++) mbar_init(&bars[k], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncwarp();

    // ---------------- load state
    Osc m2 = load_osc(p, D_M2_PTR, ch), mc = load_osc(p, D_MC_PTR, ch), st = load_osc(p, D_ST_PTR, ch), sr = load_osc(p, D_SR_PTR, ch);
    double agc_sum = LD(D_AGC_SUM), agc_val = LD(D_AGC_VAL);
    double eb_sum1 = LD(D_EB_SUM1), eb_sum2 = LD(D_EB_SUM2), eb_ebno = LD(D_EB_EBNO);
    double dly_s0 = LD(D_DLY_S0);
    double d41_0 = LD(D_DLY41_0), d41_1 = LD(D_DLY41_1), d41_2 = LD(D_DLY41_2);
    double d42_0 = LD(D_DLY42_0), d42_1 = LD(D_DLY42_1), d42_2 = LD(D_DLY42_2);
    double d8_0 = LD(D_DLY8_0), d8_1 = LD(D_DLY8_1), d8_2 = LD(D_DLY8_2);
    Biquad res = load_biquad(p, D_RES_X1, ch);
    Biquad lf = load_biquad(p, D_LF_X1, ch);
    double2 sig2_last = make_double2(LD(D_SIG2L_RE), LD(D_SIG2L_IM));
    double2 pt_d = make_double2(LD(D_PTD_RE), LD(D_PTD_IM));
    OqpskTail tl = load_oqpsk_tail(p, ch);
    int yui = LI(I_YUI), countdown = LI(I_COUNTDOWN), countdown2 = LI(I_COUNTDOWN2), dcd = LI(I_DCD);
    int sig2l_init = LI(I_SIG2L_INIT);
    int sig_true = LI(I_SIG_TRUE), sig_false = LI(I_SIG_FALSE);

    fir_window_load2(p, s_re, s_im, OQ_NT1, ch, lane);
    if (a.new_write) tl.lastmse = tl.mse;                                 // oqpskdemodulator.cpp:339

    // ---------------- FreqOffsetEstimateSlot, re-entrant in the reference: it runs after the ring write and before the mixer
    // of the same sample.
    if (a.apply_cfe)
        oqpsk_freq_offset_slot(p, ch, live, p.cfe_est_out[ch], tl.mse, dcd, m2, mc, countdown, countdown2, sig_true, sig_false);

    // ---------------- lock-step positions
    const int agc_len = p.agc_len, eb_len = p.ebno_len;
    long long S = a.sample0;                                  // samples fully processed so far: drives every sample-rate ring
    int fir_pos = (int)(S % OQ_NT1);                          // next FIR slot to write
    int bb_pos = a.bb_pos, coarse_counter = a.coarse_counter;
    const bool ebno_on = p.report_ebno != 0;
    const int16_t *row = pcm + (size_t)ch * stride;
    double2 *bb_row = p.bb + (size_t)ch * p.bb_len;
    const int bbn = p.bb_len;
    const bool cpu_reduce = p.cpu_reduce != 0;
    const double Fs = p.Fs, fbr = p.fb, ee = p.ee;
    int p41 = (int)(S % (p.k41 + 1)), p8 = (int)(S % (p.k8 + 1));   // Delay<> ring positions (lock-step)
    const int k41 = p.k41, k8 = p.k8;
    const double *__restrict__ cos_t = p.cos_t, *__restrict__ sin_t = p.sin_t;
    const MeanDiv marg_mean(p.marg_len), mse_mean(p.mse_len);
    const int eb_from = a.i1 - OQ_EBNO_TAIL;
    const long long S_end = S + (a.i1 - a.i0) - (a.stop_after_a ? 1 : 0);   // value of S when this launch returns

    // ---------------- HBM streams staged through shared memory by the bulk-copy (TMA) engine.
    // The three sample-rate rings (AGC, EbNo E and E2: [slot][channel], 256 B per slot for this warp's 32 channels) and the
    // PCM rows are moved in tiles of 32 samples: lane r copies ring row r / its own PCM row with cp.async.bulk, completion
    // is signalled on an mbarrier, two buffers per stream, the next tile is in flight while the current one is consumed and
    // updated in place; finished ring tiles go back to HBM with bulk stores. The per-sample loop therefore never waits on
    // DRAM: its ring/PCM operands are shared-memory reads.
    auto ring_rows = [&](long long tile, double *&g_agc, double *&g_e1, double *&g_e2) {
        const long long s0 = tile * OQ_T;
        g_agc = p.agc_ring + ((size_t)(s0 % agc_len) + lane) * cpad + (size_t)blockIdx.x * OQ_THREADS;
        if (ebno_on) {
            g_e1 = p.ebno_e1 + ((size_t)(s0 % eb_len) + lane) * cpad + (size_t)blockIdx.x * OQ_THREADS;
            g_e2 = p.ebno_e2 + ((size_t)(s0 % eb_len) + lane) * cpad + (size_t)blockIdx.x * OQ_THREADS;
        }
    };
    const unsigned ring_tx = (ebno_on ? 3u : 1u) * OQ_SM_RING;
    auto ring_load = [&](long long tile) {                    // all lanes call; lane r moves row r of the tile
        const int b = (int)(tile & 1);
        fence_proxy_async();
        if (lane == 0) mbar_expect_tx(&bars[b], ring_tx);
        __syncwarp();
        double *g_agc = nullptr, *g_e1 = nullptr, *g_e2 = nullptr;
        ring_rows(tile, g_agc, g_e1, g_e2);
        bulk_g2s(t_agc + (b * OQ_T + lane) * OQ_THREADS, g_agc, OQ_THREADS * 8, &bars[b]);
        if (ebno_on) {
            bulk_g2s(t_e1 + (b * OQ_T + lane) * OQ_THREADS, g_e1, OQ_THREADS * 8, &bars[b]);
            bulk_g2s(t_e2 + (b * OQ_T + lane) * OQ_THREADS, g_e2, OQ_THREADS * 8, &bars[b]);
        }
    };
    auto ring_store = [&](long long tile) {                   // write the (in-place updated) tile back to HBM
        const int b = (int)(tile & 1);
        fence_proxy_async();
        __syncwarp();
        double *g_agc = nullptr, *g_e1 = nullptr, *g_e2 = nullptr;
        ring_rows(tile, g_agc, g_e1, g_e2);
        bulk_s2g(g_agc, t_agc + (b * OQ_T + lane) * OQ_THREADS, OQ_THREADS * 8);
        if (ebno_on) {
            bulk_s2g(g_e1, t_e1 + (b * OQ_T + lane) * OQ_THREADS, OQ_THREADS * 8);
            bulk_s2g(g_e2, t_e2 + (b * OQ_T + lane) * OQ_THREADS, OQ_THREADS * 8);
        }
        bulk_commit();
    };
    // PCM: tile t covers buffer samples [32t, 32t+32) of every channel row (16 B aligned: stride % 8 == 0, host-checked)
    auto pcm_bytes = [&](int tile) -> unsigned {
        long long left = (long long)stride - (long long)tile * OQ_T;
        if (left > OQ_T) left = OQ_T;
        return left > 0 ? (unsigned)(left * 2) : 0u;
    };
    auto pcm_load = [&](int tile) {
        const int b = tile & 1;
        const unsigned nb = pcm_bytes(tile);
        fence_proxy_async();
        if (lane == 0) mbar_expect_tx(&bars[2 + b], nb * (unsigned)nlive);
        __syncwarp();
        if (live && nb) bulk_g2s(t_pcm + b * OQ_SM_PCM + lane * OQ_PROW, row + (size_t)tile * OQ_T, nb, &bars[2 + b]);
        if (PRE) {
            long long left = (long long)xstride - (long long)tile * OQ_T;
            if (left > OQ_T) left = OQ_T;
            const unsigned xb = left > 0 ? (unsigned)(left * 16) : 0u;
            if (lane == 0) mbar_expect_tx(&bars[4 + b], xb * (unsigned)nlive);
            __syncwarp();
            if (live && xb) bulk_g2s(t_x + b * OQ_SM_X + lane * OQ_XROW, xpre + (size_t)ch * xstride + (size_t)tile * OQ_T, xb, &bars[4 + b]);
        }
    };
    unsigned phases = 0u;                                     // expected parity per barrier (bit b: ring b, bit 2+b: pcm b)
#define OQ_WAIT(idx) do { mbar_wait(&bars[(idx)], (phases >> (idx)) & 1u); phases ^= (1u << (idx)); } while (0)
    long long rt = S / OQ_T;                                  // current ring tile
    int pt = a.i0 / OQ_T;                                     // current PCM tile
    bool ring_next_issued = false, pcm_next_issued = false;
    ring_load(rt);
    pcm_load(pt);
    if ((rt + 1) * OQ_T < S_end) { ring_load(rt + 1); ring_next_issued = true; }
    if ((pt + 1) * OQ_T < a.i1) { pcm_load(pt + 1); pcm_next_issued = true; }
    OQ_WAIT((int)(rt & 1));
    OQ_WAIT(2 + (pt & 1));
    if (PRE) OQ_WAIT(4 + (pt & 1));
    bool ring_dirty = false;

    // ---- table / symbol-rate operands requested ahead of use (the SM issues in order: a load stalls the warp only when
    // its result is consumed)
    double c2_re, c2_im, cs_re, cs_im, cc_re, cc_im;
    { const int t = osc_index(m2.ptr); c2_re = cos_t[t]; c2_im = sin_t[t]; }
    { const int t = osc_index(st.ptr); cs_re = cos_t[t]; cs_im = sin_t[t]; }
    { const int t = osc_index(mc.ptr); cc_re = cos_t[t]; cc_im = sin_t[t]; }
    oqpsk_tail_prefetch(p, ch, tl);
    int4 pk = make_int4(0, 0, 0, 0);                          // 8 consecutive PCM samples of this lane's channel
    bool pk_valid = false;

    // FIR output of the first sample of this launch: the 55 entries older than the slot about to be written
    // (DSP.cpp:292-304: the output excludes the sample just stored). The window that ends at logical slot q starts at
    // row q+2 of the doubled buffer.
    double fre = 0, fim = 0;
    if (!PRE) {
        int newest = fir_pos - 1; if (newest < 0) newest += OQ_NT1;
        fir54(p, s_re + (newest + 2) * OQ_THREADS + lane, s_im + (newest + 2) * OQ_THREADS + lane, fre, fim);
        fre += p.taps[54] * s_re[(newest + 56) * OQ_THREADS + lane]; fim += p.taps[54] * s_im[(newest + 56) * OQ_THREADS + lane];
    }
    double m2sum = PRE ? (a.new_write ? 0.0 : m2_freq_sum[ch]) : 0.0;     // mixer2_freq_sum (:385,447)

    for (int i = a.i0; i < a.i1; i++) {
        // ---- PCM sample from the staged tile
        const int po = i & (OQ_T - 1);
        if ((i >> 5) != pt) {                                 // entered the next PCM tile (warp-uniform)
            pt = i >> 5;
            OQ_WAIT(2 + (pt & 1));
            if (PRE) OQ_WAIT(4 + (pt & 1));
            pcm_next_issued = false;
            if ((pt + 1) * OQ_T < a.i1) { pcm_load(pt + 1); pcm_next_issued = true; }
            pk_valid = false;
        }
        if (!pk_valid || (po & 7) == 0) {
            pk = *reinterpret_cast<const int4 *>(t_pcm + (pt & 1) * OQ_SM_PCM + lane * OQ_PROW + (po >> 3) * 16);
            pk_valid = true;
        }
        int cur_pcm;
        {
            const int k = po & 7;
            const int w = (k < 2) ? pk.x : (k < 4) ? pk.y : (k < 6) ? pk.z : pk.w;
            cur_pcm = (k & 1) ? (w >> 16) : (int)(short)(w & 0xffff);
            if (!live) cur_pcm = 0;
        }
        const double dval = ((double)cur_pcm) / 32768.0;                  // :390

        // ---- A: coarse-estimator ring (:410-429); the host ends the segment on the trigger sample
        if (!(i == a.i0 && a.skip_a_first)) {
            if (coarse_counter >= Fs || !cpu_reduce) {
                if (live) bb_row[bb_pos] = make_double2(cc_re * dval, cc_im * dval);
                bb_pos++; if (bb_pos >= bbn) bb_pos = 0;
            }
        }
        if (i == a.i1 - 1 && a.stop_after_a) break;
        coarse_counter++;                                                 // :431
        // mixer_center only free-runs inside the loop: advance it now (:601) and request its next table entry a whole
        // iteration before the ring write that consumes it
        osc_next_frame(mc);
        { const int t = osc_index(mc.ptr); cc_re = cos_t[t]; cc_im = sin_t[t]; }
        // speculative request for mixer2's next entry (right unless this sample turns out to be a carrier-update strobe)
        const int m2_spec = osc_next_index(m2);
        double n2_re = cos_t[m2_spec], n2_im = sin_t[m2_spec];

        // ---- B. cval = CIS * dval (:453) goes into the FIR ring; the output for THIS sample (fre,fim) was formed from
        // the older entries in the previous iteration, the output for the NEXT sample is formed now — an independent
        // dependency chain the scheduler interleaves with the serial loop arithmetic below.
        // The 54 older terms are summed first (same order as DSP.cpp:296-303), the newest term is appended once the mixed
        // sample is available.
        double nfre = 0, nfim = 0;
        if (!PRE) fir54(p, s_re + (fir_pos + 2) * OQ_THREADS + lane, s_im + (fir_pos + 2) * OQ_THREADS + lane, nfre, nfim);
        if (PRE) {
            // sig2 = mixer2.WTCISValue()*cval_prefiltered[i] (:440); mixer2_freq_sum+=mixer2.GetFreqHz() (:447)
            double2 xv = *reinterpret_cast<const double2 *>(t_x + (pt & 1) * OQ_SM_X + lane * OQ_XROW + po * 16);
            if (!live) xv = make_double2(0.0, 0.0);
            const double2 sg = c_mul(make_double2(c2_re, c2_im), xv);
            fre = sg.x; fim = sg.y;
            m2sum += m2.freq;
        }

        const double sre = fre, sim = fim;
        const double dabval = sqrt(sre * sre + sim * sim);                // :461

        const int ro = (int)(S & (OQ_T - 1));
        const int rslot = (((int)(rt & 1)) * OQ_T + ro) * OQ_THREADS + lane;   // this sample's slot in the staged ring tiles
        if (ebno_on) {                                                    // OQPSKEbNoMeasure::Update (DSP.cpp:729-744)
            const double sq = dabval * dabval;
            ma_push(eb_sum2, t_e2[rslot], sq);
            ma_push(eb_sum1, t_e1[rslot], dabval);
            if (i >= eb_from) oqpsk_ebno_readout(p.ebno_len, p.Fs, p.fb, eb_ebno, eb_sum1, eb_sum2);
        }

        {   // AGC::Update (DSP.cpp:370-379)
            ma_push(agc_sum, t_agc[rslot], dabval);
            ring_dirty = true;
            agc_val = agc_gain(MeanDiv(agc_len), agc_sum);
        }
        double2 sig2 = make_double2(sre * agc_val, sim * agc_val);        // :466
        const double abval = hypot(sig2.x, sig2.y);                       // :469 std::abs
        if (abval > 2.84) { const double g = (2.84 / abval); sig2 = make_double2(g * sig2.x, g * sig2.y); }   // :470

        // ---- symbol timing (:473-484)
        const double w41 = p.w41v[p41], w8 = p.w8v[p8];
        p41++; if (p41 > k41) p41 = 0;
        p8++; if (p8 > k8) p8 = 0;
        const double ab2 = abval * abval;
        const double st_diff = (0.0 * ab2 + (1.0 - 0.0) * dly_s0) - (ab2);    // Delay(1): weighting 0 -> x[n-1]
        dly_s0 = ab2;
        // Delay(T/4): older = x[n-k41], newer = x[n-k41+1]  (DSP.h:357-374)
        double st_d1out, st_d2out;
        {
            const double older = (k41 == 3) ? d41_2 : (k41 == 2 ? d41_1 : d41_0);
            const double newer = (k41 == 3) ? d41_1 : (k41 == 2 ? d41_0 : st_diff);
            st_d1out = (w41 * newer + (1.0 - w41) * older);
            d41_2 = d41_1; d41_1 = d41_0; d41_0 = st_diff;
        }
        {
            const double older = (k41 == 3) ? d42_2 : (k41 == 2 ? d42_1 : d42_0);
            const double newer = (k41 == 3) ? d42_1 : (k41 == 2 ? d42_0 : st_d1out);
            st_d2out = (w41 * newer + (1.0 - w41) * older);
            d42_2 = d42_1; d42_1 = d42_0; d42_0 = st_d1out;
        }
        double st_eta = (st_d2out - st_diff) * st_d1out;
        st_eta = biquad_update(res, st_eta, p.res_a1, p.res_a2, p.res_b0, p.res_b1, p.res_b2);
        double d8out;
        {
            const double older = (k8 == 3) ? d8_2 : (k8 == 2 ? d8_1 : d8_0);
            const double newer = (k8 == 3) ? d8_1 : (k8 == 2 ? d8_0 : st_eta);
            d8out = (w8 * newer + (1.0 - w8) * older);
            d8_2 = d8_1; d8_1 = d8_0; d8_0 = st_eta;
        }
        const double2 st_out = c_mul(make_double2(cs_re, cs_im), make_double2(st_eta, -d8out));   // :478-479
        const double st_angle_error = atan2_fast(st_out.y, st_out.x);          // :480 std::arg
        osc_set_freq(st, (-st_angle_error * 0.00000001) + st.freq, Fs);   // :481 IncreseFreqHz
        osc_advance_fraction_of_wave(st, -st_angle_error * 0.01 / 360.0); // :482
        if (st.freq < (sr.freq - 0.1)) osc_set_freq(st, (sr.freq - 0.1), Fs);
        if (st.freq > (sr.freq + 0.1)) osc_set_freq(st, (sr.freq + 0.1), Fs);

        if (!sig2l_init) { sig2_last = sig2; sig2l_init = 1; }            // :487 static initialiser
        double frac;
        if (osc_have_passed_point(st, ee, frac)) {                        // :488
            const double pt_last = frac, pt_this = 1.0 - pt_last;
            const double2 pt = make_double2(pt_this * sig2.x + pt_last * sig2_last.x, pt_this * sig2.y + pt_last * sig2_last.y);
            yui ^= 1;                                                     // yui++; yui%=2;
            if (!yui) pt_d = pt;
            else {
                double2 pt_qpsk = make_double2(pt.x, pt_d.y);             // :503
                double ct_ec = ct_error(pt, pt_d);
                if (fbr > 8400) {                                         // :518-525
                    ct_ec = biquad_update(lf, ct_ec, p.lf_a1, p.lf_a2, p.lf_b0, p.lf_b1, p.lf_b2);
                    if (ct_ec > M_PI_2) ct_ec = M_PI_2;
                    if (ct_ec < -M_PI_2) ct_ec = -M_PI_2;
                    osc_increase_phase_deg(m2, 1.0 * ct_ec);
                    osc_set_freq(m2, (0.01 * ct_ec) + m2.freq, Fs);
                } else {                                                  // :526-532
                    osc_increase_phase_deg(m2, 1.0 * ct_ec);
                    const double lfo = biquad_update(lf, ct_ec, p.lf_a1, p.lf_a2, p.lf_b0, p.lf_b1, p.lf_b2);
                    osc_set_freq(m2, (0.5 * 0.01 * lfo) + m2.freq, Fs);
                }
                oqpsk_symbol_tail(p, ch, live, tl, marg_mean, mse_mean, pt_qpsk, ct_ec);   // :535-592
            }
        }
        sig2_last = sig2;                                                 // :596
        if (!PRE) {   // this sample's mixed value enters the FIR ring (:453-456); finish the next output
            const double cre = c2_re * dval, cim = c2_im * dval;
            nfre += p.taps[54] * cre; nfim += p.taps[54] * cim;
            fir_push2(s_re, s_im, OQ_NT1, lane, fir_pos, cre, cim);
        }
        osc_next_frame(m2); osc_next_frame(st); osc_next_frame(sr);       // :600-603 (mixer_center advanced above)
        {
            const int t = osc_index(m2.ptr);
            if (t == m2_spec) { c2_re = n2_re; c2_im = n2_im; } else { c2_re = cos_t[t]; c2_im = sin_t[t]; }
        }
        { const int t = osc_index(st.ptr); cs_re = cos_t[t]; cs_im = sin_t[t]; }
        fre = nfre; fim = nfim;
        // ---- ring tile bookkeeping (warp-uniform)
        S++;
        if ((S & (OQ_T - 1)) == 0) {
            ring_store(rt);                                   // the finished tile goes back to HBM
            ring_dirty = false;
            rt++;
            if (S < S_end) {
                OQ_WAIT((int)(rt & 1));                       // next tile (requested a tile ago)
                ring_next_issued = false;
                if ((rt + 1) * OQ_T < S_end) {
                    bulk_wait_read_all();                     // the buffer being refilled must have been read out by its store
                    ring_load(rt + 1); ring_next_issued = true;
                }
            }
        }
    }
    // ---------------- drain the staging pipeline
    if (ring_dirty) ring_store(rt);
    if (ring_next_issued) OQ_WAIT((int)((rt + 1) & 1));
    if (pcm_next_issued) { OQ_WAIT(2 + ((pt + 1) & 1)); if (PRE) OQ_WAIT(4 + ((pt + 1) & 1)); }
    bulk_wait_all();

    // ---------------- store state
    store_osc(p, D_M2_PTR, ch, m2); store_osc(p, D_MC_PTR, ch, mc); store_osc(p, D_ST_PTR, ch, st); store_osc(p, D_SR_PTR, ch, sr);
    LD(D_AGC_SUM) = agc_sum; LD(D_AGC_VAL) = agc_val;
    LD(D_EB_SUM1) = eb_sum1; LD(D_EB_SUM2) = eb_sum2; LD(D_EB_EBNO) = eb_ebno;
    LD(D_DLY_S0) = dly_s0;
    LD(D_DLY41_0) = d41_0; LD(D_DLY41_1) = d41_1; LD(D_DLY41_2) = d41_2;
    LD(D_DLY42_0) = d42_0; LD(D_DLY42_1) = d42_1; LD(D_DLY42_2) = d42_2;
    LD(D_DLY8_0) = d8_0; LD(D_DLY8_1) = d8_1; LD(D_DLY8_2) = d8_2;
    store_biquad(p, D_RES_X1, ch, res);
    store_biquad(p, D_LF_X1, ch, lf);
    LD(D_SIG2L_RE) = sig2_last.x; LD(D_SIG2L_IM) = sig2_last.y;
    LD(D_PTD_RE) = pt_d.x; LD(D_PTD_IM) = pt_d.y;
    store_oqpsk_tail(p, ch, tl);
    if (PRE) m2_freq_sum[ch] = m2sum;
    LI(I_YUI) = yui; LI(I_COUNTDOWN) = countdown; LI(I_COUNTDOWN2) = countdown2; LI(I_SIG2L_INIT) = sig2l_init;
    LI(I_SIG_TRUE) = sig_true; LI(I_SIG_FALSE) = sig_false;
    fir_window_store(p, s_re, s_im, OQ_NT1, ch, lane, 0, 1);
}

int oqpsk_segment_launch(const DemodParams &p, const SegmentArgs &a, const int16_t *d_pcm, size_t stride, cudaStream_t s)
{
    const int grid = (p.n_channels + OQ_THREADS - 1) / OQ_THREADS;
    if (p.xpre) {
        const size_t smem = (size_t)OQ_SM_TOTAL_PRE;
        JB_CUDA(cudaFuncSetAttribute(oqpsk_segment_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        oqpsk_segment_kernel<true><<<grid, OQ_THREADS, smem, s>>>(p, a, d_pcm, stride, p.xpre, p.xstride, p.m2_freq_sum);
    } else {
        const size_t smem = (size_t)OQ_SM_TOTAL;
        JB_CUDA(cudaFuncSetAttribute(oqpsk_segment_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        oqpsk_segment_kernel<false><<<grid, OQ_THREADS, smem, s>>>(p, a, d_pcm, stride, nullptr, 0, nullptr);
    }
    JB_CUDA(cudaGetLastError());
    return 0;
}

} // namespace jb
