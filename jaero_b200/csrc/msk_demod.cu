// K1b — fused continuous MSK demodulator segment kernel (600 / 1200 bps), one thread per channel.
//
// Replaces MskDemodulator::writeData (JAERO/mskdemodulator.cpp:313-488) and
// MskDemodulator::FreqOffsetEstimateSlot (:490-519): int16 -> coarse-estimator ring -> NCO mix ->
// half-sine matched filter 2*SPS taps x2 (:164-170, DSP.cpp:292-304) -> EbNo (DSP.cpp:493-505) -> AGC
// -> clip -> one-symbol delay (:384) -> resonator on |pt_msk| + T/2 quadrature + PLL with tanh
// weighting (:387-405) -> strobe (:408): carrier loop (:411-426), bias rotate (:429-431), MSE (:446-448),
// differential soft decode (:451-469, DSP.cpp:531-563), emit every 12 soft bits (:472-476).
// Same layout rules as K1a (oqpsk_demod.cu): lane = channel, lock-step ring positions.
#include "demod_stages.cuh"

namespace jb {

static const int MSK_THREADS = 32;

__global__ void __launch_bounds__(MSK_THREADS)
msk_segment_kernel(const __grid_constant__ DemodParams p, const SegmentArgs a, const int16_t *__restrict__ pcm, size_t stride,
                   int d8_k, double d8_w)
{
    extern __shared__ double smem_d[];
    const int nt1 = p.ntaps + 1;                       // FIR ring length (DSP.cpp:277)
    double *s_re = smem_d;                             // [nt1][32]
    double *s_im = smem_d + (size_t)nt1 * MSK_THREADS;
    const int lane = threadIdx.x;
    const int ch = blockIdx.x * MSK_THREADS + lane;
    if (ch >= p.n_channels) return;

    Osc m2 = load_osc(p, D_M2_PTR, ch), mc = load_osc(p, D_MC_PTR, ch), st = load_osc(p, D_ST_PTR, ch);
    double agc_sum, agc_val, eb_sum1, eb_sum2, eb_ebno;
    int countdown, dcd, sig_true, sig_false;
    {   // (a row pitch held across the sample loop below costs this kernel 30 registers: the loop indexes with p.cpad)
        const size_t cpad = p.cpad;
        agc_sum = LD(D_AGC_SUM); agc_val = LD(D_AGC_VAL);
        eb_sum1 = LD(D_EB_SUM1); eb_sum2 = LD(D_EB_SUM2); eb_ebno = LD(D_EB_EBNO);
        countdown = LI(I_COUNTDOWN); dcd = LI(I_DCD); sig_true = LI(I_SIG_TRUE); sig_false = LI(I_SIG_FALSE);
    }
    Biquad res = load_biquad(p, D_RES_X1, ch);
    MskTail tl = load_msk_tail(p, ch);
    fir_window_load(p, s_re, s_im, nt1, ch, lane);

    if (a.apply_cfe)
        msk_freq_offset_slot(p, ch, true, p.cfe_est_out[ch], tl.mse, dcd, m2, mc, countdown, sig_true, sig_false);

    const int agc_len = p.agc_len, eb_len = p.ebno_len;
    const int ds_len = p.sps + 1, d8_len = d8_k + 1;
    int agc_pos = (int)(a.sample0 % agc_len), eb_pos = (int)(a.sample0 % eb_len);
    int fir_pos = (int)(a.sample0 % nt1), ds_pos = (int)(a.sample0 % ds_len), d8_pos = (int)(a.sample0 % d8_len);
    int bb_pos = a.bb_pos, coarse_counter = a.coarse_counter;
    const bool ebno_on = p.report_ebno != 0;
    const int16_t *row = pcm + (size_t)ch * stride;
    const int ntaps = p.ntaps;
    const MeanDiv eb_mean(eb_len), marg_mean(p.marg_len), mse_mean(p.mse_len);

    for (int i = a.i0; i < a.i1; i++) {
        const double dval = ((double)row[i]) / 32768.0;                                  // :322
        if (!(i == a.i0 && a.skip_a_first)) {                                            // :350-367
            if (coarse_counter >= p.Fs || !p.cpu_reduce) {
                const int t = osc_index(mc.ptr);
                p.bb[(size_t)ch * p.bb_len + bb_pos] = make_double2(p.cos_t[t] * dval, p.sin_t[t] * dval);
                bb_pos++; if (bb_pos >= p.bb_len) bb_pos = 0;
            }
        }
        if (i == a.i1 - 1 && a.stop_after_a) break;
        coarse_counter++;                                                                // :368

        const int t2 = osc_index(m2.ptr);
        fir_push(s_re, s_im, nt1, lane, fir_pos, p.cos_t[t2] * dval, p.sin_t[t2] * dval);   // :369
        double sre = 0, sim = 0;
        {
            int tp = fir_pos;
#pragma unroll 8
            for (int k = 0; k < ntaps; k++) {
                sre += p.taps[k] * s_re[tp * MSK_THREADS + lane];
                sim += p.taps[k] * s_im[tp * MSK_THREADS + lane];
                tp++; if (tp >= nt1) tp = 0;
            }
        }
        const double dabval = sqrt(sre * sre + sim * sim);                                // :372
        if (ebno_on) {                                                                    // MSKEbNoMeasure::Update (DSP.cpp:493-505)
            const size_t e = (size_t)eb_pos * p.cpad + ch;
            const double sq = dabval * dabval;
            ma_push(eb_sum2, p.ebno_e2[e], sq);
            ma_push(eb_sum1, p.ebno_e1[e], dabval);
            msk_ebno_readout(eb_mean, eb_ebno, eb_sum1, eb_sum2);
        }
        eb_pos++; if (eb_pos >= eb_len) eb_pos = 0;
        {   // AGC::Update (DSP.cpp:370-379)
            ma_push(agc_sum, p.agc_ring[(size_t)agc_pos * p.cpad + ch], dabval);
            agc_pos++; if (agc_pos >= agc_len) agc_pos = 0;
            agc_val = 1.414213562 / fmax(agc_sum / ((double)agc_len), 0.000001);
            agc_val = fmax(agc_val, 0.000001);
        }
        double2 sig2 = make_double2(sre * agc_val, sim * agc_val);                        // :378
        const double abval = sqrt(sig2.x * sig2.x + sig2.y * sig2.y);                     // :381
        if (abval > 2.84) { const double g = (2.84 / abval); sig2 = make_double2(g * sig2.x, g * sig2.y); }

        // delayedsmpl.update_dont_touch(sig2): one symbol ago (:384, DSP.h:461-466)
        p.dsmpl_ring[(size_t)ds_pos * p.cpad + ch] = sig2;
        ds_pos++; if (ds_pos >= ds_len) ds_pos = 0;
        const double2 pt_d = p.dsmpl_ring[(size_t)ds_pos * p.cpad + ch];
        const double2 pt_msk = make_double2(sig2.x, pt_d.y);                              // :385

        double st_eta = biquad_update(res, hypot(pt_msk.x, pt_msk.y), p.res_a1, p.res_a2, p.res_b0, p.res_b1, p.res_b2);   // :387
        // delayt8.update(st_eta): Delay<double>(SPS/2) (DSP.h:357-374) as a ring with lock-step position
        double d8out;
        {
            p.dly8_ring[(size_t)d8_pos * p.cpad + ch] = st_eta;
            int io = d8_pos - d8_k; if (io < 0) io += d8_len;
            int in_ = io + 1; if (in_ >= d8_len) in_ = 0;
            const double older = p.dly8_ring[(size_t)io * p.cpad + ch];
            const double newer = p.dly8_ring[(size_t)in_ * p.cpad + ch];
            d8out = (d8_w * newer + (1.0 - d8_w) * older);
            d8_pos++; if (d8_pos >= d8_len) d8_pos = 0;
        }
        const int ts = osc_index(st.ptr);
        const double2 st_out = cmul(make_double2(p.cos_t[ts], p.sin_t[ts]), make_double2(st_eta, -d8out));   // :389-390
        const double st_angle_error = atan2_fast(st_out.y, st_out.x);                          // :392
        const double weighting = fabs(tanh(st_angle_error));                              // :395
        if (!dcd) osc_advance_fraction_of_wave(st, -(1.0 - weighting) * st_angle_error * (0.05 / 360.0));    // :397-405
        else osc_advance_fraction_of_wave(st, -(1.0 - weighting) * st_angle_error * (0.003 / 360.0));

        double frac;
        if (osc_have_passed_point(st, p.ee, frac)) {                                      // :408
            const double ct_xt = tanh(sig2.y) * sig2.x;
            const double ct_xt_d = tanh(pt_d.x) * pt_d.y;
            double ct_ec = ct_xt_d - ct_xt;
            if (ct_ec > M_PI) ct_ec = M_PI;
            if (ct_ec < -M_PI) ct_ec = -M_PI;
            if (ct_ec > M_PI_2) ct_ec = M_PI_2;
            if (ct_ec < -M_PI_2) ct_ec = -M_PI_2;
            double carrier_aggression = 12.0 * p.correctionfactor;                        // :422-426
            if (dcd) carrier_aggression = 8.0 * p.correctionfactor;
            osc_increase_phase_deg(m2, carrier_aggression * 1.0 * ct_ec);
            osc_set_freq(m2, (carrier_aggression * 0.01 * ct_ec) + m2.freq, p.Fs);
            msk_symbol_tail(p, ch, true, tl, marg_mean, mse_mean, pt_msk, ct_ec);        // :429-476
        }
        osc_next_frame(m2); osc_next_frame(mc); osc_next_frame(st);                       // :480-483
    }

    const size_t cpad = p.cpad;
    store_osc(p, D_M2_PTR, ch, m2); store_osc(p, D_MC_PTR, ch, mc); store_osc(p, D_ST_PTR, ch, st);
    LD(D_AGC_SUM) = agc_sum; LD(D_AGC_VAL) = agc_val;
    LD(D_EB_SUM1) = eb_sum1; LD(D_EB_SUM2) = eb_sum2; LD(D_EB_EBNO) = eb_ebno;
    store_biquad(p, D_RES_X1, ch, res);
    store_msk_tail(p, ch, tl);
    LI(I_COUNTDOWN) = countdown;
    LI(I_SIG_TRUE) = sig_true; LI(I_SIG_FALSE) = sig_false;
    fir_window_store(p, s_re, s_im, nt1, ch, lane, 0, 1);
}

int msk_segment_launch(const DemodParams &p, const SegmentArgs &a, const int16_t *d_pcm, size_t stride, cudaStream_t s)
{
    const int grid = (p.n_channels + MSK_THREADS - 1) / MSK_THREADS;
    const size_t smem = (size_t)2 * (p.ntaps + 1) * MSK_THREADS * sizeof(double);
    JB_CUDA(cudaFuncSetAttribute(msk_segment_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    int d8_k; double d8_w;
    msk_half_symbol_delay(p.sps, d8_k, d8_w);
    msk_segment_kernel<<<grid, MSK_THREADS, smem, s>>>(p, a, d_pcm, stride, d8_k, d8_w);
    JB_CUDA(cudaGetLastError());
    return 0;
}

} // namespace jb
