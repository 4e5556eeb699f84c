// K1b — warp-specialised continuous MSK demodulator segment kernel (600 / 1200 bps).
//
// Replaces MskDemodulator::writeData (JAERO/mskdemodulator.cpp:313-488) and MskDemodulator::FreqOffsetEstimateSlot
// (:490-519), in the reference's operation order; the moving-average means divide by div_exact (the IEEE quotient in three
// dependent instructions). Same decomposition as the 10500 bps OQPSK pipeline (oqpsk_pipe.cu): the matched
// filter output of sample n excludes sample n (DSP.cpp:292-304), so FIR -> EbNo -> AGC -> clip -> one-symbol delay ->
// |pt_msk| -> resonator -> T/2 delay is feed-forward from the mixed samples up to n-1, and the symbol-rate tail after the
// carrier update feeds nothing back inside a call. Five warps per 32 channels (lane = channel in every warp):
//
//   warp F  2*SPS-tap half-sine matched filter of the mixed samples                                       -> sig2raw
//   warp E  EbNo + AGC running sums (TMA-staged ring tiles), AGC gain, clip, delayedsmpl, resonator, T/2   -> sig2, pt_d, st_eta, d8out
//   warp T  input (PCM tiles, coarse-estimator ring write), timing PLL (arg, tanh weighting, NCO nudge)    -> dval, strobe
//   warp K  carrier error, carrier NCO; mixes the next input sample into the FIR ring                      -> cval, (pt_msk, ct_ec)
//   warp S  marg MA(SPS), dt delay, bias rotate, MSE MA(600), differential soft decode, soft bits
#include "demod_stages.cuh"

namespace jb {

// Warp E's staging of the three sample-rate rings (AGC, EbNo E and E2) through shared memory by the bulk-copy (TMA) engine.
// Ring layout of the pipelined kernels: [cta][slot][32 lanes], so the 32 slots x 32 channels of a tile are one contiguous
// 8 KB block and move with ONE bulk copy per ring, issued by lane 0. (With a [slot][cpad] layout every lane issued its own
// 256-byte row copy; UBLKCP is a warp-uniform instruction, so those 96 stores + 96 loads per tile boundary were issued one
// after the other: a 12 000-cycle stall every 32 samples.) The ring lengths are multiples of the tile length (host-checked).
// Tiles are updated in place and stored back; the next tile is in flight while the current one is consumed.
struct RingTiles {
    double *agc, *e1, *e2;                // [RING_NBUF][OQ_T][32] each
    unsigned long long *bars;             // [RING_NBUF] tile-full mbarriers
    unsigned phases;                      // expected parity per barrier
    long long rt;                         // current tile
    bool next_issued, dirty;              // the next tile was requested; the current one was written
};
__device__ __forceinline__ double *ring_tile_gmem(double *ring, int len, long long tile)
{ return ring + ((size_t)blockIdx.x * len + (size_t)((tile * OQ_T) % len)) * 32; }
__device__ __forceinline__ void ring_tile_load(const DemodParams &p, RingTiles &r, long long tile, int lane)
{
    const bool ebno_on = p.report_ebno != 0;
    const int b = (int)(tile % RING_NBUF);
    fence_proxy_async();                  // every lane: its generic accesses to the buffer precede the copy
    __syncwarp();
    if (lane == 0) {
        mbar_expect_tx(&r.bars[b], (ebno_on ? 3u : 1u) * OQ_SM_RING);
        bulk_g2s(r.agc + b * OQ_T * 32, ring_tile_gmem(p.agc_ring, p.agc_len, tile), OQ_SM_RING, &r.bars[b]);
        if (ebno_on) {
            bulk_g2s(r.e1 + b * OQ_T * 32, ring_tile_gmem(p.ebno_e1, p.ebno_len, tile), OQ_SM_RING, &r.bars[b]);
            bulk_g2s(r.e2 + b * OQ_T * 32, ring_tile_gmem(p.ebno_e2, p.ebno_len, tile), OQ_SM_RING, &r.bars[b]);
        }
    }
}
__device__ __forceinline__ void ring_tile_store(const DemodParams &p, RingTiles &r, long long tile, int lane)
{
    const bool ebno_on = p.report_ebno != 0;
    const int b = (int)(tile % RING_NBUF);
    fence_proxy_async();
    __syncwarp();
    if (lane == 0) {
        bulk_s2g(ring_tile_gmem(p.agc_ring, p.agc_len, tile), r.agc + b * OQ_T * 32, OQ_SM_RING);
        if (ebno_on) {
            bulk_s2g(ring_tile_gmem(p.ebno_e1, p.ebno_len, tile), r.e1 + b * OQ_T * 32, OQ_SM_RING);
            bulk_s2g(ring_tile_gmem(p.ebno_e2, p.ebno_len, tile), r.e2 + b * OQ_T * 32, OQ_SM_RING);
        }
        bulk_commit();
    }
}
__device__ __forceinline__ void ring_tile_wait(RingTiles &r, long long tile)
{ const int b = (int)(tile % RING_NBUF); mbar_wait(&r.bars[b], (r.phases >> b) & 1u); r.phases ^= (1u << b); }
// request the tile of sample S (and the next one if the launch reaches it) and wait for the first
__device__ __forceinline__ void ring_tiles_open(const DemodParams &p, RingTiles &r, long long S, long long S_end, int lane)
{
    r.phases = 0u;
    r.rt = S / OQ_T;
    r.next_issued = false; r.dirty = false;
    ring_tile_load(p, r, r.rt, lane);
    if ((r.rt + 1) * OQ_T < S_end) { ring_tile_load(p, r, r.rt + 1, lane); r.next_issued = true; }
    ring_tile_wait(r, r.rt);
}
// sample S's slot in the staged tiles (index into agc / e1 / e2)
__device__ __forceinline__ int ring_tile_slot(const RingTiles &r, long long S, int lane)
{ return (((int)(r.rt % RING_NBUF)) * OQ_T + (int)(S & (OQ_T - 1))) * 32 + lane; }
// after sample S-1: at a tile boundary store the finished tile, wait for the next, request the one after (warp-uniform)
__device__ __forceinline__ void ring_tiles_next(const DemodParams &p, RingTiles &r, long long S, long long S_end, int lane)
{
    if ((S & (OQ_T - 1)) == 0) {
        ring_tile_store(p, r, r.rt, lane);    // the finished tile goes back to HBM
        r.dirty = false;
        r.rt++;
        if (S < S_end) {
            ring_tile_wait(r, r.rt);              // next tile (requested a tile ago)
            r.next_issued = false;
            if ((r.rt + 1) * OQ_T < S_end) {
                // the buffer being refilled was stored a whole tile ago: only the store committed just now may still be
                // reading shared memory
                bulk_wait_read_1();
                ring_tile_load(p, r, r.rt + 1, lane); r.next_issued = true;
            }
        }
    }
}
__device__ __forceinline__ void ring_tiles_close(const DemodParams &p, RingTiles &r, int lane)
{
    if (r.dirty) ring_tile_store(p, r, r.rt, lane);
    if (r.next_issued) ring_tile_wait(r, r.rt + 1);
    bulk_wait_all();
}

static const int MP_THREADS = 160;
static const int MP_HF = 16;                        // doubles per lane in a hand-off slot
// named barriers (0 is __syncthreads)
enum { MB_X = 1, MB_YT = 3, MB_Z = 5, MB_W = 7, MB_V = 9, MB_YK = 11, MB_U = 13 };

// sum_{k<cnt} taps[k0+k] * ring[(start+k) % nt1] for both components, in tap order (DSP.cpp:296-303), as two
// contiguous runs of the ring
__device__ __forceinline__ void mp_fir_run(const DemodParams &p, const double *__restrict__ s_re, const double *__restrict__ s_im, int lane, int nt1, int start, int cnt,
                                           double &sre, double &sim)
{
    int k = 0, tp = start;
    const int first = min(cnt, nt1 - start);
#pragma unroll 8
    for (; k < first; k++, tp++) { sre += p.taps[k] * s_re[tp * 32 + lane]; sim += p.taps[k] * s_im[tp * 32 + lane]; }
    tp = 0;
#pragma unroll 8
    for (; k < cnt; k++, tp++) { sre += p.taps[k] * s_re[tp * 32 + lane]; sim += p.taps[k] * s_im[tp * 32 + lane]; }
}

// ptxas's register allocation for this kernel swings between 72 registers with spills and 96 on small source changes; the
// cap keeps the 92 it has without spills (launched with MP_THREADS threads)
__global__ void __maxnreg__(92)
msk_pipe_kernel(const __grid_constant__ DemodParams p, const SegmentArgs a, const int16_t *__restrict__ pcm, size_t stride, int d8_k, double d8_w)
{
    extern __shared__ __align__(128) unsigned char mp_smem_raw[];
    const int ntaps = p.ntaps, nt1 = ntaps + 1;
    const int ds_len = p.sps + 1, d8_len = d8_k + 1;
    // shared memory map
    double *s_re = reinterpret_cast<double *>(mp_smem_raw);                        // [nt1][32]
    double *s_im = s_re + (size_t)nt1 * 32;
    double *t_agc = s_im + (size_t)nt1 * 32;                                       // [RING_NBUF][T][32]
    double *t_e1 = t_agc + RING_NBUF * OQ_T * 32;
    double *t_e2 = t_e1 + RING_NBUF * OQ_T * 32;
    double2 *s_ds = reinterpret_cast<double2 *>(t_e2 + RING_NBUF * OQ_T * 32);     // delayedsmpl [ds_len][32]
    double *s_d8 = reinterpret_cast<double *>(s_ds + (size_t)ds_len * 32);         // delayt8 [d8_len][32]
    double *hand = s_d8 + (size_t)d8_len * 32;                                     // [2][MP_HF][32]
    unsigned long long *bars = reinterpret_cast<unsigned long long *>(hand + 2 * MP_HF * 32);   // ring tiles [RING_NBUF]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ch = blockIdx.x * 32 + lane;
    const bool live = ch < p.n_channels;
    const size_t cpad = p.cpad;
    if (threadIdx.x == 0) { for (int k = 0; k < RING_NBUF; k++) mbar_init(&bars[k], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();                                           // (0) mbarriers usable

    const int nB = (a.i1 - a.i0) - (a.stop_after_a ? 1 : 0);             // samples whose loop body runs in this launch
    const long long S0 = a.sample0;
    const double Fs = p.Fs;
    const double *__restrict__ cos_t = p.cos_t, *__restrict__ sin_t = p.sin_t;
    // hand-off slot: f 0,1 sig2raw (F->E) | 2..5 sig2, pt_d (E->K) | 6,7 st_eta, d8out (E->T) | 8,9 strobe, next input (T->K)
    //                | 10..13 flag, pt_msk.x, pt_msk.y, ct_ec (K->S) | 14 (slot 0) first input sample (T->K)
#define HAND(s, f) hand[((s) * MP_HF + (f)) * 32 + lane]

    // ======================================================================================= warp K: carrier loop
    if (warp == 3) {
        Osc m2 = load_osc(p, D_M2_PTR, ch);
        int dcd = LI(I_DCD);
        if (a.apply_cfe) {
            Osc mc = load_osc(p, D_MC_PTR, ch);
            int countdown = LI(I_COUNTDOWN);
            if (msk_freq_offset_slot(p, ch, live, p.cfe_est_out[ch], LD(D_MSE), dcd, m2, mc, countdown, LI(I_SIG_TRUE), LI(I_SIG_FALSE))) {
                LD(D_MC_STEP) = mc.step; LD(D_MC_FREQ) = mc.freq;     // warp T reloads mixer_center after the barrier
            }
            LI(I_COUNTDOWN) = countdown;
        }
        __syncthreads();                                       // (1) slot done, FIR ring resident
        if (nB > 0) {
            double c2_re, c2_im;
            { const int t = osc_index(m2.ptr); c2_re = cos_t[t]; c2_im = sin_t[t]; }
            int fir_pos = (int)(S0 % nt1);                     // slot of the sample being mixed
            {   // cval of the first sample (:369)
                const double dval = HAND(0, 14);
                fir_push(s_re, s_im, nt1, lane, fir_pos, c2_re * dval, c2_im * dval);
                handoff(MB_X + 0);                             // X_0
            }
            const double aggr = (dcd ? 8.0 : 12.0) * p.correctionfactor;      // :422-426
            for (int j = 0; j < nB; j++) {
                const int sl = j & 1;
                const int m2_spec = osc_next_index(m2);
                const double n2_re = cos_t[m2_spec], n2_im = sin_t[m2_spec];
                nb_sync(MB_YK + sl);                           // sig2, pt_d of this sample (warp E)
                const double2 sig2 = make_double2(HAND(sl, 2), HAND(sl, 3)), pt_d = make_double2(HAND(sl, 4), HAND(sl, 5));
                nb_sync(MB_U + sl);                            // strobe decision (warp T)
                const double strobe = HAND(sl, 8), dnext = HAND(sl, 9);
                double sy_flag = 0.0, sy_ec = 0.0;
                if (strobe != 0.0) {                                              // :408
                    double ct_ec = ct_error(sig2, pt_d);
                    if (ct_ec > M_PI_2) ct_ec = M_PI_2;
                    if (ct_ec < -M_PI_2) ct_ec = -M_PI_2;
                    osc_increase_phase_deg(m2, aggr * 1.0 * ct_ec);
                    osc_set_freq(m2, (aggr * 0.01 * ct_ec) + m2.freq, Fs);
                    sy_flag = 1.0; sy_ec = ct_ec;
                }
                osc_next_frame(m2);                                               // :480
                {
                    const int t = osc_index(m2.ptr);
                    if (t == m2_spec) { c2_re = n2_re; c2_im = n2_im; } else { c2_re = cos_t[t]; c2_im = sin_t[t]; }
                }
                if (j + 1 < nB) {   // the next sample's mixed value enters the FIR ring (:369-370)
                    fir_push(s_re, s_im, nt1, lane, fir_pos, c2_re * dnext, c2_im * dnext);
                    handoff(MB_X + ((j + 1) & 1));             // X_{j+1}
                }
                if (j >= 2) nb_sync(MB_V + sl);                // V_{j-2}: S has read slot sl
                HAND(sl, 10) = sy_flag; HAND(sl, 11) = sig2.x; HAND(sl, 12) = pt_d.y; HAND(sl, 13) = sy_ec;   // pt_msk=(sig2.re, pt_d.im) :385
                handoff(MB_W + sl);                            // W_j
            }
            if (nB >= 2) nb_sync(MB_V + (nB & 1));             // V_{nB-2}
            nb_sync(MB_V + ((nB - 1) & 1));                    // V_{nB-1}
        }
        store_osc(p, D_M2_PTR, ch, m2);
    }
    // ======================================================================================= warp S: symbol-rate tail
    else if (warp == 4) {
        MskTail tl = load_msk_tail(p, ch);
        const MeanDivExact marg_mean(p.marg_len), mse_mean(p.mse_len);
        __syncthreads();                                       // (1)
        for (int j = 0; j < nB; j++) {
            const int sl = j & 1;
            nb_sync(MB_W + sl);                                // W_j
            const double fl = HAND(sl, 10), fx = HAND(sl, 11), fy = HAND(sl, 12), fec = HAND(sl, 13);
            handoff(MB_V + sl);                                // V_j: slot read
            if (fl != 0.0) msk_symbol_tail(p, ch, live, tl, marg_mean, mse_mean, make_double2(fx, fy), fec);   // :429-476
        }
        store_msk_tail(p, ch, tl);
    }
    // ======================================================================================= warp T: input + symbol-timing PLL
    else if (warp == 2) {
        Osc st = load_osc(p, D_ST_PTR, ch);
        PcmReader in(pcm + (size_t)ch * stride, stride, live, a.i0);
        double dcur = in.dval(a.i0);
        HAND(0, 14) = dcur;
        __syncthreads();                                       // (1) the slot may have re-centred mixer_center or (wired) cleared DCD
        const int dcd = LI(I_DCD);
        Osc mc = load_osc(p, D_MC_PTR, ch);
        int bb_pos = a.bb_pos, coarse_counter = a.coarse_counter;
        double2 *bb_row = p.bb + (size_t)ch * p.bb_len;
        const int bbn = p.bb_len;
        const bool cpu_reduce = p.cpu_reduce != 0;
        const double ee = p.ee;
        const double gain = dcd ? (0.003 / 360.0) : (0.05 / 360.0);           // :397-405
        double cs_re, cs_im, cc_re, cc_im;
        { const int t = osc_index(st.ptr); cs_re = cos_t[t]; cs_im = sin_t[t]; }
        { const int t = osc_index(mc.ptr); cc_re = cos_t[t]; cc_im = sin_t[t]; }
        for (int i = a.i0; i < a.i1; i++) {
            const int j = i - a.i0, sl = j & 1;
            if (!(i == a.i0 && a.skip_a_first)) {                                            // :350-367
                if (coarse_counter >= Fs || !cpu_reduce) {
                    if (live) bb_row[bb_pos] = make_double2(cc_re * dcur, cc_im * dcur);
                    bb_pos++; if (bb_pos >= bbn) bb_pos = 0;
                }
            }
            if (i == a.i1 - 1 && a.stop_after_a) break;
            coarse_counter++;                                                                // :368
            osc_next_frame(mc);                                                              // :481
            { const int t = osc_index(mc.ptr); cc_re = cos_t[t]; cc_im = sin_t[t]; }
            const double dnxt = (i + 1 < a.i1) ? in.dval(i + 1) : 0.0;
            nb_sync(MB_YT + sl);                               // st_eta, d8out of this sample (warp E)
            const double st_eta = HAND(sl, 6), d8out = HAND(sl, 7);
            const double2 st_out = c_mul(make_double2(cs_re, cs_im), make_double2(st_eta, -d8out));   // :389-390
            const double st_angle_error = atan2_fast(st_out.y, st_out.x);                          // :392
            const double weighting = fabs(tanh(st_angle_error));                              // :395
            osc_advance_fraction_of_wave(st, -(1.0 - weighting) * st_angle_error * gain);
            double frac = 0.0;
            const bool strobe = osc_have_passed_point(st, ee, frac);                          // :408
            HAND(sl, 8) = strobe ? 1.0 : 0.0; HAND(sl, 9) = dnxt;
            handoff(MB_U + sl);
            osc_next_frame(st);                                                               // :483
            { const int t = osc_index(st.ptr); cs_re = cos_t[t]; cs_im = sin_t[t]; }
            dcur = dnxt;
        }
        store_osc(p, D_ST_PTR, ch, st);
        store_osc(p, D_MC_PTR, ch, mc);
    }
    // ======================================================================================= warp E: envelope chain
    else if (warp == 1) {
        double agc_sum = LD(D_AGC_SUM), agc_val = LD(D_AGC_VAL);
        double eb_sum1 = LD(D_EB_SUM1), eb_sum2 = LD(D_EB_SUM2), eb_ebno = LD(D_EB_EBNO);
        Biquad res = load_biquad(p, D_RES_X1, ch);
        const bool ebno_on = p.report_ebno != 0;
        const double r_agc = 1.0 / ((double)p.agc_len);
        const MeanDivExact eb_mean(p.ebno_len);
        const double res_a1 = p.res_a1, res_a2 = p.res_a2, res_b0 = p.res_b0, res_b1 = p.res_b1, res_b2 = p.res_b2;
        long long S = S0;
        int ds_pos = (int)(S % ds_len), d8_pos = (int)(S % d8_len);
        const long long S_end = S + nB;
        const int eb_from_j = (a.i1 - a.i0) - OQ_EBNO_TAIL;
        for (int k = 0; k < ds_len; k++) s_ds[k * 32 + lane] = p.dsmpl_ring[(size_t)k * cpad + ch];
        for (int k = 0; k < d8_len; k++) s_d8[k * 32 + lane] = p.dly8_ring[(size_t)k * cpad + ch];
        __syncthreads();                                       // (1)
        if (nB > 0) {
            RingTiles rg = {t_agc, t_e1, t_e2, bars};
            ring_tiles_open(p, rg, S, S_end, lane);
            for (int j = 0; j < nB; j++) {
                const int sl = j & 1;
                const int rslot = ring_tile_slot(rg, S, lane);
                nb_sync(MB_Z + sl);                            // Z_j: matched filter output of this sample
                const double sre = HAND(sl, 0), sim = HAND(sl, 1);
                const double dabval = sqrt(sre * sre + sim * sim);                                // :372
                if (ebno_on) {                                                                    // MSKEbNoMeasure::Update (DSP.cpp:493-505)
                    const double sq = dabval * dabval;
                    ma_push(eb_sum2, t_e2[rslot], sq);
                    ma_push(eb_sum1, t_e1[rslot], dabval);
                    if (j >= eb_from_j) msk_ebno_readout(eb_mean, eb_ebno, eb_sum1, eb_sum2);   // over the launch's tail only
                }
                {   // AGC::Update (DSP.cpp:370-379)
                    ma_push(agc_sum, t_agc[rslot], dabval);
                    rg.dirty = true;
                    agc_val = 1.414213562 / fmax(div_exact(agc_sum, (double)p.agc_len, r_agc), 0.000001);
                    agc_val = fmax(agc_val, 0.000001);
                }
                double2 sig2 = make_double2(sre * agc_val, sim * agc_val);                        // :378
                const double abval = sqrt(sig2.x * sig2.x + sig2.y * sig2.y);                     // :381
                if (abval > 2.84) { const double g = (2.84 / abval); sig2 = make_double2(g * sig2.x, g * sig2.y); }
                // delayedsmpl.update_dont_touch(sig2): one symbol ago (:384, DSP.h:461-466)
                s_ds[ds_pos * 32 + lane] = sig2;
                ds_pos++; if (ds_pos >= ds_len) ds_pos = 0;
                const double2 pt_d = s_ds[ds_pos * 32 + lane];
                const double2 pt_msk = make_double2(sig2.x, pt_d.y);                              // :385
                const double st_eta = biquad_update(res, hypot(pt_msk.x, pt_msk.y), res_a1, res_a2, res_b0, res_b1, res_b2);   // :387
                double d8out;                                                                     // delayt8.update(st_eta): Delay<double>(SPS/2)
                {
                    s_d8[d8_pos * 32 + lane] = st_eta;
                    int io = d8_pos - d8_k; if (io < 0) io += d8_len;
                    int in_ = io + 1; if (in_ >= d8_len) in_ = 0;
                    const double older = s_d8[io * 32 + lane], newer = s_d8[in_ * 32 + lane];
                    d8out = (d8_w * newer + (1.0 - d8_w) * older);
                    d8_pos++; if (d8_pos >= d8_len) d8_pos = 0;
                }
                HAND(sl, 2) = sig2.x; HAND(sl, 3) = sig2.y; HAND(sl, 4) = pt_d.x; HAND(sl, 5) = pt_d.y; HAND(sl, 6) = st_eta; HAND(sl, 7) = d8out;
                handoff(MB_YT + sl);                           // timing inputs -> warp T
                nb_arrive(MB_YK + sl);                         // sig2, pt_d -> warp K
                S++;
                ring_tiles_next(p, rg, S, S_end, lane);
            }
            ring_tiles_close(p, rg, lane);
        }
        for (int k = 0; k < ds_len; k++) p.dsmpl_ring[(size_t)k * cpad + ch] = s_ds[k * 32 + lane];
        for (int k = 0; k < d8_len; k++) p.dly8_ring[(size_t)k * cpad + ch] = s_d8[k * 32 + lane];
        LD(D_AGC_SUM) = agc_sum; LD(D_AGC_VAL) = agc_val;
        LD(D_EB_SUM1) = eb_sum1; LD(D_EB_SUM2) = eb_sum2; LD(D_EB_EBNO) = eb_ebno;
        store_biquad(p, D_RES_X1, ch, res);
    }
    // ======================================================================================= warp F: matched filter
    else {
        fir_window_load(p, s_re, s_im, nt1, ch, lane);
        __syncthreads();                                       // (1)
        // output j (:370) = sum over the ntaps mixed samples older than sample i0+j; the newest of them (slot `tail`) is produced
        // by warp K one sample earlier, the ntaps-1 older terms are summed ahead of that (same order as DSP.cpp:296-303)
        int tail = (int)((S0 + nt1 - 1) % nt1);
        double nfre = 0, nfim = 0;
        auto older = [&]() { nfre = 0; nfim = 0; int st0 = tail + 2; if (st0 >= nt1) st0 -= nt1; mp_fir_run(p, s_re, s_im, lane, nt1, st0, ntaps - 1, nfre, nfim); };
        if (nB > 0) older();
        for (int j = 0; j < nB; j++) {
            if (j > 0) nb_sync(MB_X + ((j - 1) & 1));         // X_{j-1}
            nfre += p.taps[ntaps - 1] * s_re[tail * 32 + lane]; nfim += p.taps[ntaps - 1] * s_im[tail * 32 + lane];
            const int sl = j & 1;
            HAND(sl, 0) = nfre; HAND(sl, 1) = nfim;
            handoff(MB_Z + sl);                                // Z_j
            tail++; if (tail >= nt1) tail = 0;
            if (j + 1 < nB) older();
        }
        if (nB > 0) nb_sync(MB_X + ((nB - 1) & 1));           // X_{nB-1}: pair the last arrival of warp K
    }
    __syncthreads();                                           // (2) every warp is done with the FIR ring
    fir_window_store(p, s_re, s_im, nt1, ch, lane, warp, 5);
#undef HAND
}

int msk_pipe_launch(const DemodParams &p, const SegmentArgs &a, const int16_t *d_pcm, size_t stride, cudaStream_t s)
{
    const int grid = (p.n_channels + 31) / 32;
    int d8_k; double w;
    msk_half_symbol_delay(p.sps, d8_k, w);
    const size_t smem = (size_t)2 * (p.ntaps + 1) * 32 * 8 + 3 * RING_NBUF * OQ_SM_RING + (size_t)(p.sps + 1) * 32 * 16 + (size_t)(d8_k + 1) * 32 * 8 +
                        (size_t)2 * MP_HF * 32 * 8 + 64;
    JB_CUDA(cudaFuncSetAttribute(msk_pipe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    msk_pipe_kernel<<<grid, MP_THREADS, smem, s>>>(p, a, d_pcm, stride, d8_k, w);
    JB_CUDA(cudaGetLastError());
    return 0;
}

} // namespace jb
