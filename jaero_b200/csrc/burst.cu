// K3 / K4 — burst MSK demodulator (600 / 1200 bps R/T-channel bursts), batched over channels.
//
// Replaces BurstMskDemodulator::writeData (JAERO/burstmskdemodulator.cpp:371-754) and the primitives only it uses
// (QJHilbertFilter DSP.cpp:754-794 over JFastFir, TMovingAverage DSP.h:145-199, PeakDetector DSP.h:491-576,
// FFTrWrapper fftrwrapper.cpp:19-27). One internal chunk (<= BURST_CHUNK samples) runs as
//   hilbert_exchange thread/channel: the sample exchange of the streaming FFT convolution (fastfir.cuh, nfft 8192) with the
//                    2048-tap Hilbert kernel, PCM in -> analytic signal out; its block kernel is the shared one of fastfir.cu
//   burst_front      thread/channel, always active: AGC(1 s), alignment delays d1/d2, burst-timing statistic
//                    (delay-conjugate-multiply -> MA -> MA -> minus delayed copy -> square), PeakDetector, trident-buffer
//                    fills; every completed fill is recorded as an event (sample index + buffer slot)
//   burst_trident    per event: two zero-padded 32768-point FFTs (Stockham radix-8, ping-pong in HBM), strongest base
//                    bin, the two side peaks of the 0101 section, carrier phase  (:443-520)
//   burst_back       thread/channel: applies each event at its sample (accept test, NCO/gain/loop reset, -1 marker),
//                    then the gated demodulator tail: mix, matched filter, preamble symbol-tone PLL, rotator carrier
//                    loop, EbNo, AGC2, MSK timing, strobes, differential soft bits (:570-749)
// Sample-rate rings of the always-active front end advance in lock-step ([slot][channel], coalesced); the tail's rings
// advance only while a channel is inside a burst, so they carry per-channel positions.
#include "demod_stages.cuh"
#include "burst.cuh"

namespace jb {

#define BD(idx) p.BD[(size_t)(idx) * p.cpad + ch]
#define BI(idx) p.BI[(size_t)(idx) * p.cpad + ch]

// ------------------------------------------------------------------------------------------------ FFT helpers
// Stockham radix-8 pass src -> dst over an n-point sequence (n a multiple of 8), any number of threads: the trident FFTs'
// ping-pong through HBM (the butterfly is dft8 of fft_device.cuh)
template <bool INV> __device__ __forceinline__ void pass8(const double2 *src, double2 *dst, int n, int Ns, const double2 *__restrict__ tw, int tw_stride)
{
    const int nb = n >> 3;
    const int wmul = tw_stride * (n / (Ns * 8));
    for (int j = threadIdx.x; j < nb; j += blockDim.x) {
        double2 v[8];
#pragma unroll
        for (int t = 0; t < 8; t++) v[t] = src[j + t * nb];
        const int k = j % Ns;
#pragma unroll
        for (int t = 1; t < 8; t++) {
            double2 w = tw[t * k * wmul];
            if (INV) w.y = -w.y;
            v[t] = c_mul(v[t], w);
        }
        dft8<INV>(v);
        const int ob = (j / Ns) * Ns * 8 + k;
#pragma unroll
        for (int t = 0; t < 8; t++) dst[ob + t * Ns] = v[t];
    }
}

// ------------------------------------------------------------------------------------------------ Hilbert (FFT-8192 FIR)
// JFastFir::update sample exchange: out[i] = previous block's result, staging block <- real PCM sample
__global__ void hilbert_exchange_kernel(FastFir h, BurstParams p, const int16_t *__restrict__ pcm, size_t stride, int pcm0, int i0, int i1, int fill0)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= p.n_channels) return;
    const int16_t *row = pcm + (size_t)ch * stride + pcm0;
    double2 *inb = h.inblk + (size_t)ch * h.L;
    const double2 *outb = h.outblk + (size_t)ch * h.L;
    double2 *a = p.analytic + (size_t)ch * p.astride;
    int fill = fill0;
    for (int i = i0; i < i1; i++) {
        a[i] = outb[fill];
        inb[fill] = make_double2(((double)row[i]) / 32768.0, 0.0);        // burstmskdemodulator.cpp:380-384
        fill++;
    }
}
// ------------------------------------------------------------------------------------------------ front end
// Everything in front of the trident test is feed-forward (AGC -> alignment delays -> burst-timing statistic -> peak
// detector), but every stage is a running sum or a delay line over a long ring in HBM: ten "value written len samples ago"
// reads per sample. All ring positions advance in lock-step, so the reads of the NEXT block of 8 samples are issued with
// cp.async (global -> shared, 8 / 16 bytes per thread, a warp's 32 channels are one contiguous row segment) while the
// current block is computed from shared memory; the per-sample loop itself never waits on HBM. Writes go straight to the rings.
static const int BF_T = 64, BF_B = 8;            // threads per CTA, samples per staged block
static const int BF_N2 = 4, BF_N1 = 7;           // staged double2 / double fields per sample
static const int BF_SMEM = 2 * BF_B * (BF_N2 * 16 + BF_N1 * 8) * BF_T;

__device__ __forceinline__ void cp_async8(void *dst, const void *src)
{ asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_async16(void *dst, const void *src)
{ asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory"); }

__global__ void __launch_bounds__(BF_T)
burst_front_kernel(BurstParams p, long long sample0, int n)
{
    extern __shared__ __align__(16) unsigned char bf_smem[];
    double2 *st2 = reinterpret_cast<double2 *>(bf_smem);                                  // [2][B][N2][T]
    double *st1 = reinterpret_cast<double *>(bf_smem + 2 * BF_B * BF_N2 * 16 * BF_T);     // [2][B][N1][T]
    const int tid = threadIdx.x;
    const int ch_raw = blockIdx.x * blockDim.x + tid;
    const bool live = ch_raw < p.n_channels;
    const int ch = live ? ch_raw : p.n_channels - 1;         // dead threads shadow the last channel (loads only; they store nothing)
    const size_t cp = p.cpad;
    double agc_sum = BD(BD_AGC_SUM), agc_val = BD(BD_AGC_VAL);
    double2 btma_sum = make_double2(BD(BD_BTMA_SUM_RE), BD(BD_BTMA_SUM_IM));
    double mav1_sum = BD(BD_MAV1_SUM), pd_lastdy = BD(BD_PD_LASTDY), pd_maxval = BD(BD_PD_MAXVAL);
    int pd_cntdown = BI(BI_PD_CNTDOWN), pd_maxposcnt = BI(BI_PD_MAXPOSCNT);
    int tri_ptr = BI(BI_TRI_PTR), tri_slot = BI(BI_TRI_SLOT), nev = 0;
    const int pd1_sz = 2 * p.pd_len + 1, pd2_sz = p.pd_len + 1, pd3_sz = 2 * p.pd_len + 1;
    // lock-step ring positions of the sample being computed
    int agc_pos = (int)(sample0 % p.agc_len), d1_pos = (int)(sample0 % p.d1_len), d2_pos = (int)(sample0 % p.d2_len);
    int btd1_pos = (int)(sample0 % p.btd1_len), btma_pos = (int)(sample0 % p.btma_len), mav1_pos = (int)(sample0 % p.mav1_len);
    int btdiff_pos = (int)(sample0 % p.btdiff_len);
    int pd1_pos = (int)(sample0 % pd1_sz), pd2_pos = (int)(sample0 % pd2_sz), pd3_pos = (int)(sample0 % pd3_sz);
    const double2 *an = p.analytic + (size_t)ch * p.astride;
    double *vtd = p.vtd + (size_t)ch * p.astride;
    double *tri = p.tri + (size_t)ch * BURST_MAXEV * p.tri_sz;
    const double r_agc = 1.0 / ((double)p.agc_len), r_btma = 1.0 / ((double)p.btma_len), r_mav1 = 1.0 / ((double)p.mav1_len);
    auto wrap = [](int v, int len) { while (v >= len) v -= len; return v; };
    // a ring shorter than the staging distance (bt_d1 of the burst OQPSK mode: 11 slots) is read at the point of use instead
    const bool btd1_direct = p.btd1_len < 2 * BF_B + 3;
    // stage the ring reads of the next `cnt` samples into buffer b (the staging stream keeps its own ring positions)
    int f_agc = agc_pos, f_d1 = d1_pos, f_d2 = d2_pos, f_btd1 = btd1_pos, f_btma = btma_pos, f_mav1 = mav1_pos, f_btdiff = btdiff_pos;
    int f_pd1 = pd1_pos, f_pd2 = pd2_pos;
    auto stage = [&](int b, int cnt) {
        for (int k = 0; k < cnt; k++) {
            double2 *d2p = st2 + ((size_t)(b * BF_B + k) * BF_N2) * BF_T + tid;
            double *d1p = st1 + ((size_t)(b * BF_B + k) * BF_N1) * BF_T + tid;
            cp_async16(d2p + 0 * BF_T, p.d1_ring + (size_t)wrap(f_d1 + 1, p.d1_len) * cp + ch);
            if (!btd1_direct) {
                cp_async16(d2p + 1 * BF_T, p.btd1_ring + (size_t)wrap(f_btd1 + 1, p.btd1_len) * cp + ch);
                cp_async16(d2p + 2 * BF_T, p.btd1_ring + (size_t)wrap(f_btd1 + 2, p.btd1_len) * cp + ch);
            }
            cp_async16(d2p + 3 * BF_T, p.btma_ring + (size_t)f_btma * cp + ch);
            cp_async8(d1p + 0 * BF_T, p.agc_ring + (size_t)f_agc * cp + ch);
            cp_async8(d1p + 1 * BF_T, p.d2_ring + (size_t)wrap(f_d2 + 1, p.d2_len) * cp + ch);
            cp_async8(d1p + 2 * BF_T, p.mav1_ring + (size_t)f_mav1 * cp + ch);
            cp_async8(d1p + 3 * BF_T, p.btdiff_ring + (size_t)wrap(f_btdiff + 1, p.btdiff_len) * cp + ch);
            cp_async8(d1p + 4 * BF_T, p.btdiff_ring + (size_t)wrap(f_btdiff + 2, p.btdiff_len) * cp + ch);
            cp_async8(d1p + 5 * BF_T, p.pd1_ring + (size_t)wrap(f_pd1 + 1, pd1_sz) * cp + ch);
            cp_async8(d1p + 6 * BF_T, p.pd2_ring + (size_t)wrap(f_pd2 + 1, pd2_sz) * cp + ch);
            f_agc = wrap(f_agc + 1, p.agc_len); f_d1 = wrap(f_d1 + 1, p.d1_len); f_d2 = wrap(f_d2 + 1, p.d2_len);
            f_btd1 = wrap(f_btd1 + 1, p.btd1_len); f_btma = wrap(f_btma + 1, p.btma_len); f_mav1 = wrap(f_mav1 + 1, p.mav1_len);
            f_btdiff = wrap(f_btdiff + 1, p.btdiff_len); f_pd1 = wrap(f_pd1 + 1, pd1_sz); f_pd2 = wrap(f_pd2 + 1, pd2_sz);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    stage(0, min(BF_B, n));
    for (int blk = 0, i0 = 0; i0 < n; blk++, i0 += BF_B) {
        const int b = blk & 1, cnt = min(BF_B, n - i0);
        if (i0 + BF_B < n) { stage(b ^ 1, min(BF_B, n - i0 - BF_B)); asm volatile("cp.async.wait_group 1;" ::: "memory"); }
        else asm volatile("cp.async.wait_group 0;" ::: "memory");
        for (int k = 0; k < cnt; k++) {
            const int i = i0 + k;
            const double2 *s2 = st2 + ((size_t)(b * BF_B + k) * BF_N2) * BF_T + tid;
            const double *s1 = st1 + ((size_t)(b * BF_B + k) * BF_N1) * BF_T + tid;
            double2 cval = an[i];
            {   // agc->Update(std::abs(cval)); cval*=agc->AGCVal  (:412-413)
                const double ab = hypot(cval.x, cval.y);
                agc_sum = agc_sum - s1[0 * BF_T]; agc_sum = agc_sum + fabs(ab);
                if (live) p.agc_ring[(size_t)agc_pos * cp + ch] = fabs(ab);
                agc_pos++; if (agc_pos >= p.agc_len) agc_pos = 0;
                agc_val = 1.414213562 / fmax(div_exact(agc_sum, (double)p.agc_len, r_agc), 0.000001);
                agc_val = fmax(agc_val, 0.000001);
                cval = make_double2(cval.x * agc_val, cval.y * agc_val);
            }
            // d1.update_dont_touch(cval) (:416): the slot read is the one after the slot written
            if (live) p.d1_ring[(size_t)d1_pos * cp + ch] = cval;
            d1_pos++; if (d1_pos >= p.d1_len) d1_pos = 0;
            const double2 cval_d = s2[0 * BF_T];
            {                                                                 // d2.update_dont_touch(real(cval_d)) (:419)
                if (live) p.d2_ring[(size_t)d2_pos * cp + ch] = cval_d.x;
                d2_pos++; if (d2_pos >= p.d2_len) d2_pos = 0;
                if (live) vtd[i] = s1[1 * BF_T];
            }
            // burst timing statistic (:422-427)
            double2 dly;                                                      // bt_d1.update(cval): Delay<cpx>(SPS)
            {
                if (live) p.btd1_ring[(size_t)btd1_pos * cp + ch] = cval;
                double2 older, newer;
                if (btd1_direct) {
                    __syncwarp();                                                 // (dead threads never store; live ones read their own column)
                    older = p.btd1_ring[(size_t)wrap(btd1_pos + 1, p.btd1_len) * cp + ch];
                    newer = p.btd1_ring[(size_t)wrap(btd1_pos + 2, p.btd1_len) * cp + ch];
                } else { older = s2[1 * BF_T]; newer = s2[2 * BF_T]; }
                const double w = p.btd1_wv[btd1_pos];
                dly = make_double2(w * newer.x + (1.0 - w) * older.x, w * newer.y + (1.0 - w) * older.y);
                btd1_pos++; if (btd1_pos >= p.btd1_len) btd1_pos = 0;
            }
            const double2 prod = c_mul(cval, make_double2(dly.x, -dly.y));     // cval*std::conj(...)
            double2 mav;                                                       // bt_ma1.UpdateSigned (TMovingAverage<cpx>)
            {
                const double2 old = s2[3 * BF_T];
                btma_sum = make_double2(btma_sum.x - old.x, btma_sum.y - old.y);
                btma_sum = make_double2(btma_sum.x + prod.x, btma_sum.y + prod.y);
                if (live) p.btma_ring[(size_t)btma_pos * cp + ch] = prod;
                btma_pos++; if (btma_pos >= p.btma_len) btma_pos = 0;
                mav = make_double2(div_exact(btma_sum.x, (double)p.btma_len, r_btma), div_exact(btma_sum.y, (double)p.btma_len, r_btma));
            }
            double fastarm = hypot(mav.x, mav.y);
            {   // mav1->UpdateSigned
                mav1_sum = mav1_sum - s1[2 * BF_T]; mav1_sum = mav1_sum + (fastarm);
                if (live) p.mav1_ring[(size_t)mav1_pos * cp + ch] = (fastarm);
                mav1_pos++; if (mav1_pos >= p.mav1_len) mav1_pos = 0;
                fastarm = div_exact(mav1_sum, (double)p.mav1_len, r_mav1);
            }
            {   // fastarm-=bt_ma_diff.update(fastarm): Delay<double>(126*SPS)
                if (live) p.btdiff_ring[(size_t)btdiff_pos * cp + ch] = fastarm;
                const double older = s1[3 * BF_T], newer = s1[4 * BF_T];
                const double w = p.btdiff_wv[btdiff_pos];
                fastarm -= (w * newer + (1.0 - w) * older);
                btdiff_pos++; if (btdiff_pos >= p.btdiff_len) btdiff_pos = 0;
            }
            if (fastarm < 0) fastarm = 0;
            double bt_sig = fastarm * fastarm;
            if (bt_sig > 500) bt_sig = 500;
            // PeakDetector::update (DSP.h:526-562)
            bool peak = false;
            {
                double val = bt_sig;
                if (live) p.pd3_ring[(size_t)pd3_pos * cp + ch] = val;        // d3.update_dont_touch
                pd3_pos++; if (pd3_pos >= pd3_sz) pd3_pos = 0;
                if (live) p.pd1_ring[(size_t)pd1_pos * cp + ch] = val;        // d1.update_dont_touch
                pd1_pos++; if (pd1_pos >= pd1_sz) pd1_pos = 0;
                const double dy = val - s1[5 * BF_T];
                if (live) p.pd2_ring[(size_t)pd2_pos * cp + ch] = val;        // d2.update(val)
                pd2_pos++; if (pd2_pos >= pd2_sz) pd2_pos = 0;
                val = s1[6 * BF_T];
                if ((!pd_cntdown) && (val > p.pd_threshold) && ((pd_lastdy >= 0 && dy < 0))) {
                    pd_cntdown = 2 * p.pd_len;
                    // d3.findmaxpos: scan the ring from its current position, first maximum wins (DSP.h:467-481)
                    int mp = 0, q = pd3_pos;
                    double mv = p.pd3_ring[(size_t)q * cp + ch];
                    for (int kk = 0; kk < pd3_sz; kk++) {
                        const double x = p.pd3_ring[(size_t)q * cp + ch];
                        if (x > mv) { mv = x; mp = kk; }
                        q++; if (q >= pd3_sz) q = 0;
                    }
                    pd_maxval = mv; pd_maxposcnt = mp;
                }
                if (pd_cntdown > 0) pd_cntdown--;
                pd_lastdy = dy;
                if (!pd_maxposcnt) { pd_maxposcnt--; peak = true; }
                else if (pd_maxposcnt > 0) pd_maxposcnt--;
            }
            if (peak) tri_ptr = 0;                                            // :430-435
            if (tri_ptr < p.tri_sz) {                                         // :437-442
                if (live) tri[(size_t)tri_slot * p.tri_sz + tri_ptr] = cval_d.x;
                tri_ptr++;
            } else if (tri_ptr == p.tri_sz) {                                 // fill complete -> event; the FFTs run after this kernel
                tri_ptr++;
                if (nev < BURST_MAXEV) {
                    if (live) p.ev_sample[(size_t)ch * BURST_MAXEV + nev] = i | (tri_slot << 24);
                    nev++;
                    tri_slot++; if (tri_slot >= BURST_MAXEV) tri_slot = 0;
                }
            }
        }
    }
    if (!live) return;
    BD(BD_AGC_SUM) = agc_sum; BD(BD_AGC_VAL) = agc_val; BD(BD_BTMA_SUM_RE) = btma_sum.x; BD(BD_BTMA_SUM_IM) = btma_sum.y;
    BD(BD_MAV1_SUM) = mav1_sum; BD(BD_PD_LASTDY) = pd_lastdy; BD(BD_PD_MAXVAL) = pd_maxval;
    BI(BI_PD_CNTDOWN) = pd_cntdown; BI(BI_PD_MAXPOSCNT) = pd_maxposcnt; BI(BI_TRI_PTR) = tri_ptr; BI(BI_TRI_SLOT) = tri_slot; BI(BI_NEV) = nev;
}

// ------------------------------------------------------------------------------------------------ trident FFTs + peak logic
// Block reduction over 1024 threads of (value, index) pairs: the maximum, the lowest index on ties. Index INT_MAX marks a
// thread without a candidate and loses to every real one. (The MSK peak search records a candidate only for m > 0, so there
// a real candidate also beats the (0.0, INT_MAX) sentinel by value.)
__device__ __forceinline__ int argmax_first(double *s_val, int *s_idx, double v, int idx)
{
    s_val[threadIdx.x] = v; s_idx[threadIdx.x] = idx;
    __syncthreads();
    for (int st = 512; st > 0; st >>= 1) {
        if (threadIdx.x < st) {
            const double ov = s_val[threadIdx.x + st]; const int oi = s_idx[threadIdx.x + st];
            if (oi != 0x7fffffff && (s_idx[threadIdx.x] == 0x7fffffff || ov > s_val[threadIdx.x] || (ov == s_val[threadIdx.x] && oi < s_idx[threadIdx.x]))) { s_val[threadIdx.x] = ov; s_idx[threadIdx.x] = oi; }
        }
        __syncthreads();
    }
    const int r = s_idx[0];
    __syncthreads();
    return r;
}

// one CTA per (event, base/top): zero-padded 32768-point complex FFT of a real segment, ping-pong between two HBM buffers
__global__ void __launch_bounds__(1024)
trident_fft_kernel(BurstParams p, const int *__restrict__ ev_list, int n_events, double2 *wa, double2 *wb, const double2 *__restrict__ tw)
{
    const int e = blockIdx.x >> 1, which = blockIdx.x & 1;
    if (e >= n_events) return;
    const int ch = ev_list[2 * e], ev = ev_list[2 * e + 1];
    const int slot = p.ev_sample[(size_t)ch * BURST_MAXEV + ev] >> 24;
    const double *buf = p.tri + ((size_t)ch * BURST_MAXEV + slot) * p.tri_sz;
    const int nb = p.tri_nb, nt = p.tri_nt;
    const int off = which ? nb : 0, cnt = which ? nt : nb;
    double2 *a = wa + (size_t)blockIdx.x * TRI_N, *b = wb + (size_t)blockIdx.x * TRI_N;
    for (int j = threadIdx.x; j < TRI_N; j += blockDim.x)
        a[j] = make_double2((j < cnt && off + j < p.tri_sz) ? buf[off + j] : 0.0, 0.0);
    __syncthreads();
    // 32768 = 8^5
    pass8<false>(a, b, TRI_N, 1, tw, 1); __syncthreads();
    pass8<false>(b, a, TRI_N, 8, tw, 1); __syncthreads();
    pass8<false>(a, b, TRI_N, 64, tw, 1); __syncthreads();
    pass8<false>(b, a, TRI_N, 512, tw, 1); __syncthreads();
    pass8<false>(a, b, TRI_N, 4096, tw, 1); __syncthreads();      // spectrum in b
}
// one CTA per event: strongest base bin and the two side peaks of the top section (:478-520)
__global__ void __launch_bounds__(1024)
trident_peaks_kernel(BurstParams p, const int *__restrict__ ev_list, int n_events, const double2 *__restrict__ wb)
{
    __shared__ double s_val[1024];
    __shared__ int s_idx[1024];
    __shared__ int s_minbin;
    const int e = blockIdx.x;
    if (e >= n_events) return;
    const int ch = ev_list[2 * e], ev = ev_list[2 * e + 1];
    const double2 *base = wb + (size_t)(2 * e) * TRI_N, *top = wb + (size_t)(2 * e + 1) * TRI_N;
    const int half = TRI_N / 2;
    const double hzperbin = p.Fs / ((double)TRI_N);
    const int peakspacingbins = (int)rint((0.5 * p.fb) / hzperbin);     // qRound of a positive value
    // strongest base bin: strict '>' scanning upwards from (0, bin 0)
    double bv = 0.0; int bi = 0x7fffffff;
    for (int k = threadIdx.x; k < half; k += blockDim.x) { const double m = hypot(base[k].x, base[k].y); if (m > bv) { bv = m; bi = k; } }
    int minvalbin = argmax_first(s_val, s_idx, bv, bi);
    if (minvalbin == 0x7fffffff) minvalbin = 0;
    if (threadIdx.x == 0) s_minbin = minvalbin;
    __syncthreads();
    minvalbin = s_minbin;
    const double minval = hypot(base[minvalbin].x, base[minvalbin].y) > 0.0 ? hypot(base[minvalbin].x, base[minvalbin].y) : 0.0;
    double lv = 0.0, hv = 0.0; int li = 0x7fffffff, hi = 0x7fffffff;
    for (int k = threadIdx.x; k < half; k += blockDim.x) {
        if (k > 50) {
            const double m = hypot(top[k].x, top[k].y);
            if ((k < minvalbin - (peakspacingbins / 2)) && m > lv) { lv = m; li = k; }
            if ((k > minvalbin + (peakspacingbins / 2)) && m > hv) { hv = m; hi = k; }
        }
    }
    int maxtoppos = argmax_first(s_val, s_idx, lv, li); if (maxtoppos == 0x7fffffff) maxtoppos = 0;
    int maxtopposhigh = argmax_first(s_val, s_idx, hv, hi); if (maxtopposhigh == 0x7fffffff) maxtopposhigh = 0;
    if (threadIdx.x == 0) {
        double *r = p.ev_result + ((size_t)ch * BURST_MAXEV + ev) * 8;
        r[0] = (double)minvalbin; r[1] = minval; r[2] = (double)maxtoppos; r[3] = (double)maxtopposhigh;
        r[4] = atan2(base[minvalbin].y, base[minvalbin].x);              // std::arg(out_base[minvalbin])
    }
}

// burst OQPSK: three-peak "trident" on |top|-|base| plus the strongest base bin (burstoqpskdemodulator.cpp:416-465)
__global__ void __launch_bounds__(1024)
trident_peaks_oqpsk_kernel(BurstParams p, const int *__restrict__ ev_list, int n_events, const double2 *__restrict__ wb, double2 *__restrict__ wa)
{
    __shared__ double s_val[1024];
    __shared__ int s_idx[1024];
    const int e = blockIdx.x;
    if (e >= n_events) return;
    const int ch = ev_list[2 * e], ev = ev_list[2 * e + 1];
    const double2 *base = wb + (size_t)(2 * e) * TRI_N, *top = wb + (size_t)(2 * e + 1) * TRI_N;
    double *diff = reinterpret_cast<double *>(wa + (size_t)(2 * e) * TRI_N);      // scratch: the FFT input buffer is free now
    const int half = TRI_N / 2;
    const double hzperbin = p.Fs / ((double)TRI_N);
    const int bps = (int)rint((0.25 * p.fb) / hzperbin);
    for (int k = threadIdx.x; k < half; k += blockDim.x) diff[k] = (hypot(top[k].x, top[k].y) - hypot(base[k].x, base[k].y));
    __syncthreads();
    // maxval over i in [firstbin, lstbin): starts at (testval(firstbin), firstbin), strict '>' -> first maximum
    const int firstbin = bps, lstbin = half - bps;
    double tv = 0.0; int ti = 0x7fffffff;
    for (int k = firstbin + threadIdx.x; k < lstbin; k += blockDim.x) {
        const double t = diff[k - bps] + diff[k + bps] - diff[k];
        if (ti == 0x7fffffff || t > tv) { tv = t; ti = k; }
    }
    int maxvalbin = argmax_first(s_val, s_idx, tv, ti); if (maxvalbin == 0x7fffffff) maxvalbin = firstbin;
    const double maxval = diff[maxvalbin - bps] + diff[maxvalbin + bps] - diff[maxvalbin];
    double bv = 0.0; int bi = 0x7fffffff;
    for (int k = threadIdx.x; k < half; k += blockDim.x) { const double m = hypot(base[k].x, base[k].y); if (bi == 0x7fffffff || m > bv) { bv = m; bi = k; } }
    int minvalbin = argmax_first(s_val, s_idx, bv, bi); if (minvalbin == 0x7fffffff) minvalbin = 0;
    if (threadIdx.x == 0) {
        double *r = p.ev_result + ((size_t)ch * BURST_MAXEV + ev) * 8;
        r[0] = (double)minvalbin; r[1] = hypot(base[minvalbin].x, base[minvalbin].y); r[2] = (double)maxvalbin; r[3] = maxval;
        r[4] = atan2(base[minvalbin].y, base[minvalbin].x);
    }
}

// ------------------------------------------------------------------------------------------------ demodulator tails
// Stages both tails use that the continuous demodulators do not; the shared ones come from demod_stages.cuh.

// chunk-relative sample of channel ch's trident event ev, or -1 after the last one
__device__ __forceinline__ int event_sample(const BurstParams &p, int ch, int ev, int nev)
{ return ev < nev ? (p.ev_sample[(size_t)ch * BURST_MAXEV + ev] & 0xffffff) : -1; }

// FIR::FIRUpdateAndProcess's sum (DSP.cpp:296-303) of the burst OQPSK tail over the nt1 = ntaps + 1 row delay line, taps in
// reference order from the oldest entry (row pos, the one after the newest) on
__device__ __forceinline__ double2 fir_wrapped(const BurstParams &p, const double *s_re, const double *s_im, int nt1, int lane, int pos)
{
    double sre = 0, sim = 0;
    for (int k = 0; k < p.ntaps; k++) {
        sre += p.taps[k] * s_re[pos * 32 + lane]; sim += p.taps[k] * s_im[pos * 32 + lane];
        pos++; if (pos >= nt1) pos = 0;
    }
    return make_double2(sre, sim);
}

// Delay<double> of k whole samples plus a fraction (DSP.h:357-374) as a ring of k + 1 rows [row][cpad] at position pos:
// stores x, returns w * x[n-k+1] + (1 - w) * x[n-k] with w the weight of the current position
__device__ __forceinline__ double ring_delay(double *ring, size_t cpad, int ch, int &pos, int k, double w, double x)
{
    const int len = k + 1;
    ring[(size_t)pos * cpad + ch] = x;
    int io = pos - k; if (io < 0) io += len;
    int in_ = io + 1; if (in_ >= len) in_ = 0;
    const double out = (w * ring[(size_t)in_ * cpad + ch] + (1.0 - w) * ring[(size_t)io * cpad + ch]);
    pos++; if (pos >= len) pos = 0;
    return out;
}

// Preamble symbol-tone PLL (burstmskdemodulator.cpp:606-626, burstoqpskdemodulator.cpp:538-558): strot follows the symbol
// tone of sig2 with loop gain `gain`, savrot <- keep * savrot + mix * strot. The tone, with its imaginary part replaced by its
// real part half a symbol earlier (a1), is compared with oscillator o; returns that phase error, unscaled.
__device__ __forceinline__ double symbol_tone_error(const BurstParams &p, int ch, double2 sig2, double gain, double keep, double mix,
                                                    double2 &strot, double2 &savrot, int &a1_pos, const Osc &o)
{
    const double2 spt = c_mul(c_mul(sig2, strot), make_double2(0.0, 1.0));
    const double er = tanh(spt.y) * (spt.x);
    const double ang = (1.0 * er) * gain;
    strot = c_mul(strot, make_double2(cos(ang), sin(ang)));
    savrot = make_double2(savrot.x * keep + mix * strot.x, savrot.y * keep + mix * strot.y);
    const double a1out = ring_delay(p.a1_ring, p.cpad, ch, a1_pos, p.a1_k, p.a1_wv[a1_pos], spt.x);   // a1.update(spt.real())
    const int t = osc_index(o.ptr);
    const double2 q = c_mul(make_double2(p.cos_t[t], p.sin_t[t]), make_double2(spt.x, -a1out));
    return atan2(q.y, q.x);
}

// Delay<double>(T/4) and Delay<double>(T/8) of the OQPSK symbol timing (DSP.h:357-374) for a delay of k = 1..3 samples, the
// three most recent inputs held in registers. w is the interpolation weight of the current ring position. (The
// continuous OQPSK kernels keep their inline form: compiled through this struct their SASS changes.)
struct Delay3 {
    double d0, d1, d2;                    // x[n-1], x[n-2], x[n-3]
    __device__ __forceinline__ double update(int k, double w, double x)
    {
        const double older = (k == 3) ? d2 : (k == 2 ? d1 : d0);
        const double newer = (k == 3) ? d1 : (k == 2 ? d0 : x);
        const double out = (w * newer + (1.0 - w) * older);
        d2 = d1; d1 = d0; d0 = x;
        return out;
    }
};

// a soft bit: qRound, clamped to 0..255
__device__ __forceinline__ int soft_byte(double v)
{
    int ibit = q_round(v);
    if (ibit > 255) ibit = 255;
    if (ibit < 0) ibit = 0;
    return ibit;
}
// RxDataBits.push_back of the burst demodulators. Unlike push_soft, a value past the ring's capacity only flags the overflow
// and is not counted as pending, and the value goes in as given: the start-of-burst marker -1 is not clamped.
__device__ __forceinline__ void burst_push_soft(const BurstParams &p, int ch, int count, int &pending, int &overflow, int v)
{
    const int pos = count + pending;
    if (pos < p.soft_cap) { p.soft[(size_t)ch * p.soft_cap + pos] = (int16_t)v; pending++; } else overflow = 1;
}

// ------------------------------------------------------------------------------------------------ burst MSK tail
__global__ void __launch_bounds__(32)
burst_back_kernel(const __grid_constant__ BurstParams p, int n)
{
    extern __shared__ double bsm[];
    const int lane = threadIdx.x;
    const int ch = blockIdx.x * 32 + lane;
    if (ch >= p.n_channels) return;
    const size_t cp = p.cpad;
    const int nt1 = p.ntaps + 1;
    double *s_re = bsm, *s_im = bsm + (size_t)nt1 * 32;
    for (int k = 0; k < nt1; k++) { s_re[k * 32 + lane] = p.fir_re[(size_t)k * cp + ch]; s_im[k * 32 + lane] = p.fir_im[(size_t)k * cp + ch]; }
    Osc m2 = {BD(BD_M2_PTR), BD(BD_M2_STEP), BD(BD_M2_FREQ), BD(BD_M2_LAST)};
    Osc mc = {BD(BD_MC_PTR), BD(BD_MC_STEP), BD(BD_MC_FREQ), BD(BD_MC_LAST)};
    Osc st = {BD(BD_ST_PTR), BD(BD_ST_STEP), BD(BD_ST_FREQ), BD(BD_ST_LAST)};
    Osc sh = {BD(BD_SH_PTR), BD(BD_SH_STEP), BD(BD_SH_FREQ), BD(BD_SH_LAST)};
    double vol_gain = BD(BD_VOL_GAIN), mse = BD(BD_MSE), msema_sum = BD(BD_MSEMA_SUM), rot_freq = BD(BD_ROT_FREQ);
    double2 rot = make_double2(BD(BD_ROT_RE), BD(BD_ROT_IM)), strot = make_double2(BD(BD_STR_RE), BD(BD_STR_IM)), savrot = make_double2(BD(BD_SAV_RE), BD(BD_SAV_IM));
    double eb_sum1 = BD(BD_EB_SUM1), eb_sum2 = BD(BD_EB_SUM2), eb_ebno = BD(BD_EB_EBNO), agc2_sum = BD(BD_AGC2_SUM), agc2_val = BD(BD_AGC2_VAL);
    Biquad res = {BD(BD_RES_X1), BD(BD_RES_X2), BD(BD_RES_Y1), BD(BD_RES_Y2)};
    double diff_last = BD(BD_DIFF_LAST), last_ebno_emit = BD(BD_LAST_EBNO_EMIT);
    int cntr = BI(BI_CNTR), startstop = BI(BI_STARTSTOP), dcd = BI(BI_DCD);
    int fir_pos = BI(BI_FIR_POS), a1_pos = BI(BI_A1_POS), eb_pos = BI(BI_EB_POS), agc2_pos = BI(BI_AGC2_POS), ds_pos = BI(BI_DS_POS), d8_pos = BI(BI_D8_POS), msema_pos = BI(BI_MSEMA_POS);
    int soft_count = BI(BI_SOFT_COUNT), soft_pending = BI(BI_SOFT_PENDING), soft_overflow = BI(BI_SOFT_OVERFLOW);
    int sig_true = BI(BI_SIG_TRUE), sig_false = BI(BI_SIG_FALSE), ebno_emits = BI(BI_EBNO_EMITS);
    const int nev = BI(BI_NEV);
    int next_ev = 0;
    int next_ev_sample = event_sample(p, ch, 0, nev);
    const double *vtd = p.vtd + (size_t)ch * p.astride;
    const double sps = (double)p.sps;
    const MeanDiv eb_mean(p.eb_len), agc2_mean(p.agc2_len), msema_mean(p.msema_len);
    for (int i = 0; i < n; i++) {
        if (i == next_ev_sample) {
            // trident test (:474-568) with the spectra computed by burst_trident for this fill
            const double *r = p.ev_result + ((size_t)ch * BURST_MAXEV + next_ev) * 8;
            const int minvalbin = (int)r[0], maxtoppos = (int)r[2], maxtopposhigh = (int)r[3];
            const double minval = r[1];
            const double hzperbin = p.Fs / ((double)TRI_N);
            const int peakspacingbins = (int)rint((0.5 * p.fb) / hzperbin);
            const int distfrompeak = abs(maxtoppos - minvalbin);
            if (minval > 500.0 && abs(distfrompeak - peakspacingbins) < abs(peakspacingbins / 20) && !(dcd) && !(cntr > 0 && cntr < (500 * sps))) {
                vol_gain = 1.4142 * (500.0 / (minval / 3));
                const double carrierphase = r[4] - (M_PI / 4.0);
                osc_set_phase_deg(m2, (180.0 / M_PI) * carrierphase);
                osc_set_freq(m2, ((maxtopposhigh + maxtoppos) / 2) * hzperbin, p.Fs);
                {   // CenterFreqChangedSlot (:326-343)
                    double fc = ((maxtopposhigh + maxtoppos) / 2) * hzperbin;
                    if (fc < (0.75 * p.fb)) fc = 0.75 * p.fb;
                    if (fc > (p.Fs / 2.0 - 0.75 * p.fb)) fc = p.Fs / 2.0 - 0.75 * p.fb;
                    mc.freq = fc; if (mc.freq < 0) mc.freq = 0;
                    mc.step = (mc.freq) * ((double)WTSIZE) / ((double)((float)((int)p.Fs)));   // SetFreq(freq,Fs)
                    while (((int)mc.ptr) >= WTSIZE) mc.ptr -= WTSIZE;
                    if (p.afc) osc_set_freq(m2, mc.freq, p.Fs);
                    if ((m2.freq - mc.freq) > (p.lockingbw / 2.0)) osc_set_freq(m2, mc.freq + (p.lockingbw / 2.0), p.Fs);
                    if ((m2.freq - mc.freq) < (-p.lockingbw / 2.0)) osc_set_freq(m2, mc.freq - (p.lockingbw / 2.0), p.Fs);
                }
                startstop = p.startstopstart; cntr = 0; sig_true++;
                soft_pending = 0; burst_push_soft(p, ch, soft_count, soft_pending, soft_overflow, -1);   // RxDataBits.clear(); push_back(-1)
                mse = 0;
                for (int k = 0; k < p.msema_len; k++) p.msema_ring[(size_t)k * cp + ch] = 0.0;   // msema->Zero()
                msema_pos = 0; msema_sum = 0;
                savrot = make_double2(1.0, 0.0); strot = make_double2(1.0, 0.0); rot = make_double2(1.0, 0.0); rot_freq = 0;
                res.x1 = res.x2 = res.y1 = res.y2 = 0;                    // st_iir_resonator.init()
                osc_set_phase_deg(st, 0); osc_set_phase_deg(sh, 0);
            }
            next_ev++;
            next_ev_sample = event_sample(p, ch, next_ev, nev);
        }
        if (startstop > 0) {                                              // :571-586
            if (cntr >= (p.start_processing * sps)) startstop--;
            if (cntr < 1000000) cntr++;
            if (mse < p.signalthreshold) startstop = p.startstopstart;
        }
        if (startstop == 0) { startstop--; sig_false++; cntr = 0; mse = 1; }   // :588-596
        if (startstop > 0 || mse < p.signalthreshold) {                  // :599
            const int t2 = osc_index(m2.ptr);
            const double v = vtd[i];
            const double cre = (p.cos_t[t2] * (v)) * vol_gain, cim = (p.sin_t[t2] * (v)) * vol_gain;   // CIS*(val)*vol_gain
            // the FIR written out: through fir_push and fir_wrapped this kernel compiles to 56 more instructions and the
            // 1200 bps burst workload runs 0.5 % slower
            s_re[fir_pos * 32 + lane] = cre; s_im[fir_pos * 32 + lane] = cim;
            fir_pos++; if (fir_pos >= nt1) fir_pos = 0;
            double sre = 0, sim = 0;
            { int tp = fir_pos; for (int k = 0; k < p.ntaps; k++) { sre += p.taps[k] * s_re[tp * 32 + lane]; sim += p.taps[k] * s_im[tp * 32 + lane]; tp++; if (tp >= nt1) tp = 0; } }
            double2 sig2 = make_double2(sre, sim);
            if (cntr > (p.start_processing * sps) && cntr < p.end_rotation) {       // :606-626 preamble symbol tone
                double st_err = symbol_tone_error(p, ch, sig2, 0.5, 0.999, 0.001, strot, savrot, a1_pos, sh);
                double progress = (double)cntr - (sps * (p.start_processing));
                const double goal = p.end_rotation - (sps * p.start_processing);
                progress = progress / goal;
                st_err *= 0.5 * (1.0 - progress * progress);
                osc_advance_fraction_of_wave(sh, -(1.0 / (2.0 * M_PI)) * st_err * 0.05);
                osc_set_phase_deg(st, (360.0 * sh.ptr / ((double)WTSIZE)) + (360.0 * (1.0 - p.ee)));
            }
            sig2 = c_mul(sig2, savrot);                                    // :628-630
            rot = c_mul(rot, make_double2(cos(rot_freq), sin(rot_freq)));
            sig2 = c_mul(sig2, rot);
            {   // MSKEbNoMeasure::Update(std::abs(sig2)) (DSP.cpp:493-505)
                const double ab = hypot(sig2.x, sig2.y), sq = ab * ab;
                const size_t e = (size_t)eb_pos * cp + ch;
                ma_push(eb_sum2, p.eb2_ring[e], sq);
                ma_push(eb_sum1, p.eb1_ring[e], ab);
                eb_pos++; if (eb_pos >= p.eb_len) eb_pos = 0;
                msk_ebno_readout(eb_mean, eb_ebno, eb_sum1, eb_sum2);
                if (cntr == p.end_rotation + (200 * p.sps)) { last_ebno_emit = eb_ebno; ebno_emits++; }   // :637-640
                // sig2*=agc2->Update(std::abs(sig2)) (:643)
                ma_push(agc2_sum, p.agc2_ring[(size_t)agc2_pos * cp + ch], ab);
                agc2_pos++; if (agc2_pos >= p.agc2_len) agc2_pos = 0;
                agc2_val = agc_gain(agc2_mean, agc2_sum);
                sig2 = make_double2(sig2.x * agc2_val, sig2.y * agc2_val);
            }
            const double abval = hypot(sig2.x, sig2.y);
            if (abval > 2.84) { const double g = (2.84 / abval); sig2 = make_double2(g * sig2.x, g * sig2.y); }
            double2 pt_d;                                                 // delayedsmpl.update_dont_touch(sig2) (:650)
            { p.ds_ring[(size_t)ds_pos * cp + ch] = sig2; ds_pos++; if (ds_pos >= p.ds_len) ds_pos = 0; pt_d = p.ds_ring[(size_t)ds_pos * cp + ch]; }
            const double2 pt_msk = make_double2(sig2.x, pt_d.y);
            double st_eta = biquad_update(res, hypot(pt_msk.x, pt_msk.y), p.res_a1, p.res_a2, p.res_b0, p.res_b1, p.res_b2);
            const double d8out = ring_delay(p.d8_ring, cp, ch, d8_pos, p.d8_k, p.d8_w, st_eta);
            const int ts = osc_index(st.ptr);
            const double2 st_out = c_mul(make_double2(p.cos_t[ts], p.sin_t[ts]), make_double2(st_eta, -d8out));
            const double st_angle_error = atan2_fast(st_out.y, st_out.x);
            if (cntr > p.end_rotation) osc_advance_fraction_of_wave(st, -st_angle_error * 0.002 / 360.0);   // :661-665
            double frac;
            if (osc_have_passed_point(st, p.ee, frac)) {                  // :668
                double ct_ec = ct_error(sig2, pt_d);
                if (ct_ec > M_PI_2) ct_ec = M_PI_2;
                if (ct_ec < -M_PI_2) ct_ec = -M_PI_2;
                if (cntr > (p.start_processing * sps)) {                  // :680-687
                    const double ang = (1.0 * ct_ec) * 0.25;
                    rot = c_mul(rot, make_double2(cos(ang), sin(ang)));
                    if (cntr > p.end_rotation) rot_freq = rot_freq + ct_ec * 0.0001;
                }
                if (cntr > (p.start_processing * sps)) {                  // :706-711 msema MA(75)
                    const double tda = (fabs(pt_msk.x * 0.75) - 1.0), tdb = (fabs(pt_msk.y * 0.75) - 1.0);
                    ma_push(msema_sum, p.msema_ring[(size_t)msema_pos * cp + ch], (tda * tda) + (tdb * tdb));
                    msema_pos++; if (msema_pos >= p.msema_len) msema_pos = 0;
                    mse = msema_mean(msema_sum);
                }
                const double r1 = diff_update_soft(diff_last, pt_msk.y);    // DiffDecode::UpdateSoft (DSP.cpp:531-563)
                burst_push_soft(p, ch, soft_count, soft_pending, soft_overflow, soft_byte((r1) * 127.0 + 128.0));
                const double r2 = -diff_update_soft(diff_last, pt_msk.x);
                burst_push_soft(p, ch, soft_count, soft_pending, soft_overflow, soft_byte((r2) * 127.0 + 128.0));
                if (soft_pending >= 12) { soft_count += soft_pending; soft_pending = 0; }   // :735-739
            }
            osc_next_frame(st); osc_next_frame(sh); osc_next_frame(m2); osc_next_frame(mc);   // :744-748
        }
    }
    for (int k = 0; k < nt1; k++) { p.fir_re[(size_t)k * cp + ch] = s_re[k * 32 + lane]; p.fir_im[(size_t)k * cp + ch] = s_im[k * 32 + lane]; }
    BD(BD_M2_PTR) = m2.ptr; BD(BD_M2_STEP) = m2.step; BD(BD_M2_FREQ) = m2.freq; BD(BD_M2_LAST) = m2.last;
    BD(BD_MC_PTR) = mc.ptr; BD(BD_MC_STEP) = mc.step; BD(BD_MC_FREQ) = mc.freq; BD(BD_MC_LAST) = mc.last;
    BD(BD_ST_PTR) = st.ptr; BD(BD_ST_STEP) = st.step; BD(BD_ST_FREQ) = st.freq; BD(BD_ST_LAST) = st.last;
    BD(BD_SH_PTR) = sh.ptr; BD(BD_SH_STEP) = sh.step; BD(BD_SH_FREQ) = sh.freq; BD(BD_SH_LAST) = sh.last;
    BD(BD_VOL_GAIN) = vol_gain; BD(BD_MSE) = mse; BD(BD_MSEMA_SUM) = msema_sum; BD(BD_ROT_FREQ) = rot_freq;
    BD(BD_ROT_RE) = rot.x; BD(BD_ROT_IM) = rot.y; BD(BD_STR_RE) = strot.x; BD(BD_STR_IM) = strot.y; BD(BD_SAV_RE) = savrot.x; BD(BD_SAV_IM) = savrot.y;
    BD(BD_EB_SUM1) = eb_sum1; BD(BD_EB_SUM2) = eb_sum2; BD(BD_EB_EBNO) = eb_ebno; BD(BD_AGC2_SUM) = agc2_sum; BD(BD_AGC2_VAL) = agc2_val;
    BD(BD_RES_X1) = res.x1; BD(BD_RES_X2) = res.x2; BD(BD_RES_Y1) = res.y1; BD(BD_RES_Y2) = res.y2;
    BD(BD_DIFF_LAST) = diff_last; BD(BD_LAST_EBNO_EMIT) = last_ebno_emit;
    BI(BI_CNTR) = cntr; BI(BI_STARTSTOP) = startstop;
    BI(BI_FIR_POS) = fir_pos; BI(BI_A1_POS) = a1_pos; BI(BI_EB_POS) = eb_pos; BI(BI_AGC2_POS) = agc2_pos; BI(BI_DS_POS) = ds_pos; BI(BI_D8_POS) = d8_pos; BI(BI_MSEMA_POS) = msema_pos;
    BI(BI_SOFT_COUNT) = soft_count; BI(BI_SOFT_PENDING) = soft_pending; BI(BI_SOFT_OVERFLOW) = soft_overflow;
    BI(BI_SIG_TRUE) = sig_true; BI(BI_SIG_FALSE) = sig_false; BI(BI_EBNO_EMITS) = ebno_emits;
}

// ------------------------------------------------------------------------------------------------ burst OQPSK tail
// BurstOqpskDemodulator::writeDataSlot after the trident check (burstoqpskdemodulator.cpp:508-733). Unlike the MSK burst
// tail this one runs on every sample, so all its sample-rate rings advance in lock-step.
__global__ void __launch_bounds__(32)
burst_oqpsk_back_kernel(const __grid_constant__ BurstParams p, long long sample0, int n, int new_write)
{
    extern __shared__ double bsm[];
    const int lane = threadIdx.x;
    const int ch = blockIdx.x * 32 + lane;
    if (ch >= p.n_channels) return;
    const size_t cp = p.cpad;
    const int nt1 = p.ntaps + 1;
    double *s_re = bsm, *s_im = bsm + (size_t)nt1 * 32;
    for (int k = 0; k < nt1; k++) { s_re[k * 32 + lane] = p.fir_re[(size_t)k * cp + ch]; s_im[k * 32 + lane] = p.fir_im[(size_t)k * cp + ch]; }
    Osc m2 = {BD(BD_M2_PTR), BD(BD_M2_STEP), BD(BD_M2_FREQ), BD(BD_M2_LAST)};
    Osc st = {BD(BD_ST_PTR), BD(BD_ST_STEP), BD(BD_ST_FREQ), BD(BD_ST_LAST)};
    Osc sr = {BD(BD_SR_PTR), BD(BD_SR_STEP), BD(BD_SR_FREQ), BD(BD_SR_LAST)};
    Osc sq = {BD(BD_SH_PTR), BD(BD_SH_STEP), BD(BD_SH_FREQ), BD(BD_SH_LAST)};      // st_osc_quarter
    double vol_gain = BD(BD_VOL_GAIN), mse = BD(BD_MSE), msema_sum = BD(BD_MSEMA_SUM), rot_freq = BD(BD_ROT_FREQ);
    double2 rot = make_double2(BD(BD_ROT_RE), BD(BD_ROT_IM)), strot = make_double2(BD(BD_STR_RE), BD(BD_STR_IM)), savrot = make_double2(BD(BD_SAV_RE), BD(BD_SAV_IM));
    double eb_sum1 = BD(BD_EB_SUM1), eb_sum2 = BD(BD_EB_SUM2), eb_ebno = BD(BD_EB_EBNO), agc2_sum = BD(BD_AGC2_SUM), agc2_val = BD(BD_AGC2_VAL);
    Biquad res = {BD(BD_RES_X1), BD(BD_RES_X2), BD(BD_RES_Y1), BD(BD_RES_Y2)};
    double dly_s0 = BD(BD_DLY_S0);
    Delay3 d41 = {BD(BD_DLY41_0), BD(BD_DLY41_1), BD(BD_DLY41_2)}, d42 = {BD(BD_DLY42_0), BD(BD_DLY42_1), BD(BD_DLY42_2)};
    Delay3 d8 = {BD(BD_DLY8_0), BD(BD_DLY8_1), BD(BD_DLY8_2)};
    double2 sig2_last = make_double2(BD(BD_SIG2L_RE), BD(BD_SIG2L_IM)), pt_d = make_double2(BD(BD_PTD_RE), BD(BD_PTD_IM));
    double lastmse = BD(BD_LASTMSE), last_ebno_emit = BD(BD_LAST_EBNO_EMIT);
    if (new_write) lastmse = mse;                                         // :317
    int cntr = BI(BI_CNTR), startstop = BI(BI_STARTSTOP), yui = BI(BI_YUI), insertpreamble = BI(BI_INSERTPREAMBLE);
    int a1_pos = BI(BI_A1_POS), msema_pos = BI(BI_MSEMA_POS);
    int soft_count = BI(BI_SOFT_COUNT), soft_pending = BI(BI_SOFT_PENDING), soft_overflow = BI(BI_SOFT_OVERFLOW);
    int sig_true = BI(BI_SIG_TRUE), sig_false = BI(BI_SIG_FALSE), ebno_emits = BI(BI_EBNO_EMITS);
    const int nev = BI(BI_NEV);
    int next_ev = 0;
    int next_ev_sample = event_sample(p, ch, 0, nev);
    const double *vtd = p.vtd + (size_t)ch * p.astride;
    const double SPS = p.spsd;
    int fir_pos = (int)(sample0 % nt1), eb_pos = (int)(sample0 % p.eb_len), agc2_pos = (int)(sample0 % p.agc2_len);
    int p41 = (int)(sample0 % (p.k41 + 1)), p8 = (int)(sample0 % (p.k8 + 1));
    const MeanDiv agc2_mean(p.agc2_len), msema_mean(p.msema_len);
    for (int i = 0; i < n; i++) {
        if (i == next_ev_sample) {                                        // trident test outcome (:466-504)
            const double *r = p.ev_result + ((size_t)ch * BURST_MAXEV + next_ev) * 8;
            const double minvalbin = r[0], minval = r[1], maxvalbin = r[2], maxval = r[3];
            const double hzperbin = p.Fs / ((double)TRI_N);
            if ((maxval > 500.0) && (fabs((((double)(maxvalbin - minvalbin))) * hzperbin) < 20.0)) {
                const double carrierphase = r[4] - (M_PI / 4.0);
                osc_set_freq(m2, hzperbin * minvalbin, p.Fs);
                osc_set_phase_deg(m2, (180.0 / M_PI) * carrierphase);
                vol_gain = 1.4142 * 500.0 / minval;
                osc_set_freq(st, sr.freq, p.Fs);
                osc_set_phase_deg(st, 0); osc_set_phase_deg(sr, 0);
                res.x1 = res.x2 = res.y1 = res.y2 = 0;
                startstop = p.startstopstart; cntr = 0; rot = make_double2(1.0, 0.0); insertpreamble = 1; rot_freq = 0;
                savrot = make_double2(1.0, 0.0);
                sig_true++;
                mse = 0;
                for (int k = 0; k < p.msema_len; k++) p.msema_ring[(size_t)k * cp + ch] = 0.0;
                msema_pos = 0; msema_sum = 0;
            }
            next_ev++;
            next_ev_sample = event_sample(p, ch, next_ev, nev);
        }
        // mix + RRC (:509-512)
        const int t2 = osc_index(m2.ptr);
        const double gv = (vol_gain * vtd[i]);
        fir_push(s_re, s_im, nt1, lane, fir_pos, p.cos_t[t2] * gv, p.sin_t[t2] * gv);
        double2 sig2 = fir_wrapped(p, s_re, s_im, nt1, lane, fir_pos);
        if (startstop > 0) { startstop--; if (cntr < 1000000) cntr++; if (mse < 0.75) startstop = p.startstopstart; }   // :515-524
        if (startstop == 0) { startstop--; sig_false++; }                 // :525-529
        if ((cntr > ((256 - 10) * SPS)) && insertpreamble) {             // :531-535
            burst_push_soft(p, ch, soft_count, soft_pending, soft_overflow, -1); insertpreamble = 0;
        }
        if ((cntr > SPS * (128 + 10)) && (cntr < ((256 - 10) * SPS))) {  // :538-558
            const double progress = (((double)cntr) - (SPS * (128 + 10))) / (((256 - 10) * SPS) - (SPS * (128 + 10)));
            double st_err = symbol_tone_error(p, ch, sig2, 0.01, 0.95, 0.05, strot, savrot, a1_pos, sq);
            st_err *= 1.5 * (1.0 - progress * progress);
            osc_advance_fraction_of_wave(sq, -(1.0 / (2.0 * M_PI)) * st_err * 0.1);
            osc_set_phase_deg(st, ((360.0 * sq.ptr / ((double)WTSIZE))) * 4.0 + (360.0 * p.ee));
        }
        sig2 = c_mul(sig2, savrot);                                        // :562-565
        rot = c_mul(rot, make_double2(cos(rot_freq), sin(rot_freq)));
        sig2 = c_mul(sig2, rot);
        const double sig2abs = hypot(sig2.x, sig2.y);
        {   // OQPSKEbNoMeasure::Update (DSP.cpp:729-744)
            const size_t e = (size_t)eb_pos * cp + ch;
            ma_push(eb_sum2, p.eb2_ring[e], sig2abs * sig2abs);
            ma_push(eb_sum1, p.eb1_ring[e], sig2abs);
            eb_pos++; if (eb_pos >= p.eb_len) eb_pos = 0;
            oqpsk_ebno_readout(p.eb_len, p.Fs, p.fb, eb_ebno, eb_sum1, eb_sum2);
        }
        if (fabs(cntr - ((128.0 + 128.0 + 128.0) * SPS)) < 0.5) { last_ebno_emit = eb_ebno; ebno_emits++; }   // :573
        {   // sig2*=agc2->Update(sig2abs) (:576)
            ma_push(agc2_sum, p.agc2_ring[(size_t)agc2_pos * cp + ch], sig2abs);
            agc2_pos++; if (agc2_pos >= p.agc2_len) agc2_pos = 0;
            agc2_val = agc_gain(agc2_mean, agc2_sum);
            sig2 = make_double2(sig2.x * agc2_val, sig2.y * agc2_val);
        }
        const double abval = hypot(sig2.x, sig2.y);
        if (abval > 2.84) { const double g = (2.84 / abval); sig2 = make_double2(g * sig2.x, g * sig2.y); }
        // symbol timing (:583-603)
        const double ab2 = abval * abval;
        const double st_diff = (0.0 * ab2 + (1.0 - 0.0) * dly_s0) - (ab2);
        dly_s0 = ab2;
        const double w41 = p.w41v[p41], w8 = p.w8v[p8];
        p41++; if (p41 > p.k41) p41 = 0;
        p8++; if (p8 > p.k8) p8 = 0;
        const double st_d1out = d41.update(p.k41, w41, st_diff);
        const double st_d2out = d42.update(p.k41, w41, st_d1out);
        double st_eta = (st_d2out - st_diff) * st_d1out;
        const double resy = biquad_update(res, st_eta, p.res_a1, p.res_a2, p.res_b0, p.res_b1, p.res_b2);
        if (cntr > SPS * (128 + 128)) st_eta = resy;
        const double d8out = d8.update(p.k8, w8, st_eta);
        const int ts = osc_index(st.ptr);
        const double2 st_out = c_mul(make_double2(p.cos_t[ts], p.sin_t[ts]), make_double2(st_eta, -d8out));
        const double st_angle_error = atan2_fast(st_out.y, st_out.x);
        if (cntr > SPS * (128 + 64)) {
            osc_set_freq(st, (-st_angle_error * 0.00000001) + st.freq, p.Fs);
            osc_advance_fraction_of_wave(st, -st_angle_error * 0.01 / 360.0);
        }
        if (st.freq < (sr.freq - 0.1)) osc_set_freq(st, (sr.freq - 0.1), p.Fs);
        if (st.freq > (sr.freq + 0.1)) osc_set_freq(st, (sr.freq + 0.1), p.Fs);
        double frac;
        if (osc_have_passed_point(st, p.ee, frac)) {                      // :606
            const double pt_last = frac, pt_this = 1.0 - pt_last;
            const double2 pt = make_double2(pt_this * sig2.x + pt_last * sig2_last.x, pt_this * sig2.y + pt_last * sig2_last.y);
            const double twospeed = -4.0 * ((fmod(((360.0 * sq.ptr / ((double)WTSIZE))) * 2.0 + (360.0 * p.ee * 0.5), 360.0) / 360.0) - (0.34046 + 0.4111 * p.ee));
            bool even = true;
            if (twospeed < 0) even = false;
            yui++; yui %= 2;
            if (cntr < ((128 + 128) * SPS)) { if ((even && yui == 1) || (!even && yui == 0)) { yui++; yui %= 2; } }
            if (!yui) pt_d = pt;
            else {
                const double2 pt_qpsk = make_double2(pt.x, pt_d.y);
                double ct_ec = ct_error(pt, pt_d);
                if (ct_ec > M_PI_2) ct_ec = M_PI_2;
                if (ct_ec < -M_PI_2) ct_ec = -M_PI_2;
                if (cntr > ((128 + 10) * SPS)) {                          // :641-645
                    const double ang = (1.0 * ct_ec) * 0.1;
                    rot = c_mul(rot, make_double2(cos(ang), sin(ang)));
                    rot_freq = rot_freq + ct_ec * 0.0001;
                }
                if (cntr > ((128 + 10) * SPS)) {                          // :684-689 msema MA(128)
                    const double tda = (fabs(pt_qpsk.x) - 1.0), tdb = (fabs(pt_qpsk.y) - 1.0);
                    ma_push(msema_sum, p.msema_ring[(size_t)msema_pos * cp + ch], (tda * tda) + (tdb * tdb));
                    msema_pos++; if (msema_pos >= p.msema_len) msema_pos = 0;
                    mse = msema_mean(msema_sum);
                }
                if (startstop > 0) {                                      // :692-722
                    burst_push_soft(p, ch, soft_count, soft_pending, soft_overflow, soft_byte(0.75 * pt_qpsk.y * 127.0 + 128.0));
                    burst_push_soft(p, ch, soft_count, soft_pending, soft_overflow, soft_byte(0.75 * pt_qpsk.x * 127.0 + 128.0));
                    if (soft_pending >= 32) {
                        if (!p.sql || mse < p.signalthreshold || lastmse < p.signalthreshold) soft_count += soft_pending;
                        soft_pending = 0;
                    }
                }
            }
        }
        sig2_last = sig2;                                                 // :727
        osc_next_frame(m2); osc_next_frame(st); osc_next_frame(sr); osc_next_frame(sq);
    }
    for (int k = 0; k < nt1; k++) { p.fir_re[(size_t)k * cp + ch] = s_re[k * 32 + lane]; p.fir_im[(size_t)k * cp + ch] = s_im[k * 32 + lane]; }
    BD(BD_M2_PTR) = m2.ptr; BD(BD_M2_STEP) = m2.step; BD(BD_M2_FREQ) = m2.freq; BD(BD_M2_LAST) = m2.last;
    BD(BD_ST_PTR) = st.ptr; BD(BD_ST_STEP) = st.step; BD(BD_ST_FREQ) = st.freq; BD(BD_ST_LAST) = st.last;
    BD(BD_SR_PTR) = sr.ptr; BD(BD_SR_STEP) = sr.step; BD(BD_SR_FREQ) = sr.freq; BD(BD_SR_LAST) = sr.last;
    BD(BD_SH_PTR) = sq.ptr; BD(BD_SH_STEP) = sq.step; BD(BD_SH_FREQ) = sq.freq; BD(BD_SH_LAST) = sq.last;
    BD(BD_MC_FREQ) = m2.freq;
    BD(BD_VOL_GAIN) = vol_gain; BD(BD_MSE) = mse; BD(BD_MSEMA_SUM) = msema_sum; BD(BD_ROT_FREQ) = rot_freq;
    BD(BD_ROT_RE) = rot.x; BD(BD_ROT_IM) = rot.y; BD(BD_STR_RE) = strot.x; BD(BD_STR_IM) = strot.y; BD(BD_SAV_RE) = savrot.x; BD(BD_SAV_IM) = savrot.y;
    BD(BD_EB_SUM1) = eb_sum1; BD(BD_EB_SUM2) = eb_sum2; BD(BD_EB_EBNO) = eb_ebno; BD(BD_AGC2_SUM) = agc2_sum; BD(BD_AGC2_VAL) = agc2_val;
    BD(BD_RES_X1) = res.x1; BD(BD_RES_X2) = res.x2; BD(BD_RES_Y1) = res.y1; BD(BD_RES_Y2) = res.y2;
    BD(BD_DLY_S0) = dly_s0; BD(BD_DLY41_0) = d41.d0; BD(BD_DLY41_1) = d41.d1; BD(BD_DLY41_2) = d41.d2;
    BD(BD_DLY42_0) = d42.d0; BD(BD_DLY42_1) = d42.d1; BD(BD_DLY42_2) = d42.d2; BD(BD_DLY8_0) = d8.d0; BD(BD_DLY8_1) = d8.d1; BD(BD_DLY8_2) = d8.d2;
    BD(BD_SIG2L_RE) = sig2_last.x; BD(BD_SIG2L_IM) = sig2_last.y; BD(BD_PTD_RE) = pt_d.x; BD(BD_PTD_IM) = pt_d.y;
    BD(BD_LASTMSE) = lastmse; BD(BD_LAST_EBNO_EMIT) = last_ebno_emit;
    BI(BI_CNTR) = cntr; BI(BI_STARTSTOP) = startstop; BI(BI_YUI) = yui; BI(BI_INSERTPREAMBLE) = insertpreamble;
    BI(BI_A1_POS) = a1_pos; BI(BI_MSEMA_POS) = msema_pos;
    BI(BI_SOFT_COUNT) = soft_count; BI(BI_SOFT_PENDING) = soft_pending; BI(BI_SOFT_OVERFLOW) = soft_overflow;
    BI(BI_SIG_TRUE) = sig_true; BI(BI_SIG_FALSE) = sig_false; BI(BI_EBNO_EMITS) = ebno_emits;
}

// ------------------------------------------------------------------------------------------------ launches
int hilbert_exchange_launch(const FastFir &h, const BurstParams &p, const int16_t *pcm, size_t stride, int pcm0, int i0, int i1, int fill0, cudaStream_t s)
{
    hilbert_exchange_kernel<<<(p.n_channels + 63) / 64, 64, 0, s>>>(h, p, pcm, stride, pcm0, i0, i1, fill0);
    JB_CUDA(cudaGetLastError());
    return 0;
}
int burst_front_launch(const BurstParams &p, long long sample0, int n, cudaStream_t s)
{
    JB_CUDA(cudaFuncSetAttribute(burst_front_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BF_SMEM));
    burst_front_kernel<<<(p.n_channels + BF_T - 1) / BF_T, BF_T, BF_SMEM, s>>>(p, sample0, n);
    JB_CUDA(cudaGetLastError());
    return 0;
}
int burst_trident_fft_launch(const BurstParams &p, const int *d_ev_list, int n_events, double2 *wa, double2 *wb, const double2 *tw, cudaStream_t s)
{
    trident_fft_kernel<<<2 * n_events, 1024, 0, s>>>(p, d_ev_list, n_events, wa, wb, tw);
    JB_CUDA(cudaGetLastError());
    if (p.kind == 1) trident_peaks_oqpsk_kernel<<<n_events, 1024, 0, s>>>(p, d_ev_list, n_events, wb, wa);
    else trident_peaks_kernel<<<n_events, 1024, 0, s>>>(p, d_ev_list, n_events, wb);
    JB_CUDA(cudaGetLastError());
    return 0;
}
int burst_back_launch(const BurstParams &p, long long sample0, int n, int new_write, cudaStream_t s)
{
    const size_t smem = (size_t)2 * (p.ntaps + 1) * 32 * sizeof(double);
    if (p.kind == 1) {
        burst_oqpsk_back_kernel<<<(p.n_channels + 31) / 32, 32, smem, s>>>(p, sample0, n, new_write);
        JB_CUDA(cudaGetLastError());
        return 0;
    }
    JB_CUDA(cudaFuncSetAttribute(burst_back_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    burst_back_kernel<<<(p.n_channels + 31) / 32, 32, smem, s>>>(p, n);
    JB_CUDA(cudaGetLastError());
    return 0;
}

} // namespace jb
