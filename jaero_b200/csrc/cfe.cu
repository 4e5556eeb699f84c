// K2 — batched coarse frequency estimator.
//
// Replaces CoarseFreqEstimate::ProcessBasebandData (JAERO/coarsefreqestimate.cpp:90-137) for all
// channels of a batch: out=FFT(ring) -> zero bins [startbin,stopbin] (or raised-cosine window for
// 8400) -> in=N*IFFT(out) -> in=in^2 -> out=FFT(in) -> fftshift -> y=0.9y+0.1*10log10(max(|out|,1))
// -> fold search around the expected symbol-rate lines -> freq_offset_est, plus the
// emptyingcountdown gate (:134-135) and bigchange() (:84-88).
//
// Mapping: N = n1*n2 (128x128 for 2^14, 128x64 for 2^13) four-step FFT in double precision.
// The three transforms are fused into four memory passes by pairing the steps that work on the
// same row / column of the n1 x n2 matrix:
//   P1  column FFT (over r) of the linearised ring + twiddle                       ring -> A
//   P2  row FFT (over c) -> mask/window -> row IFFT + conj twiddle                 A    -> B
//   P3  column IFFT (over k1) -> square -> column FFT (over r) + twiddle           B    -> A
//   P4  row FFT (over c) -> |.| -> 10log10 -> smoothing into y (fft-shifted)       A    -> y
//   P5  fold search + emit gate (one warp per channel)
// Each pass moves 16-row / 16-column tiles (256 B segments) through shared memory; the 16 independent
// n<=128-point FFTs of a tile run as Stockham radix-8/4 passes with the butterflies in registers. FFT rounding differs from the
// CPU oracle's radix-2 (different factorisation) at the 1e-13 level; the bin decision is integer.
#include "demod_device.cuh"
#include "fft_device.cuh"
#include <cooperative_groups.h>
#include <cstring>

namespace jb {

static const int TILE = 16;
static const int MAXN = 128;
static const int CFE_THREADS = 256;

// ---- TILE independent length-n FFTs (n = 32, 64 or 128) held in natural order in s[f][.], natural order out.
// Stockham autosort with radix-8 / radix-4 butterflies kept in registers (fft_device.cuh): 128 = 8*4*4, 64 = 8*8, 32 = 8*4, i.e.
// two or three passes over shared memory instead of log2(n) radix-2 passes. tw = W_N^k table (N = big transform), tw_stride = N/n.
template <bool INV, int R>
__device__ __forceinline__ void stockham_pass(double2 (*s)[MAXN + 1], int n, int Ns, const double2 *__restrict__ tw, int tw_stride)
{
    stockham_pass<INV, R, TILE, MAXN + 1, CFE_THREADS>(s, n, Ns, tw, tw_stride);
}

template <bool INV>
__device__ __forceinline__ void tile_fft(double2 (*s)[MAXN + 1], int n, const double2 *__restrict__ tw, int tw_stride)
{
    stockham_pass<INV, 8>(s, n, 1, tw, tw_stride);
    if (n == 128) { stockham_pass<INV, 4>(s, n, 8, tw, tw_stride); stockham_pass<INV, 4>(s, n, 32, tw, tw_stride); }
    else if (n == 64) stockham_pass<INV, 8>(s, n, 8, tw, tw_stride);
    else stockham_pass<INV, 4>(s, n, 8, tw, tw_stride);          // n == 32
}

// P1 / P3: column pass. grid = (n2/TILE, channels)
template <bool FUSED_INV_SQUARE>
__global__ void __launch_bounds__(CFE_THREADS)
cfe_col_kernel(CfePlan pl, const double2 *__restrict__ src, double2 *__restrict__ dst, size_t src_pitch, int rot, int ring_len, int ch0)
{
    __shared__ double2 s[TILE][MAXN + 1];
    const int ch = blockIdx.y;
    const int c0 = blockIdx.x * TILE;
    const int n1 = pl.n1, n2 = pl.n2, N = pl.nfft;
    const double2 *in = src + (size_t)(ch0 + ch) * src_pitch;
    double2 *out = dst + (size_t)ch * N;
    // load column tile: element (r, c0+cc) of the n1 x n2 matrix, n = n2*r + c  (rot linearises the ring:
    // bbtmpbuff[j] = bbcycbuff[(ptr+j)%N], oqpskdemodulator.cpp:418-424)
    for (int e = threadIdx.x; e < n1 * TILE; e += CFE_THREADS) {
        const int r = e / TILE, cc = e - r * TILE;
        int n = n2 * r + c0 + cc;
        if (!FUSED_INV_SQUARE) { n += rot; if (n >= ring_len) n -= ring_len; }
        s[cc][r] = in[n];
    }
    __syncthreads();
    if (FUSED_INV_SQUARE) {
        // column IFFT over k1 -> x'[n2*r+c]; square; then forward again
        tile_fft<true>(s, n1, pl.tw, N / n1);
        // square in place (natural order in, natural order out of the Stockham passes)
        for (int e = threadIdx.x; e < n1 * TILE; e += CFE_THREADS) {
            const int cc = e / n1, r = e - cc * n1;
            const double2 x = s[cc][r];
            s[cc][r] = make_double2(x.x * x.x - x.y * x.y, x.x * x.y + x.y * x.x);   // in[i]*in[i] (:103)
        }
        __syncthreads();
    }
    tile_fft<false>(s, n1, pl.tw, N / n1);
    // twiddle W_N^{c*k1} and store A[k1][c]
    for (int e = threadIdx.x; e < n1 * TILE; e += CFE_THREADS) {
        const int k1 = e / TILE, cc = e - k1 * TILE;
        const int c = c0 + cc;
        const double2 w = pl.tw[(c * k1) & (N - 1)];
        const double2 x = s[cc][k1];
        out[(size_t)k1 * n2 + c] = make_double2(x.x * w.x - x.y * w.y, x.x * w.y + x.y * w.x);
    }
}

// P2: row pass, forward -> mask -> inverse -> conj twiddle. grid = (n1/TILE, channels)
__global__ void __launch_bounds__(CFE_THREADS)
cfe_row_mask_kernel(CfePlan pl, const double2 *__restrict__ src, double2 *__restrict__ dst)
{
    __shared__ double2 s[TILE][MAXN + 1];
    const int ch = blockIdx.y;
    const int r0 = blockIdx.x * TILE;
    const int n1 = pl.n1, n2 = pl.n2, N = pl.nfft;
    const double2 *in = src + (size_t)ch * N;
    double2 *out = dst + (size_t)ch * N;
    for (int e = threadIdx.x; e < n2 * TILE; e += CFE_THREADS) {
        const int rr = e / n2, c = e - rr * n2;
        s[rr][c] = in[(size_t)(r0 + rr) * n2 + c];
    }
    __syncthreads();
    tile_fft<false>(s, n2, pl.tw, N / n2);
    // X[k1 + n1*k2] sits at s[k1-r0][k2]; mask (:99-100) in place
    for (int e = threadIdx.x; e < n2 * TILE; e += CFE_THREADS) {
        const int rr = e / n2, k2 = e - rr * n2;
        const int k = (r0 + rr) + n1 * k2;
        double2 x = s[rr][k2];
        if (!pl.is8400) { if (k >= pl.startbin && k <= pl.stopbin) x = make_double2(0.0, 0.0); }
        else { const double w = pl.window[k]; x = make_double2(x.x * w, x.y * w); }
        s[rr][k2] = x;
    }
    __syncthreads();
    tile_fft<true>(s, n2, pl.tw, N / n2);
    for (int e = threadIdx.x; e < n2 * TILE; e += CFE_THREADS) {
        const int rr = e / n2, c = e - rr * n2;
        const int k1 = r0 + rr;
        double2 w = pl.tw[(c * k1) & (N - 1)];
        w.y = -w.y;
        const double2 x = s[rr][c];
        out[(size_t)k1 * n2 + c] = make_double2(x.x * w.x - x.y * w.y, x.x * w.y + x.y * w.x);
    }
}

// P4: row pass, forward -> |.| -> log -> smoothing. grid = (n1/TILE, channels)
__global__ void __launch_bounds__(CFE_THREADS)
cfe_row_logmag_kernel(CfePlan pl, DemodParams p, const double2 *__restrict__ src, int ch0)
{
    __shared__ double2 s[TILE][MAXN + 1];
    const int ch = blockIdx.y;
    const int r0 = blockIdx.x * TILE;
    const int n1 = pl.n1, n2 = pl.n2, N = pl.nfft;
    const double2 *in = src + (size_t)ch * N;
    double *y = pl.y + (size_t)(ch0 + ch) * N;
    const bool bigchange = p.I[(size_t)I_ZERO_BB * p.cpad + ch0 + ch] != 0;     // y[i]=20 pending (coarsefreqestimate.cpp:87)
    for (int e = threadIdx.x; e < n2 * TILE; e += CFE_THREADS) {
        const int rr = e / n2, c = e - rr * n2;
        s[rr][c] = in[(size_t)(r0 + rr) * n2 + c];
    }
    __syncthreads();
    tile_fft<false>(s, n2, pl.tw, N / n2);
    // Y[k1 + n1*k2]; fftshift (:105): shifted index i = (k + N/2) % N = k1 + n1*((k2 + n2/2) % n2)
    for (int e = threadIdx.x; e < n2 * TILE; e += CFE_THREADS) {
        const int k2 = e / TILE, rr = e - k2 * TILE;         // rr fastest -> 16 consecutive i per k2
        const int k1 = r0 + rr;
        const int k2s = (k2 + (n2 >> 1)) & (n2 - 1);
        const int i = k1 + n1 * k2s;
        const double2 x = s[rr][k2];
        const double mag = hypot(x.x, x.y);
        const double yo = bigchange ? 20.0 : y[i];
        y[i] = yo * 0.9 + 0.1 * 10 * log10(fmax(mag, 1.0));                    // :108
    }
}

// P5: fold search (:112-131) + emit gate (:134-135). One warp per channel.
__global__ void __launch_bounds__(128)
cfe_search_kernel(CfePlan pl, DemodParams p)
{
    const int lane = threadIdx.x & 31;
    const int ch = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (ch >= p.n_channels) return;
    const double *y = pl.y + (size_t)ch * pl.nfft;
    const int N = pl.nfft, epb = pl.expectedpeakbin;
    double best = 0.0; int besti = 0x7fffffff;
    int i0 = pl.lo;
    if (pl.lo - epb - 1 >= 0 && pl.hi + epb + 1 < N) {
        // every index of the fold is inside the spectrum (true for all four rates): no per-bin range tests, and four
        // candidate bins per lane and round, their 24 loads requested together (the loop is load-latency bound otherwise)
        for (; i0 + 128 <= pl.hi; i0 += 128) {
            double a[4][3], c[4][3];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const int i = i0 + lane + 32 * u;
#pragma unroll
                for (int j = -1; j <= 1; j++) { a[u][j + 1] = y[i - epb - j]; c[u][j + 1] = y[i + epb + j]; }
            }
#pragma unroll
            for (int u = 0; u < 4; u++) {
                double val = 0;
#pragma unroll
                for (int j = 0; j < 3; j++) val += (a[u][j] + c[u][j]);
                if (val > best) { best = val; besti = i0 + lane + 32 * u; }   // ascending i per lane: the first maximum wins
            }
        }
    }
    for (int i = i0 + lane; i < pl.hi; i += 32) {
        if ((i < 0) || (i >= N)) continue;
        double val = 0;
        for (int j = -1; j <= 1; j++) {
            if (((i - epb - j) < 0) || ((i + epb + j) >= N)) continue;
            val += (y[i - epb - j] + y[i + epb + j]);
        }
        if (val > best) { best = val; besti = i; }           // strict >: the first maximum wins
    }
    for (int off = 16; off > 0; off >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, off);
        const int oi = __shfl_xor_sync(0xffffffffu, besti, off);
        if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
    }
    if (lane == 0) {
        const int zmaxloc = (best > 0.0) ? besti : N / 2;    // zmax starts at 0, zmaxloc at nfft/2
        const double est = -((double)(zmaxloc - N / 2)) * pl.hzperbin * 0.5;   // :131
        p.D[(size_t)D_CFE_EST * p.cpad + ch] = est;
        int &emptying = p.I[(size_t)I_EMPTYING * p.cpad + ch];
        if (emptying <= 0) p.cfe_est_out[ch] = est;
        else { emptying--; p.cfe_est_out[ch] = 0.0; }
        p.I[(size_t)I_ZERO_BB * p.cpad + ch] = 0;
    }
}

// ================================================================================================ cluster-resident estimator
// nfft = 16384 (both OQPSK modes). One thread-block cluster of 8 CTAs owns one channel at a time and keeps the whole
// 128 x 128 working matrix (256 KB of complex doubles) in the distributed shared memory of its CTAs through all three
// transforms: CTA q holds 16 columns (column passes) or 16 rows (row passes); the three layout changes are pulls from
// the peers' shared memory (DSMEM) with the four-step twiddle folded into the pull. A CTA needs 74 KB of shared memory
// and 128 threads; two clusters' CTAs share an SM, so one channel's barrier / pull latency is covered by the other's
// butterflies (a third CTA would fit the shared memory, but its 168-register cap makes the kernel spill, which measured
// slower on H100). HBM traffic per channel falls to the ring read (256 KB) plus the
// read-modify-write of y (2 x 128 KB), from eight 256 KB matrix passes before.
namespace cgx = cooperative_groups;

static const int CC_CL = 8, CC_T = 128, CC_SEQ = 16, CC_RS = 143;             // cluster size, threads, sequences per CTA, row stride
static const int CC_BUF = CC_SEQ * CC_RS * 16;                                // one working buffer (bytes)
static const int CC_TW2 = 128, CC_TW3 = 152;                                  // offsets (in double2) of the per-pass twiddle copies
static const int CC_SM_TOTAL = 2 * CC_BUF + (128 + 24 + 32) * 16;

__device__ __forceinline__ int cc_ph(int e) { return e + (e >> 3); }          // padded position inside a 128-point sequence

// log10 for finite x >= 1 (the argument is max(|X|^2, 1)): fdlibm's log kernel — x = 2^k m, m in [sqrt(1/2), sqrt(2)),
// s = (m-1)/(m+1), degree-14 polynomial in s — with the quotient by div_fast and the final scaling split as in fdlibm's
// e_log10.c. Within 2 ulp of glibc's log10 over [1, DBL_MAX] as this unit compiles it, with contraction, exactly k at 10^k
// (tests/test_gpu_math.py; host twin without contraction: tools/micro/log10_test.c; the library call it replaces is itself
// only specified to 1 ulp), about half the instructions; the smoothed spectrum feeds an arg-max over
// sums of six bins, where differences of that size cannot matter unless the library's own rounding would.
__device__ __forceinline__ double log10_ge1(double x)
{
    const double Lg1 = 6.666666666666735130e-01, Lg2 = 3.999999999940941908e-01, Lg3 = 2.857142874366239149e-01, Lg4 = 2.222219843214978396e-01,
                 Lg5 = 1.818357216161805012e-01, Lg6 = 1.531383769920937332e-01, Lg7 = 1.479819860511658591e-01;
    const double ivln10 = 4.34294481903251816668e-01, log10_2hi = 3.01029995663611771306e-01, log10_2lo = 3.69423907715893078616e-13;
    int hi = __double2hiint(x);
    const int lo = __double2loint(x);
    int k = (hi >> 20) - 1023;
    hi &= 0x000fffff;
    const int i = (hi + 0x95f64) & 0x100000;                 // m >= sqrt(2): halve it
    hi |= (i ^ 0x3ff00000);
    k += (i >> 20);
    const double f = __hiloint2double(hi, lo) - 1.0;
    const double s = div_fast(f, 2.0 + f);
    const double z = s * s, w = z * z;
    const double t1 = w * (Lg2 + w * (Lg4 + w * Lg6));
    const double t2 = z * (Lg1 + w * (Lg3 + w * (Lg5 + w * Lg7)));
    const double hfsq = 0.5 * f * f;
    const double lg = f - (hfsq - s * (hfsq + (t2 + t1)));
    const double dk = (double)k;
    return (dk * log10_2lo + ivln10 * lg) + dk * log10_2hi;
}

// 16 x FFT-128 (same factorisation and arithmetic as tile_fft for n = 128: Stockham radix 8, 4, 4), with the passes after the
// first one in registers. Pass 2 (radix 4, Ns = 8) butterfly 8m + k writes positions 32m + k + 8t and pass 3 (radix 4, Ns = 32)
// butterfly k + 8u reads positions k + 8u + 32i: for each k in 0..7 both passes close over the 16 positions k + 8p of the
// sequence. Lane k of sequence f = threadIdx.x >> 3 holds those 16 values (x[p] = position k + 8p) and runs both passes without
// touching shared memory; a warp owns four whole sequences, so only __syncwarp() orders lanes of a sequence. Pass 3 leaves
// position k + 8p in x[p] again, and those are the inputs of the next transform's first-pass (radix 8, Ns = 1) butterflies
// k (positions k + 16t = x[2t]) and k + 8 (x[2t + 1]): a transform chained to another is stored once, after that first pass.
// The first pass of a transform that starts from the ring or from the peers' buffers runs from the registers of the load /
// pull, whose eight values are exactly one butterfly's inputs.
__device__ __forceinline__ void cc_load16(const double2 *row, int k, double2 (&x)[16])
{
#pragma unroll
    for (int p = 0; p < 16; p++) x[p] = row[cc_ph(k + 8 * p)];
}

__device__ __forceinline__ void cc_store16(double2 *row, int k, const double2 (&x)[16])
{
#pragma unroll
    for (int p = 0; p < 16; p++) row[cc_ph(k + 8 * p)] = x[p];
}

template <bool INV>
__device__ __forceinline__ void cc_pass23(double2 (&x)[16], int k, const double2 *__restrict__ tws)
{
    // The twiddles of a pass depend on the lane only. Read straight from the 128-entry table the second pass's strides
    // (4k, 8k, 12k) put a quarter-warp's eight 16-byte loads on two, one and two bank groups (4-, 8- and 4-way conflicts) and
    // the third pass's 2l on four (2-way); the kernel keeps compact copies instead: tws[CC_TW2 + 8(m-1) + k] = W^(4mk),
    // tws[CC_TW3 + l] = W^(2l). Same table values, so the arithmetic is unchanged.
    auto radix4 = [](double2 &v0, double2 &v1, double2 &v2, double2 &v3, double2 w1, double2 w2, double2 w3) {
        if (INV) { w1.y = -w1.y; w2.y = -w2.y; w3.y = -w3.y; }
        v1 = c_mul(v1, w1); v2 = c_mul(v2, w2); v3 = c_mul(v3, w3);
        dft4<INV>(v0, v1, v2, v3);
    };
    double2 y[16];
    {   // radix 4, Ns = 8: butterfly 8m + k reads positions k + 8(m + 4t), writes k + 8(4m + t)
        const double2 w1 = tws[CC_TW2 + k], w2 = tws[CC_TW2 + 8 + k], w3 = tws[CC_TW2 + 16 + k];
#pragma unroll
        for (int m = 0; m < 4; m++) {
            double2 v0 = x[m], v1 = x[m + 4], v2 = x[m + 8], v3 = x[m + 12];
            radix4(v0, v1, v2, v3, w1, w2, w3);
            y[4 * m] = v0; y[4 * m + 1] = v1; y[4 * m + 2] = v2; y[4 * m + 3] = v3;
        }
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {   // radix 4, Ns = 32: butterfly l = k + 8u reads and writes positions k + 8(u + 4i)
        const int l = k + 8 * u;
        double2 v0 = y[u], v1 = y[u + 4], v2 = y[u + 8], v3 = y[u + 12];
        radix4(v0, v1, v2, v3, tws[l], tws[CC_TW3 + l], tws[3 * l]);
        x[u] = v0; x[u + 4] = v1; x[u + 8] = v2; x[u + 12] = v3;
    }
}

// the next transform's first pass from pass 3's registers: butterflies k and k + 8, stored in place as row[8j + t]
template <bool INV>
__device__ __forceinline__ void cc_pass1_store(const double2 (&x)[16], double2 *row, int k)
{
    double2 a[8], b[8];
#pragma unroll
    for (int t = 0; t < 8; t++) { a[t] = x[2 * t]; b[t] = x[2 * t + 1]; }
    dft8<INV>(a);
    dft8<INV>(b);
    __syncwarp();                          // the sequence's other lanes have read their 16 values
#pragma unroll
    for (int t = 0; t < 8; t++) { row[cc_ph(8 * k + t)] = a[t]; row[cc_ph(8 * k + 64 + t)] = b[t]; }
    __syncwarp();
}

__global__ void __launch_bounds__(CC_T, 2)
cfe_cluster_kernel(CfePlan pl, DemodParams p, int oldest)
{
    extern __shared__ __align__(128) unsigned char cc_smem[];
    double2 *bufA = reinterpret_cast<double2 *>(cc_smem);
    double2 *bufB = reinterpret_cast<double2 *>(cc_smem + CC_BUF);
    double2 *tws = reinterpret_cast<double2 *>(cc_smem + 2 * CC_BUF);
    cgx::cluster_group cluster = cgx::this_cluster();
    const int q = (int)cluster.block_rank();
    const int n_clusters = gridDim.x / CC_CL, cid = blockIdx.x / CC_CL;
    const int N = 16384, ring_len = p.bb_len;
    const double2 *__restrict__ twN = pl.tw;
    for (int t = threadIdx.x; t < 128 + 24 + 32; t += CC_T) {
        if (t < 128) tws[t] = twN[t * (N / 128)];
        else if (t < 128 + 24) { const int e = t - 128, m = e >> 3, k = e & 7; tws[CC_TW2 + e] = twN[(4 * (m + 1) * k) * (N / 128)]; }
        else { const int l = t - 152; tws[CC_TW3 + l] = twN[(2 * l) * (N / 128)]; }
    }
    // The four-step twiddles W_N^(c*k1) are read from the same table the reference-order transforms use (a product of two
    // smaller tables breaks the exact conjugate symmetry of the table and with it the estimator's tie-breaks on symmetric
    // spectra). Their indices do not depend on the data, so the loads are issued ahead of the cluster barrier they follow.
    __syncthreads();
    bool arrived = false;
    cluster.sync();                        // every CTA of the cluster is resident before the first remote access
    const int f = threadIdx.x >> 3, k = threadIdx.x & 7;                    // lane k of sequence f in the passes after the first
    double2 *const rowA = bufA + f * CC_RS, *const rowB = bufB + f * CC_RS;
    for (int ch = cid; ch < p.n_channels; ch += n_clusters) {
        double2 x[16];
        // ---- this CTA's 16 columns of the linearised ring (oqpskdemodulator.cpp:418-424) -> A[cc][r]: 256 B runs per r
        double2 colv[2][8];
        {
            const double2 *ring = p.bb + (size_t)ch * ring_len;
            const int cc = threadIdx.x & 15, r0i = threadIdx.x >> 4;
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    int n = oldest + 128 * (r0i + 8 * h + 16 * i) + 16 * q + cc;
                    if (n >= ring_len) n -= ring_len;
                    if (n >= ring_len) n -= ring_len;
                    colv[h][i] = ring[n];
                }
        }
        // ---- P1: column FFT over r                                                   A[cc][k1]
        // this thread's samples r = r0i + 8h + 16 i of column cc are butterflies r0i and r0i + 8 of the first pass
        dft8<false>(colv[0]);
        dft8<false>(colv[1]);
        if (arrived) { cluster.barrier_wait(); arrived = false; }   // the peers have pulled the previous channel's P3 result out of A
        {
            const int cc = threadIdx.x & 15, r0i = threadIdx.x >> 4;
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
                for (int i = 0; i < 8; i++) bufA[cc * CC_RS + cc_ph(8 * (r0i + 8 * h) + i)] = colv[h][i];
        }
        __syncthreads();
        cc_load16(rowA, k, x);
        cc_pass23<false>(x, k, tws);
        cc_store16(rowA, k, x);
        double2 tw8[2][8];
        {
            const int kk = threadIdx.x & 15, cc = threadIdx.x >> 4;
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
                for (int s = 0; s < 8; s++) tw8[h][s] = __ldg(&twN[((16 * s + cc + 8 * h) * (16 * q + kk)) & (N - 1)]);
        }
        cluster.sync();
        // rows k1 = 16q+kk, all c: B[kk][c] = A_src[cc][k1] * W_N^{c k1}   (kk fastest: contiguous remote reads)
        {
            const int kk = threadIdx.x & 15;
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int cc = (threadIdx.x >> 4) + 8 * h;
                double2 v[8];
#pragma unroll
                for (int s = 0; s < 8; s++) v[s] = c_mul(cluster.map_shared_rank(bufA, s)[cc * CC_RS + cc_ph(16 * q + kk)], tw8[h][s]);
                dft8<false>(v);            // c = cc + 16 s: butterfly cc of row kk's first pass
#pragma unroll
                for (int s = 0; s < 8; s++) bufB[kk * CC_RS + cc_ph(8 * cc + s)] = v[s];
            }
        }
        __syncthreads();
        // ---- P2: row FFT over c -> mask (:99-100) -> row IFFT, in place               B[kk][c]
        cc_load16(rowB, k, x);
        cc_pass23<false>(x, k, tws);
#pragma unroll
        for (int e = 0; e < 16; e++) {
            const int bin = (16 * q + f) + 128 * (k + 8 * e);  // X[k1 + n1*k2]
            if (!pl.is8400) { if (bin >= pl.startbin && bin <= pl.stopbin) x[e] = make_double2(0.0, 0.0); }
            else {
                // the product is rounded on its own (it must not be contracted into the inverse butterflies' adds)
                const double w = pl.window[bin];
                x[e] = make_double2(__dmul_rn(x[e].x, w), __dmul_rn(x[e].y, w));
            }
        }
        cc_pass1_store<true>(x, rowB, k);
        cc_load16(rowB, k, x);
        cc_pass23<true>(x, k, tws);
        cc_store16(rowB, k, x);
        {
            const int cc = threadIdx.x & 15, kk = threadIdx.x >> 4;
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
                for (int s = 0; s < 8; s++) tw8[h][s] = __ldg(&twN[((16 * q + cc) * (16 * s + kk + 8 * h)) & (N - 1)]);
        }
        cluster.sync();                    // every peer has finished reading A (it passed the pull above before its own P2)
        // columns c = 16q+cc, all k1: A[cc][k1] = B_src[kk][c] * conj(W_N^{c k1})   (cc fastest: contiguous remote reads)
        {
            const int cc = threadIdx.x & 15;
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int kk = (threadIdx.x >> 4) + 8 * h;
                double2 v[8];
#pragma unroll
                for (int s = 0; s < 8; s++) {
                    double2 w = tw8[h][s]; w.y = -w.y;
                    v[s] = c_mul(cluster.map_shared_rank(bufB, s)[kk * CC_RS + cc_ph(16 * q + cc)], w);
                }
                dft8<true>(v);             // k1 = kk + 16 s: butterfly kk of column cc's first pass
#pragma unroll
                for (int s = 0; s < 8; s++) bufA[cc * CC_RS + cc_ph(8 * kk + s)] = v[s];
            }
        }
        __syncthreads();
        // ---- P3: column IFFT over k1 -> square (:103) -> column FFT over r, in place  A[cc][k1]
        cc_load16(rowA, k, x);
        cc_pass23<true>(x, k, tws);
#pragma unroll
        for (int e = 0; e < 16; e++) x[e] = make_double2(x[e].x * x[e].x - x[e].y * x[e].y, x[e].x * x[e].y + x[e].y * x[e].x);
        cc_pass1_store<false>(x, rowA, k);
        cc_load16(rowA, k, x);
        cc_pass23<false>(x, k, tws);
        cc_store16(rowA, k, x);
        {
            const int kk = threadIdx.x & 15, cc = threadIdx.x >> 4;
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
                for (int s = 0; s < 8; s++) tw8[h][s] = __ldg(&twN[((16 * s + cc + 8 * h) * (16 * q + kk)) & (N - 1)]);
        }
        cluster.sync();
        {
            const int kk = threadIdx.x & 15;
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int cc = (threadIdx.x >> 4) + 8 * h;
                double2 v[8];
#pragma unroll
                for (int s = 0; s < 8; s++) v[s] = c_mul(cluster.map_shared_rank(bufA, s)[cc * CC_RS + cc_ph(16 * q + kk)], tw8[h][s]);
                dft8<false>(v);
#pragma unroll
                for (int s = 0; s < 8; s++) bufB[kk * CC_RS + cc_ph(8 * cc + s)] = v[s];
            }
        }
        cluster.barrier_arrive();          // split barrier: this CTA is done reading its peers' A (waited on before A is refilled)
        arrived = true;
        __syncthreads();
        // ---- P4: row FFT over c -> |.| -> 10 log10 -> smoothing into y (:105-108)      B
        {
            double *y = pl.y + (size_t)ch * N;
            const bool bigchange = p.I[(size_t)I_ZERO_BB * p.cpad + ch] != 0;     // y[i]=20 pending (coarsefreqestimate.cpp:87)
            // y is only ever read by the fold search, for bins within [lo-epb-1, hi+epb+1] (coarsefreqestimate.cpp:112-130):
            // bins outside that window are neither loaded, evaluated (log10) nor stored. Y[k1 + n1*k2] with k1 = 16q + f and
            // k2 = k + 8e; fftshift (:105): i = k1 + n1*((k2 + n2/2) % n2). The four sequences of a warp fill 32-byte sectors.
            const int need_lo = pl.lo - pl.expectedpeakbin - 1, need_hi = pl.hi + pl.expectedpeakbin + 1;
            double yo[16];                                                        // requested before the transform, consumed after it
#pragma unroll
            for (int e = 0; e < 16; e++) {
                const int i_sh = (16 * q + f) + 128 * ((k + 8 * e + 64) & 127);
                yo[e] = (bigchange || i_sh < need_lo || i_sh > need_hi) ? 20.0 : y[i_sh];
            }
            cc_load16(rowB, k, x);
            cc_pass23<false>(x, k, tws);
#pragma unroll
            for (int e = 0; e < 16; e++) {
                const int i_sh = (16 * q + f) + 128 * ((k + 8 * e + 64) & 127);
                if (i_sh < need_lo || i_sh > need_hi) continue;
                // 10*log10(max(|x|,1)) = 5*log10(max(|x|^2,1))
                y[i_sh] = yo[e] * 0.9 + 0.1 * 5 * log10_ge1(fmax(x[e].x * x[e].x + x[e].y * x[e].y, 1.0));   // :108
            }
        }
        __syncthreads();
    }
    if (arrived) cluster.barrier_wait();
    cluster.sync();                        // no CTA leaves while a peer may still read its shared memory
}

int cfe_cluster_run(const CfePlan &pl, const DemodParams &p, int oldest, int n_clusters, cudaStream_t s, long long *launches)
{
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.gridDim = dim3((unsigned)(n_clusters * CC_CL)); cfg.blockDim = dim3(CC_T); cfg.dynamicSmemBytes = CC_SM_TOTAL; cfg.stream = s;
    cudaLaunchAttribute at; at.id = cudaLaunchAttributeClusterDimension; at.val.clusterDim.x = CC_CL; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
    cfg.attrs = &at; cfg.numAttrs = 1;
    JB_CUDA(cudaLaunchKernelEx(&cfg, cfe_cluster_kernel, pl, p, oldest));
    cfe_search_kernel<<<(p.n_channels + 3) / 4, 128, 0, s>>>(pl, p);
    JB_CUDA(cudaGetLastError());
    *launches += 2;
    return 0;
}
// number of clusters that can be co-resident (0: the device cannot run the cluster kernel)
int cfe_cluster_capacity()
{
    if (cudaFuncSetAttribute(cfe_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CC_SM_TOTAL) != cudaSuccess) { cudaGetLastError(); return 0; }
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.gridDim = dim3(CC_CL * 64); cfg.blockDim = dim3(CC_T); cfg.dynamicSmemBytes = CC_SM_TOTAL;
    cudaLaunchAttribute at; at.id = cudaLaunchAttributeClusterDimension; at.val.clusterDim.x = CC_CL; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
    cfg.attrs = &at; cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, cfe_cluster_kernel, &cfg) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

// `oldest` = ring index of the oldest sample (the linearisation origin, oqpskdemodulator.cpp:418-424)
int cfe_run(const CfePlan &pl, const DemodParams &p, int oldest, cudaStream_t s, long long *launches)
{
    const int C = p.n_channels;
    for (int ch0 = 0; ch0 < C; ch0 += pl.group) {
        const int g = (C - ch0 < pl.group) ? C - ch0 : pl.group;
        dim3 gc(pl.n2 / TILE, g), gr(pl.n1 / TILE, g);
        cfe_col_kernel<false><<<gc, CFE_THREADS, 0, s>>>(pl, p.bb, pl.work_a, (size_t)p.bb_len, oldest, p.bb_len, ch0);
        cfe_row_mask_kernel<<<gr, CFE_THREADS, 0, s>>>(pl, pl.work_a, pl.work_b);
        cfe_col_kernel<true><<<gc, CFE_THREADS, 0, s>>>(pl, pl.work_b, pl.work_a, (size_t)pl.nfft, 0, pl.nfft, 0);
        cfe_row_logmag_kernel<<<gr, CFE_THREADS, 0, s>>>(pl, p, pl.work_a, ch0);
        *launches += 4;
    }
    cfe_search_kernel<<<(C + 3) / 4, 128, 0, s>>>(pl, p);
    *launches += 1;
    JB_CUDA(cudaGetLastError());
    return 0;
}

} // namespace jb

// ---- test support (jaero_probe_math): log10_ge1 and div_fast as this unit compiles them (without -fmad=false)
#include "../../include/jaero_b200.h"

namespace jb {

__global__ void probe_math_cfe_kernel(int op, size_t n, const double *__restrict__ a, const double *__restrict__ b, double *__restrict__ out)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        out[i] = op == JAERO_MATH_LOG10_GE1 ? log10_ge1(a[i]) : div_fast(a[i], b[i]);
}

int probe_math_cfe_launch(int op, size_t n, const double *a, const double *b, double *out, cudaStream_t s)
{
    const size_t blocks = (n + 255) / 256;
    probe_math_cfe_kernel<<<(unsigned)(blocks < 4096 ? blocks : 4096), 256, 0, s>>>(op, n, a, b, out);
    JB_CUDA(cudaGetLastError());
    return 0;
}

} // namespace jb
