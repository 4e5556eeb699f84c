// Mode identifier: averaged power spectrum of each PCM channel's squared analytic signal (include/jaero_b200.h states the
// contract, jaero_ident_create). Squaring an MSK or OQPSK carrier at fc leaves two lines at 2 fc +- fb / 2; the host classifier
// finds them in this spectrum.
//
// Every frame that a write completes goes through three FP64 transforms of nfft = n1 x n2 points (n1 = n2 = 128 at 2^14), each a
// four-step FFT whose two halves run in different kernels. The inverse of the second transform starts from the forward's
// transposed output, so each kernel boundary falls where a transform changes from columns to rows or back:
//   load    per CTA 16 columns c: x[n2 r + c] w[n2 r + c] / 32768, n1-point FFT over r, twiddle W_N^(c k1)       -> w0[k1][c]
//   mask    per CTA 16 rows k1: n2-point FFT over c -> X[k1 + n1 k2]; A = X 2/N for 0 < k < N/2, else 0;
//           inverse n2-point FFT over k2, twiddle W_N^(-c k1)                                                      -> w1[k1][c]
//   square  per CTA 16 columns c: inverse n1-point FFT over k1 -> a[n2 r + c]; a^2; n1-point FFT over r;
//           twiddle W_N^(c k1)                                                                                     -> w0[k1][c]
//   power   per CTA 16 rows k1: n2-point FFT over c -> Y[k1 + n1 k2]; |Y|^2 / (sum w^2)^2 at its fftshift index -> pw[g][i]
//   acc     one thread per (channel, bin): sum[c][i] += pw[g][i] over the pass's frames of channel c, in frame order
// The pass's work matrices (IDENT_PASS_ELEMS frame bins, 2 x 16 MB; pw reuses w1) stay in L2 between kernels. Every frame takes
// the same instructions wherever it sits in a pass, and each channel's sum is one sequence of additions in frame order, so the
// result does not depend on how the stream is cut into writes, nor on the batch's other channels.
#include "ident.cuh"
#include "fft_device.cuh"
#include "common.cuh"
#include <algorithm>

namespace jb {

typedef double2 IdentRow[IDENT_MAXN + 1];

template <bool INV>
__device__ __forceinline__ void ident_tile_fft(IdentRow *s, int n, const double2 *__restrict__ tw, int tw_stride)
{
    tile_fft<INV, IDENT_TILE, IDENT_MAXN, IDENT_THREADS>(s, n, tw, tw_stride);
}
__device__ __forceinline__ void ident_store_cols(const IdentPlan &p, IdentRow *s, int c0, double2 *__restrict__ out)
{
    store_cols_twiddled<IDENT_TILE, IDENT_MAXN + 1, IDENT_THREADS>(s, p.n1, p.n2, p.nfft, c0, p.tw, out);
}

// grid (n2 / IDENT_TILE, frames of the pass); pass item j0 + blockIdx.y is frame f0 + (j mod F) of channel j / F
__global__ void __launch_bounds__(IDENT_THREADS) ident_load_kernel(IdentPlan p, const int16_t *__restrict__ xs, size_t pitch, long long x0,
                                                                   long long f0, long long F, long long j0, double2 *__restrict__ w0)
{
    extern __shared__ double2 ident_smem[];
    IdentRow *s = reinterpret_cast<IdentRow *>(ident_smem);
    const int n1 = p.n1, n2 = p.n2;
    const int c0 = blockIdx.x * IDENT_TILE;
    const long long j = j0 + blockIdx.y, ch = j / F;
    const int16_t *x = xs + ch * pitch + ((f0 + (j - ch * F)) * p.hop - x0);
    for (int e = threadIdx.x; e < n1 * IDENT_TILE; e += IDENT_THREADS) {
        const int r = e / IDENT_TILE, cc = e - r * IDENT_TILE;
        const int n = n2 * r + c0 + cc;
        s[cc][r] = make_double2((double)x[n] * (1.0 / 32768.0) * __ldg(p.win + n), 0.0);
    }
    __syncthreads();
    ident_tile_fft<false>(s, n1, p.tw, p.nfft / n1);
    ident_store_cols(p, s, c0, w0 + (size_t)blockIdx.y * p.nfft);
}

// grid (n1 / IDENT_TILE, frames of the pass)
__global__ void __launch_bounds__(IDENT_THREADS) ident_mask_kernel(IdentPlan p, const double2 *__restrict__ w0, double2 *__restrict__ w1)
{
    extern __shared__ double2 ident_smem[];
    IdentRow *s = reinterpret_cast<IdentRow *>(ident_smem);
    const int n1 = p.n1, n2 = p.n2, N = p.nfft;
    const int r0 = blockIdx.x * IDENT_TILE;
    load_rows<IDENT_TILE, IDENT_MAXN + 1, IDENT_THREADS>(s, n2, r0, w0 + (size_t)blockIdx.y * N);
    __syncthreads();
    ident_tile_fft<false>(s, n2, p.tw, N / n2);
    // X[k1 + n1 k2] sits at s[k1 - r0][k2]. 2/N is a power of two, so folding the inverse's 1/N in here rounds nothing.
    const double g = 2.0 / N;
    for (int e = threadIdx.x; e < n2 * IDENT_TILE; e += IDENT_THREADS) {
        const int rr = e / n2, k2 = e - rr * n2;
        const int k = r0 + rr + n1 * k2;
        const double2 v = s[rr][k2];
        s[rr][k2] = (k > 0 && k < (N >> 1)) ? make_double2(v.x * g, v.y * g) : make_double2(0.0, 0.0);
    }
    __syncthreads();
    ident_tile_fft<true>(s, n2, p.tw, N / n2);
    double2 *out = w1 + (size_t)blockIdx.y * N;
    for (int e = threadIdx.x; e < n2 * IDENT_TILE; e += IDENT_THREADS) {
        const int rr = e / n2, c = e - rr * n2;
        const int k1 = r0 + rr;
        const double2 t = __ldg(p.tw + ((c * k1) & (N - 1)));
        out[(size_t)k1 * n2 + c] = c_mul(s[rr][c], make_double2(t.x, -t.y));
    }
}

// grid (n2 / IDENT_TILE, frames of the pass)
__global__ void __launch_bounds__(IDENT_THREADS) ident_square_kernel(IdentPlan p, const double2 *__restrict__ w1, double2 *__restrict__ w0)
{
    extern __shared__ double2 ident_smem[];
    IdentRow *s = reinterpret_cast<IdentRow *>(ident_smem);
    const int n1 = p.n1, n2 = p.n2, N = p.nfft;
    const int c0 = blockIdx.x * IDENT_TILE;
    const double2 *in = w1 + (size_t)blockIdx.y * N;
    for (int e = threadIdx.x; e < n1 * IDENT_TILE; e += IDENT_THREADS) {
        const int k1 = e / IDENT_TILE, cc = e - k1 * IDENT_TILE;
        s[cc][k1] = in[(size_t)k1 * n2 + c0 + cc];
    }
    __syncthreads();
    ident_tile_fft<true>(s, n1, p.tw, N / n1);
    // s[c - c0][r] = a[n2 r + c]
    for (int e = threadIdx.x; e < n1 * IDENT_TILE; e += IDENT_THREADS) {
        const int cc = e / n1, r = e - cc * n1;
        const double2 v = s[cc][r];
        s[cc][r] = make_double2(v.x * v.x - v.y * v.y, 2.0 * v.x * v.y);
    }
    __syncthreads();
    ident_tile_fft<false>(s, n1, p.tw, N / n1);
    ident_store_cols(p, s, c0, w0 + (size_t)blockIdx.y * N);
}

// grid (n1 / IDENT_TILE, frames of the pass)
__global__ void __launch_bounds__(IDENT_THREADS) ident_power_kernel(IdentPlan p, const double2 *__restrict__ w0, double *__restrict__ pw)
{
    extern __shared__ double2 ident_smem[];
    IdentRow *s = reinterpret_cast<IdentRow *>(ident_smem);
    const int n1 = p.n1, n2 = p.n2, N = p.nfft;
    const int r0 = blockIdx.x * IDENT_TILE;
    load_rows<IDENT_TILE, IDENT_MAXN + 1, IDENT_THREADS>(s, n2, r0, w0 + (size_t)blockIdx.y * N);
    __syncthreads();
    ident_tile_fft<false>(s, n2, p.tw, N / n2);
    store_power_shifted<IDENT_TILE, IDENT_MAXN + 1, IDENT_THREADS>(s, n1, n2, r0, p.inv_wss2, pw + (size_t)blockIdx.y * N);
}

// grid (nfft / 256, channels the pass touches); pw row g is pass item j0 + g
__global__ void ident_accumulate_kernel(IdentPlan p, const double *__restrict__ pw, long long F, long long j0, int g)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.nfft) return;
    const long long ch = j0 / F + blockIdx.y;
    const long long a = max(j0, ch * F), b = min(j0 + g, (ch + 1) * F);
    double *sum = p.sum + ch * p.nfft + i;
    double s = *sum;
    for (long long j = a; j < b; j++) s += pw[(size_t)(j - j0) * p.nfft + i];
    *sum = s;
}

int ident_frames(const IdentPlan &p, const int16_t *xs, size_t pitch, long long x0, long long f0, long long F, int G, double2 *w0,
                 double2 *w1, cudaStream_t st, long long *launches)
{
    static_assert(IDENT_SMEM <= 48 * 1024, "the tile fits the default dynamic shared-memory limit");
    const long long total = (long long)p.n_channels * F;
    for (long long a = 0; a < total; a += G) {
        const int g = (int)std::min<long long>(G, total - a);
        const int nch = (int)((a + g - 1) / F - a / F + 1);
        ident_load_kernel<<<dim3(p.n2 / IDENT_TILE, g), IDENT_THREADS, IDENT_SMEM, st>>>(p, xs, pitch, x0, f0, F, a, w0);
        ident_mask_kernel<<<dim3(p.n1 / IDENT_TILE, g), IDENT_THREADS, IDENT_SMEM, st>>>(p, w0, w1);
        ident_square_kernel<<<dim3(p.n2 / IDENT_TILE, g), IDENT_THREADS, IDENT_SMEM, st>>>(p, w1, w0);
        ident_power_kernel<<<dim3(p.n1 / IDENT_TILE, g), IDENT_THREADS, IDENT_SMEM, st>>>(p, w0, reinterpret_cast<double *>(w1));
        ident_accumulate_kernel<<<dim3((p.nfft + 255) / 256, nch), 256, 0, st>>>(p, reinterpret_cast<const double *>(w1), F, a, g);
        JB_CUDA(cudaGetLastError());
        *launches += 5;
    }
    return 0;
}

} // namespace jb
