// Wideband carrier scanner: averaged and max-held power spectrum of one complex IQ stream (include/jaero_b200.h states the
// contract, jaero_scan_create).
//
// Every frame that a write completes is windowed and transformed by a four-step FP64 FFT, nfft = n1 x n2 (n1 = n2 = 256 at 2^16):
//   col   per CTA 16 columns of up to SCAN_TILE frames' n1 x n2 matrices: load x[f hop + n2 r + c] w[n2 r + c] (256 B segments),
//         n1-point Stockham FFT over r in shared memory, twiddle W_N^(c k1), store A[f][k1][c]
//   row   per CTA 16 rows: n2-point FFT over c -> X[k1 + n1 k2]; |X|^2 / sum w^2 stored at its fftshift index into pw[f][i]
//   acc   one thread per bin: sum[i] += pw[f][i], maxh[i] = max(maxh[i], pw[f][i]) for f in frame order
// The work matrix of one pass (SCAN_PASS_ELEMS frame bins, 48 MB) is written and read back while it is still in L2. Accumulating
// per bin in frame order makes the running sum the same sequence of additions however the stream is cut into writes.
#include "scan.cuh"
#include "ddc.cuh"
#include "fft_device.cuh"
#include "common.cuh"
#include <algorithm>

namespace jb {

typedef double2 ScanRow[SCAN_MAXN + 1];

__device__ __forceinline__ void scan_tile_fft(ScanRow *s, int n, const double2 *__restrict__ tw, int tw_stride)
{
    tile_fft<false, SCAN_TILE, SCAN_MAXN, SCAN_THREADS>(s, n, tw, tw_stride);
}

__global__ void scan_convert_kernel(const void *raw, int format, long long n, double2 *xd)
{
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        xd[i] = iq_sample(raw, i, format);
}

// grid (n2 / SCAN_TILE, frames of the pass)
__global__ void __launch_bounds__(SCAN_THREADS) scan_col_kernel(ScanPlan p, const double2 *__restrict__ xd, long long x0, long long f0,
                                                                double2 *__restrict__ work)
{
    extern __shared__ double2 scan_smem[];
    ScanRow *s = reinterpret_cast<ScanRow *>(scan_smem);
    const int n1 = p.n1, n2 = p.n2, N = p.nfft;
    const int c0 = blockIdx.x * SCAN_TILE;
    const double2 *x = xd + ((f0 + blockIdx.y) * p.hop - x0);
    for (int e = threadIdx.x; e < n1 * SCAN_TILE; e += SCAN_THREADS) {
        const int r = e / SCAN_TILE, cc = e - r * SCAN_TILE;
        const int n = n2 * r + c0 + cc;
        const double2 v = x[n];
        const double w = __ldg(p.win + n);
        s[cc][r] = make_double2(v.x * w, v.y * w);
    }
    __syncthreads();
    scan_tile_fft(s, n1, p.tw, N / n1);
    store_cols_twiddled<SCAN_TILE, SCAN_MAXN + 1, SCAN_THREADS>(s, n1, n2, N, c0, p.tw, work + (size_t)blockIdx.y * N);
}

// grid (n1 / SCAN_TILE, frames of the pass)
__global__ void __launch_bounds__(SCAN_THREADS) scan_row_kernel(ScanPlan p, const double2 *__restrict__ work, double *__restrict__ pw)
{
    extern __shared__ double2 scan_smem[];
    ScanRow *s = reinterpret_cast<ScanRow *>(scan_smem);
    const int n1 = p.n1, n2 = p.n2, N = p.nfft;
    const int r0 = blockIdx.x * SCAN_TILE;
    load_rows<SCAN_TILE, SCAN_MAXN + 1, SCAN_THREADS>(s, n2, r0, work + (size_t)blockIdx.y * N);
    __syncthreads();
    scan_tile_fft(s, n2, p.tw, N / n2);
    store_power_shifted<SCAN_TILE, SCAN_MAXN + 1, SCAN_THREADS>(s, n1, n2, r0, p.inv_wss, pw + (size_t)blockIdx.y * N);
}

__global__ void scan_accumulate_kernel(ScanPlan p, const double *__restrict__ pw, int F)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.nfft) return;
    double s = p.sum[i], m = p.maxh[i];
#pragma unroll 8
    for (int f = 0; f < F; f++) {
        const double v = pw[(size_t)f * p.nfft + i];
        s += v;
        m = fmax(m, v);
    }
    p.sum[i] = s;
    p.maxh[i] = m;
}

int scan_convert(const void *d_iq, int format, long long n, double2 *xd, cudaStream_t st, long long *launches)
{
    const int grid = (int)std::min<long long>((n + 255) / 256, 4L * 132 * 16);
    scan_convert_kernel<<<grid, 256, 0, st>>>(d_iq, format, n, xd);
    JB_CUDA(cudaGetLastError());
    ++*launches;
    return 0;
}

int scan_frames(const ScanPlan &p, const double2 *xd, long long x0, long long f0, long long F, int G, double2 *work, double *pw,
                cudaStream_t st, long long *launches)
{
    JB_CUDA(cudaFuncSetAttribute(scan_col_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SCAN_SMEM));
    JB_CUDA(cudaFuncSetAttribute(scan_row_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SCAN_SMEM));
    for (long long a = 0; a < F; a += G) {
        const int g = (int)std::min<long long>(G, F - a);
        scan_col_kernel<<<dim3(p.n2 / SCAN_TILE, g), SCAN_THREADS, SCAN_SMEM, st>>>(p, xd, x0, f0 + a, work);
        scan_row_kernel<<<dim3(p.n1 / SCAN_TILE, g), SCAN_THREADS, SCAN_SMEM, st>>>(p, work, pw);
        scan_accumulate_kernel<<<(p.nfft + 255) / 256, 256, 0, st>>>(p, pw, g);
        JB_CUDA(cudaGetLastError());
        *launches += 3;
    }
    return 0;
}

} // namespace jb
