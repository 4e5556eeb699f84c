// PCM rate converter: n_channels int16 PCM streams at input_rate -> int16 PCM at input_rate * L / M.
//
// Per channel c (include/jaero_b200.h, jaero_resample_create, states the contract):
//   v_c[m] = sum_r h[phi_m + r L] x_c[q_m - r],  q_m = floor(m M / L), phi_m = m M - q_m L
//            (the polyphase form of sum_k h[k] w_c[m M - k], w_c the x L zero-stuffed x_c)
//   pcm_c[m] = clamp(rint(v_c[m]), -32768, 32767)
// The phase depends on the sample index only, so the output does not depend on how the stream is cut into writes: every
// output is the same sum in the same order whichever write completes it.
//
// A write runs three kernels on the resampler's stream:
//   stage_in   the carried rows -> head of xd; the write's channel-major int16 rows transposed through a shared-memory tile into
//              the [row][channel] double rows after them (reads along a channel's samples, writes along a row's channels)
//   poly       one output per thread, lanes over channels, a warp per output m: the phase is warp-uniform, so each tap is one
//              warp-wide broadcast from the [L][R] phase table and each input row one coalesced 256-byte read
//   carry      the last H rows of xd become the history of the next write
#include "resample.cuh"
#include "common.cuh"
#include <algorithm>

namespace jb {

__global__ void __launch_bounds__(RS_TILE * 8) resample_stage_in_kernel(ResampleParams p, const int16_t *__restrict__ in, size_t in_stride,
                                                                        long long n, double *__restrict__ xd)
{
    __shared__ double tile[RS_TILE][RS_TILE + 1];
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int c0 = blockIdx.y * RS_TILE;
    const size_t H = p.H, cpad = p.cpad;
    for (long long s0 = (long long)blockIdx.x * RS_TILE; s0 < n; s0 += (long long)gridDim.x * RS_TILE) {
        __syncthreads();
        for (int cy = ty; cy < RS_TILE; cy += blockDim.y) {
            const int c = c0 + cy;
            const long long s = s0 + tx;
            tile[cy][tx] = c < p.n_channels && s < n ? (double)in[(size_t)c * in_stride + (size_t)s] : 0.0;
        }
        __syncthreads();
        for (int sy = ty; sy < RS_TILE; sy += blockDim.y) {
            const long long s = s0 + sy;
            if (s < n) xd[(H + (size_t)s) * cpad + c0 + tx] = tile[tx][sy];
        }
    }
    const long long nh = (long long)H * p.cpad;
    const long long tid = ((long long)blockIdx.y * gridDim.x + blockIdx.x) * (blockDim.x * blockDim.y) + ty * blockDim.x + tx;
    for (long long i = tid; i < nh; i += (long long)gridDim.x * gridDim.y * blockDim.x * blockDim.y) xd[i] = p.hist[i];
}

// Output m sums the ceil((K - phi) / L) taps h[phi + r L] against rows x[q_m - r] in ascending r; the zero-stuffed samples of
// the x L interpolation contribute nothing and are skipped. A CTA takes RS_WARPS * RS_WARP_M consecutive outputs, interleaved
// over its warps: at any time its warps read one window of about R + RS_WARPS rows, and the few windows an SM holds fit in L1.
__global__ void __launch_bounds__(RS_WARPS * 32) resample_poly_kernel(ResampleParams p, const double *__restrict__ xd, long long n0, long long m_lo,
                                                            long long M_out, int16_t *__restrict__ out, size_t out_stride)
{
    const int c = blockIdx.x * 32 + (threadIdx.x & 31), warp = threadIdx.x >> 5;
    if (c >= p.n_channels) return;
    const int L = p.L, R = p.R, K = p.K;
    const size_t cpad = p.cpad;
    const long long chunk = (long long)RS_WARPS * RS_WARP_M;
    unsigned long long clipped = 0;
    for (long long mc = m_lo + (long long)blockIdx.y * chunk; mc < m_lo + M_out; mc += (long long)gridDim.y * chunk) {
        const long long m_end = min(mc + chunk, m_lo + M_out);
        for (long long m = mc + warp; m < m_end; m += RS_WARPS) {
            const long long mM = m * p.M, q = mM / L;
            const int phi = (int)(mM - q * L), taps = (K - phi + L - 1) / L;
            const double *x = xd + ((size_t)(q - n0) + p.H) * cpad + c;       // x_c[q_m]
            const double *h = p.hp + (size_t)phi * R;
            double v = 0.0;
            for (int r = 0; r < taps; r++) v = fma(__ldg(h + r), x[-(ptrdiff_t)r * cpad], v);
            const double rv = rint(v);
            int16_t s;
            if (rv > 32767.0) { s = 32767; clipped++; }
            else if (rv < -32768.0) { s = -32768; clipped++; }
            else s = (int16_t)rv;
            out[(size_t)c * out_stride + (size_t)(m - m_lo)] = s;
        }
    }
    if (clipped) atomicAdd(p.clipped + c, clipped);
}

__global__ void resample_carry_kernel(ResampleParams p, const double *xd, long long n)
{
    const long long nh = (long long)p.H * p.cpad;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nh; i += (long long)gridDim.x * blockDim.x)
        p.hist[i] = xd[n * p.cpad + i];
}

int resample_run(const ResampleParams &p, const int16_t *pcm_in, size_t in_stride, long long n0, long long n, double *xd,
                 int16_t *out, size_t out_stride, cudaStream_t st, long long *launches)
{
    // outputs m with floor(m M / L) in [n0, n0 + n)
    const long long m_lo = (n0 * p.L + p.M - 1) / p.M, M_out = ((n0 + n) * p.L + p.M - 1) / p.M - m_lo;
    const int groups = p.cpad / 32;
    {
        dim3 grid((unsigned)std::min<long long>((n + RS_TILE - 1) / RS_TILE, 1LL << 20), groups);
        resample_stage_in_kernel<<<grid, dim3(RS_TILE, 8), 0, st>>>(p, pcm_in, in_stride, n, xd);
        JB_CUDA(cudaGetLastError());
        ++*launches;
    }
    if (M_out > 0) {
        const long long chunk = (long long)RS_WARPS * RS_WARP_M;
        dim3 grid(groups, (unsigned)std::min<long long>((M_out + chunk - 1) / chunk, 65535));
        resample_poly_kernel<<<grid, RS_WARPS * 32, 0, st>>>(p, xd, n0, m_lo, M_out, out, out_stride);
        JB_CUDA(cudaGetLastError());
        ++*launches;
    }
    const long long nh = (long long)p.H * p.cpad;
    resample_carry_kernel<<<(int)std::min<long long>((nh + 255) / 256, 4L * 132 * 16), 256, 0, st>>>(p, xd, n);
    JB_CUDA(cudaGetLastError());
    ++*launches;
    return 0;
}

} // namespace jb
