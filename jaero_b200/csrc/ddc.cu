// Wideband IQ digital down-converter: one complex IQ stream -> per-channel real int16 PCM at Fs_in * L / (D1 * D2).
//
// Per channel c (include/jaero_b200.h, jaero_ddc_create_rational, states the contract):
//   u_c[j] = exp(-2 pi i ((j D1 T_c) mod 2^32) / 2^32) * sum_k h1c_c[k] x[j D1 - k]    (mix folded into complex taps)
//   v_c[m] = sum_r h2[phi_m + r L] u_c[q_m - r],  q_m = floor(m D2 / L), phi_m = m D2 - q_m L
//            (the polyphase form of sum_k h2[k] w_c[m D2 - k], w_c the x L zero-stuffed u_c; L = 1: sum_k h2[k] u_c[m D2 - k])
//   pcm_c[m] = clamp(rint(g 32768 Re{v_c[m] exp(+2 pi i ((m S_c) mod 2^32) / 2^32)}))
// The phases depend on the sample index only, so the output does not depend on how the stream is cut into writes: every
// output is the same sum in the same order whichever write completes it.
//
// A write runs four kernels on the DDC's stream:
//   stage_in  the shared input history + the new samples converted to double -> xd; the stage-1 history -> head of ubuf
//   stage1    per CTA 32 channels (one per lane) x DDC_TILE_J outputs (DDC_WARP_J per thread); the input tile sits in
//             shared memory and is read as a warp-wide broadcast, the folded taps come from L2 ([k][channel], coalesced)
//   stage2    one output per thread, lanes over channels: ubuf is [row][channel] so every tap reads 32 consecutive values;
//             for L > 1 (ddc_stage2_poly_kernel) a warp's outputs share one phase, so its taps are one warp-wide broadcast
//   carry     the tails of xd and ubuf become the histories of the next write
#include "ddc.cuh"
#include "common.cuh"
#include "../../include/jaero_b200.h"
#include <algorithm>

namespace jb {

// exp(sign * 2 pi i w / 2^32)
__device__ __forceinline__ double2 phasor(uint32_t w)
{
    double s, c;
    sincospi((double)w * (1.0 / 2147483648.0), &s, &c);
    return make_double2(c, s);
}

__global__ void ddc_stage_in_kernel(DdcParams p, const void *raw, int format, long long n, double2 *xd, double2 *ubuf)
{
    const long long H1 = p.K1 - 1, nx = H1 + n, nu = (long long)p.H2 * p.cpad;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nx + nu; i += (long long)gridDim.x * blockDim.x) {
        if (i < H1) xd[i] = p.xhist[i];
        else if (i < nx) xd[i] = iq_sample(raw, i - H1, format);
        else ubuf[i - nx] = p.uhist[i - nx];
    }
}

__global__ void __launch_bounds__(DDC_WARPS * 32) ddc_stage1_kernel(DdcParams p, const double2 *__restrict__ xd, long long n0,
                                                                    long long nxd, long long j_lo, long long J, double2 *__restrict__ ubuf)
{
    extern __shared__ double2 xs[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + lane;
    const int D1 = p.D1, K1 = p.K1;
    const int tile = (DDC_TILE_J - 1) * D1 + K1;
    const size_t H2 = p.H2;
    const double2 *__restrict__ taps = p.h1c + c;
    const uint32_t T = c < p.n_channels ? p.T[c] : 0u;
    for (long long jt0 = j_lo + (long long)blockIdx.y * DDC_TILE_J; jt0 < j_lo + J; jt0 += (long long)gridDim.y * DDC_TILE_J) {
        // xd index of input jt0 D1 - (K1 - 1), the oldest sample the tile's first output reads
        const long long base = jt0 * D1 - n0;
        __syncthreads();
        for (int i = threadIdx.x; i < tile; i += blockDim.x)
            xs[i] = base + i < nxd ? xd[base + i] : make_double2(0.0, 0.0);
        __syncthreads();
        double2 acc[DDC_WARP_J];
#pragma unroll
        for (int r = 0; r < DDC_WARP_J; r++) acc[r] = make_double2(0.0, 0.0);
        const double2 *xw = xs + warp * DDC_WARP_J * D1 + K1 - 1;
        for (int k = 0; k < K1; k++) {
            const double2 h = __ldg(taps + (size_t)k * p.cpad);
#pragma unroll
            for (int r = 0; r < DDC_WARP_J; r++) {
                const double2 x = xw[r * D1 - k];
                acc[r].x = fma(h.x, x.x, fma(-h.y, x.y, acc[r].x));
                acc[r].y = fma(h.x, x.y, fma(h.y, x.x, acc[r].y));
            }
        }
        if (c < p.n_channels) {
#pragma unroll
            for (int r = 0; r < DDC_WARP_J; r++) {
                const long long j = jt0 + warp * DDC_WARP_J + r;
                if (j >= j_lo + J) break;
                const double2 w = phasor((uint32_t)(unsigned long long)(j * D1) * T);   // exp(-i theta) = conj(w)
                ubuf[(H2 + (size_t)(j - j_lo)) * p.cpad + c] = make_double2(w.x * acc[r].x + w.y * acc[r].y, w.x * acc[r].y - w.y * acc[r].x);
            }
        }
    }
}

// L = 1: v_c[m] = sum_k h2[k] u_c[m D2 - k], all K2 taps in ascending order (H2 = K2 - 1)
__global__ void __launch_bounds__(128) ddc_stage2_kernel(DdcParams p, const double2 *__restrict__ ubuf, long long j_lo, long long m_lo,
                                                         long long M, int16_t *__restrict__ pcm, size_t pcm_stride)
{
    const int c = blockIdx.x * 32 + (threadIdx.x & 31);
    if (c >= p.n_channels) return;
    const size_t H2 = p.K2 - 1;
    const uint32_t S = p.S[c];
    for (long long m = m_lo + (long long)blockIdx.y * 4 + (threadIdx.x >> 5); m < m_lo + M; m += (long long)gridDim.y * 4) {
        const double2 *u = ubuf + (H2 + (size_t)(m * p.D2 - j_lo)) * p.cpad + c;   // u_c[m D2]
        double vr = 0.0, vi = 0.0;
        for (int k = 0; k < p.K2; k++) {
            const double h = __ldg(p.h2 + k);
            const double2 x = u[-(ptrdiff_t)k * p.cpad];
            vr = fma(h, x.x, vr);
            vi = fma(h, x.y, vi);
        }
        const double2 w = phasor((uint32_t)(unsigned long long)m * S);
        const double r = rint(p.scale * (vr * w.x - vi * w.y));
        int16_t q;
        if (r > 32767.0) { q = 32767; atomicAdd(p.clipped + c, 1ull); }
        else if (r < -32768.0) { q = -32768; atomicAdd(p.clipped + c, 1ull); }
        else q = (int16_t)r;
        pcm[(size_t)c * pcm_stride + (size_t)(m - m_lo)] = q;
    }
}

// L > 1: output m sums taps h2[phi + r L] against rows u[q_m - r], q_m = floor(m D2 / L), phi = m D2 - q_m L; the zero-stuffed
// samples of the x L interpolation contribute nothing and are skipped. phi depends on m only, so it is uniform across a warp
// (lanes are channels). With L = 1 this would be the sum above; the integer rates keep that kernel as it is, because the phase
// arithmetic here changes how the compiler schedules the tap loop (fewer loads in flight, a slower kernel).
__global__ void __launch_bounds__(128) ddc_stage2_poly_kernel(DdcParams p, const double2 *__restrict__ ubuf, long long j_lo, long long m_lo,
                                                              long long M, int16_t *__restrict__ pcm, size_t pcm_stride)
{
    const int c = blockIdx.x * 32 + (threadIdx.x & 31);
    if (c >= p.n_channels) return;
    const size_t H2 = p.H2;
    const uint32_t S = p.S[c];
    for (long long m = m_lo + (long long)blockIdx.y * 4 + (threadIdx.x >> 5); m < m_lo + M; m += (long long)gridDim.y * 4) {
        const long long mD2 = m * p.D2, qm = mD2 / p.L;
        const int phi = (int)(mD2 - qm * p.L), taps = (p.K2 - phi + p.L - 1) / p.L;
        const double2 *u = ubuf + (H2 + (size_t)(qm - j_lo)) * p.cpad + c;         // u_c[q_m]
        const double *h2 = p.h2 + (size_t)phi * p.R;
        double vr = 0.0, vi = 0.0;
        for (int k = 0; k < taps; k++) {
            const double h = __ldg(h2 + k);
            const double2 x = u[-(ptrdiff_t)k * p.cpad];
            vr = fma(h, x.x, vr);
            vi = fma(h, x.y, vi);
        }
        const double2 w = phasor((uint32_t)(unsigned long long)m * S);
        const double r = rint(p.scale * (vr * w.x - vi * w.y));
        int16_t q;
        if (r > 32767.0) { q = 32767; atomicAdd(p.clipped + c, 1ull); }
        else if (r < -32768.0) { q = -32768; atomicAdd(p.clipped + c, 1ull); }
        else q = (int16_t)r;
        pcm[(size_t)c * pcm_stride + (size_t)(m - m_lo)] = q;
    }
}

__global__ void ddc_carry_kernel(DdcParams p, const double2 *xd, long long n, const double2 *ubuf, long long J)
{
    const long long H1 = p.K1 - 1, nu = (long long)p.H2 * p.cpad;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < H1 + nu; i += (long long)gridDim.x * blockDim.x) {
        if (i < H1) p.xhist[i] = xd[n + i];
        else p.uhist[i - H1] = ubuf[J * p.cpad + (i - H1)];
    }
}

static int grid_for(long long work, int block) { return (int)std::min<long long>((work + block - 1) / block, 4L * 132 * 16); }

int ddc_run(const DdcParams &p, const void *d_iq, int format, long long n0, long long n, double2 *xd, double2 *ubuf,
            int16_t *pcm, size_t pcm_stride, cudaStream_t st, long long *launches)
{
    const long long D = (long long)p.D1 * p.D2;
    const long long j_lo = (n0 + p.D1 - 1) / p.D1, J = (n0 + n + p.D1 - 1) / p.D1 - j_lo;
    const long long m_lo = (n0 * p.L + D - 1) / D, M = ((n0 + n) * p.L + D - 1) / D - m_lo;   // outputs m with floor(m D / L) in [n0, n0 + n)
    const long long nxd = p.K1 - 1 + n, nu = (long long)p.H2 * p.cpad;
    const int groups = p.cpad / 32;
    ddc_stage_in_kernel<<<grid_for(nxd + nu, 256), 256, 0, st>>>(p, d_iq, format, n, xd, ubuf);
    JB_CUDA(cudaGetLastError());
    ++*launches;
    if (J > 0) {
        const int smem = ((DDC_TILE_J - 1) * p.D1 + p.K1) * (int)sizeof(double2);
        JB_CUDA(cudaFuncSetAttribute(ddc_stage1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        const long long tiles = (J + DDC_TILE_J - 1) / DDC_TILE_J;
        dim3 grid(groups, (unsigned)std::min<long long>(tiles, 65535));
        ddc_stage1_kernel<<<grid, DDC_WARPS * 32, smem, st>>>(p, xd, n0, nxd, j_lo, J, ubuf);
        JB_CUDA(cudaGetLastError());
        ++*launches;
    }
    if (M > 0) {
        dim3 grid(groups, (unsigned)std::min<long long>((M + 3) / 4, 65535));
        if (p.L == 1) ddc_stage2_kernel<<<grid, 128, 0, st>>>(p, ubuf, j_lo, m_lo, M, pcm, pcm_stride);
        else ddc_stage2_poly_kernel<<<grid, 128, 0, st>>>(p, ubuf, j_lo, m_lo, M, pcm, pcm_stride);
        JB_CUDA(cudaGetLastError());
        ++*launches;
    }
    ddc_carry_kernel<<<grid_for(p.K1 - 1 + nu, 256), 256, 0, st>>>(p, xd, n, ubuf, J);
    JB_CUDA(cudaGetLastError());
    ++*launches;
    return 0;
}

} // namespace jb
