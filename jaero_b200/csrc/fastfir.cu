// The overlap-save block of the FFT convolution (fastfir.cuh): one CTA per channel, the whole transform in shared memory
// (nfft 4096: 64 KB, 512 threads; nfft 8192: 128 KB, 1024 threads). Stockham radix-8 passes with one butterfly per thread in
// registers; 8192 = 8^4 * 2 ends with a radix-2 pass. Built with -fmad=false, like the reference's FFT.
#include "common.cuh"
#include "fastfir.cuh"
#include "fft_device.cuh"

namespace jb {

// one Stockham radix-8 pass (stride Ns) over the NFFT-point sequence s, in place: NFFT/8 threads, one butterfly each
template <int NFFT, bool INV> __device__ __forceinline__ void ff_pass8(double2 *s, int Ns, const double2 *__restrict__ tw)
{
    constexpr int NB = NFFT / 8;
    const int j = threadIdx.x;
    double2 v[8];
#pragma unroll
    for (int t = 0; t < 8; t++) v[t] = s[j + t * NB];
    __syncthreads();
    const int k = j % Ns;
    const int wmul = NFFT / (Ns * 8);
#pragma unroll
    for (int t = 1; t < 8; t++) {
        double2 w = tw[t * k * wmul];
        if (INV) w.y = -w.y;
        v[t] = c_mul(v[t], w);
    }
    dft8<INV>(v);
    const int ob = (j / Ns) * Ns * 8 + k;
#pragma unroll
    for (int t = 0; t < 8; t++) s[ob + t * Ns] = v[t];
    __syncthreads();
}
// the last pass of NFFT = 8^4 * 2: radix-2 with Ns = NFFT/2, so k = j and the twiddle step is 1; 4 butterflies per thread
template <int NFFT, bool INV> __device__ __forceinline__ void ff_pass2_last(double2 *s, const double2 *__restrict__ tw)
{
    constexpr int NT = NFFT / 8, HALF = NFFT / 2, PER = HALF / NT;
    double2 a[PER], b[PER];
    for (int q = 0; q < PER; q++) { const int j = threadIdx.x + q * NT; a[q] = s[j]; b[q] = s[j + HALF]; }
    __syncthreads();
    for (int q = 0; q < PER; q++) {
        const int j = threadIdx.x + q * NT;
        double2 w = tw[j];
        if (INV) w.y = -w.y;
        const double2 bw = c_mul(b[q], w);
        s[j] = c_add(a[q], bw); s[j + HALF] = c_sub(a[q], bw);
    }
    __syncthreads();
}
template <int NFFT, bool INV> __device__ __forceinline__ void ff_fft(double2 *s, const double2 *__restrict__ tw)
{
    static_assert(NFFT == 4096 || NFFT == 8192, "FFT convolution sizes: 8^4 and 8^4 * 2");
    // unrolled at 4096 (512 threads may use 128 registers); at 8192 the 64 registers of 1024 threads only hold one pass at a time
#pragma unroll (NFFT == 4096 ? 4 : 1)
    for (int Ns = 1; Ns <= 512; Ns *= 8) ff_pass8<NFFT, INV>(s, Ns, tw);
    if (NFFT == 8192) ff_pass2_last<NFFT, INV>(s, tw);
}

// JFastFir::update's compute step when the staging block fills: one CTA per channel
template <int NFFT, int K>
__global__ void __launch_bounds__(NFFT / 8)
fastfir_block_kernel(FastFir f, int first_block)
{
    extern __shared__ double2 fs[];
    constexpr int NT = NFFT / 8, K1 = K - 1, L = NFFT - K + 1;
    static_assert(L >= K1, "the new history must lie inside the new block");
    const int ch = blockIdx.x;
    double2 *hist = f.hist + (size_t)ch * K1, *inb = f.inblk + (size_t)ch * L, *outb = f.outblk + (size_t)ch * L;
    for (int j = threadIdx.x; j < L; j += NT) {
        const double2 x = inb[j];
        fs[K1 + j] = x;
        if (j < K1) {                     // new history = last K-1 samples of [history | block], all of them in the block
            fs[j] = hist[j];
            hist[j] = inb[L - K1 + j];
        }
    }
    __syncthreads();
    ff_fft<NFFT, false>(fs, f.tw);
    for (int j = threadIdx.x; j < NFFT; j += NT) fs[j] = c_mul(fs[j], f.H[j]);
    __syncthreads();
    ff_fft<NFFT, true>(fs, f.tw);
    const double sc = 1.0 / (double)NFFT;         // JFFT::ifft is 1/N-normalised
    for (int j = threadIdx.x; j < L; j += NT) {
        const double2 y = fs[K1 + j];             // positions K-1 .. K-1+L-1 are the valid (non-circular) outputs
        outb[j] = first_block ? make_double2(0.0, 0.0) : make_double2(y.x * sc, y.y * sc);
    }
}

template <int NFFT, int K> static int block_launch(const FastFir &f, int n_channels, int first_block, cudaStream_t s)
{
    const int smem = NFFT * (int)sizeof(double2);
    JB_CUDA(cudaFuncSetAttribute(fastfir_block_kernel<NFFT, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    fastfir_block_kernel<NFFT, K><<<n_channels, NFFT / 8, smem, s>>>(f, first_block);
    JB_CUDA(cudaGetLastError());
    return 0;
}
int fastfir_block_launch(const FastFir &f, int n_channels, int first_block, cudaStream_t s)
{
    return f.nfft == 4096 ? block_launch<4096, 2049>(f, n_channels, first_block, s) : block_launch<8192, 2048>(f, n_channels, first_block, s);
}

} // namespace jb
