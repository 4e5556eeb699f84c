// Double-precision complex arithmetic and FFT building blocks: the complex helpers and butterflies of every device FFT (coarse
// estimator, wideband scanner, FFT convolution, trident FFTs) and the demodulators' complex products, plus the Stockham autosort
// pass with radix-8 / radix-4 butterflies kept in registers over TILE independent sequences held in natural order in shared
// memory rows s[f][.] (row pitch LD) that the estimator and the scanner use.
#pragma once
#include <cuda_runtime.h>

namespace jb {

// Written in std::complex<double>'s evaluation order. Whether the products and sums contract into FMAs is decided by the flags of
// the translation unit that inlines them: prefilter.cu, fastfir.cu, burst.cu and demod_kernels.cu are built with -fmad=false,
// so that they round as the CPU reference does (x86-64 has no implicit FMA contraction); cfe.cu and scan.cu let them contract.
__device__ __forceinline__ double2 c_add(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ double2 c_sub(double2 a, double2 b) { return make_double2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ double2 c_mul(double2 a, double2 b) { return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
template <bool INV> __device__ __forceinline__ double2 c_rot(double2 a)      // multiply by -i (forward) / +i (inverse)
{ return INV ? make_double2(-a.y, a.x) : make_double2(a.y, -a.x); }

template <bool INV> __device__ __forceinline__ void dft4(double2 &a0, double2 &a1, double2 &a2, double2 &a3)
{
    const double2 t0 = c_add(a0, a2), t1 = c_sub(a0, a2), t2 = c_add(a1, a3), t3 = c_rot<INV>(c_sub(a1, a3));
    a0 = c_add(t0, t2); a1 = c_add(t1, t3); a2 = c_sub(t0, t2); a3 = c_sub(t1, t3);
}
template <bool INV> __device__ __forceinline__ void dft8(double2 *v)
{
    // even / odd split: X[k] = E[k] + W8^k O[k], X[k+4] = E[k] - W8^k O[k]
    double2 e0 = v[0], e1 = v[2], e2 = v[4], e3 = v[6], o0 = v[1], o1 = v[3], o2 = v[5], o3 = v[7];
    dft4<INV>(e0, e1, e2, e3);
    dft4<INV>(o0, o1, o2, o3);
    const double h = 0.70710678118654752440;
    // W8^1 = (1 -/+ i)/sqrt2, W8^2 = -/+ i, W8^3 = (-1 -/+ i)/sqrt2   (upper sign: forward)
    const double2 w1 = INV ? make_double2(h, h) : make_double2(h, -h);
    const double2 w3 = INV ? make_double2(-h, h) : make_double2(-h, -h);
    o1 = c_mul(o1, w1); o2 = c_rot<INV>(o2); o3 = c_mul(o3, w3);
    v[0] = c_add(e0, o0); v[4] = c_sub(e0, o0);
    v[1] = c_add(e1, o1); v[5] = c_sub(e1, o1);
    v[2] = c_add(e2, o2); v[6] = c_sub(e2, o2);
    v[3] = c_add(e3, o3); v[7] = c_sub(e3, o3);
}

// One radix-R pass (stride Ns) of TILE length-n transforms in s[f][0..n), THREADS threads. Every pass is "all threads read their
// inputs, barrier, compute + write, barrier" so it runs in place. tw = W_N^k table (N = big transform), tw_stride = N/n.
template <bool INV, int R, int TILE, int LD, int THREADS>
__device__ __forceinline__ void stockham_pass(double2 (*s)[LD], int n, int Ns, const double2 *__restrict__ tw, int tw_stride)
{
    constexpr int PER = 8 / R;                       // butterflies per thread per round (8 complex values in registers)
    const int nb = n / R;                            // butterflies per sequence
    const int total = TILE * nb;
    const int wmul = tw_stride * (n / (Ns * R));     // table step of exp(-2 pi i /(Ns R))
    for (int base = 0; base < total; base += THREADS * PER) {
        double2 v[8];
        int ff[PER], jj[PER];
#pragma unroll
        for (int q = 0; q < PER; q++) {
            const int b = base + threadIdx.x + q * THREADS;
            ff[q] = -1;
            if (b < total) {
                const int f = b / nb, j = b - f * nb;
                ff[q] = f; jj[q] = j;
#pragma unroll
                for (int t = 0; t < R; t++) v[q * R + t] = s[f][j + t * nb];
            }
        }
        __syncthreads();
#pragma unroll
        for (int q = 0; q < PER; q++) {
            if (ff[q] >= 0) {
                const int j = jj[q], k = j % Ns;
#pragma unroll
                for (int t = 1; t < R; t++) {
                    double2 w = tw[(t * k * wmul)];
                    if (INV) w.y = -w.y;
                    v[q * R + t] = c_mul(v[q * R + t], w);
                }
                if (R == 8) dft8<INV>(&v[q * R]);
                else dft4<INV>(v[q * R + 0], v[q * R + 1], v[q * R + 2], v[q * R + 3]);
                const int ob = (j / Ns) * Ns * R + k;
#pragma unroll
                for (int t = 0; t < R; t++) s[ff[q]][ob + t * Ns] = v[q * R + t];
            }
        }
        __syncthreads();
    }
}

} // namespace jb
