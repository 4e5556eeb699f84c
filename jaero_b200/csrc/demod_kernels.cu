// Single translation unit for the continuous demodulator kernels; each file also compiles on its own.
// Built with -fmad=false: see demod_device.cuh.
#include "oqpsk_demod.cu"
#include "oqpsk_pipe.cu"
#include "msk_pipe.cu"

// ---- test support (jaero_probe_math, jaero_probe_osc): the primitives of demod_device.cuh as this unit compiles them
#include "../../include/jaero_b200.h"

namespace jb {

__global__ void probe_math_kernel(int op, size_t n, const double *__restrict__ a, const double *__restrict__ b, double *__restrict__ out)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const double x = a[i];
        double r = 0.0;
        switch (op) {
        case JAERO_MATH_DIV_EXACT: { const double d = b[i]; r = div_exact(x, d, 1.0 / d); break; }   // rcp as MeanDivExact forms it
        case JAERO_MATH_DIV_FAST: r = div_fast(x, b[i]); break;
        case JAERO_MATH_ATAN2_FAST: r = atan2_fast(x, b[i]); break;
        case JAERO_MATH_HYPOT_FAST: r = hypot_fast(x, b[i]); break;
        case JAERO_MATH_OSC_INDEX: r = osc_index(x); break;
        case JAERO_MATH_Q_ROUND: r = q_round(x); break;
        case JAERO_MATH_FMOD360: r = fmod360(x); break;
        }
        out[i] = r;
    }
}

int probe_math_launch(int op, size_t n, const double *a, const double *b, double *out, cudaStream_t s)
{
    const size_t blocks = (n + 255) / 256;
    probe_math_kernel<<<(unsigned)(blocks < 4096 ? blocks : 4096), 256, 0, s>>>(op, n, a, b, out);
    JB_CUDA(cudaGetLastError());
    return 0;
}

// thread per lane: one oscillator running its own script
__global__ void probe_osc_kernel(int n_lanes, int n_ops, const int32_t *__restrict__ op, const double *__restrict__ arg, double samplerate,
                                 double *__restrict__ log)
{
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= n_lanes) return;
    Osc o = {0.0, 0.0, 0.0, 0.0};
    double frac = 0.0;
    for (int k = 0; k < n_ops; k++) {
        const size_t e = (size_t)l * n_ops + k;
        const double x = arg[e];
        int index = -1;
        bool flag = false;
        switch (op[e]) {
        case JAERO_OSC_SET_FREQ: osc_set_freq(o, x, samplerate); break;
        case JAERO_OSC_SET_FREQ_SR: osc_set_freq_wrap(o, x, (int)samplerate); break;
        case JAERO_OSC_NEXT_FRAME: osc_next_frame(o); break;
        case JAERO_OSC_NEXT_INDEX: index = osc_next_index(o); break;
        case JAERO_OSC_INCREASE_PHASE_DEG: osc_increase_phase_deg(o, x); break;
        case JAERO_OSC_SET_PHASE_DEG: osc_set_phase_deg(o, x); break;
        case JAERO_OSC_ADVANCE_FRACTION: osc_advance_fraction_of_wave(o, x); break;
        case JAERO_OSC_HAVE_PASSED_POINT: flag = osc_have_passed_point(o, x, frac); break;
        }
        if (index < 0) index = osc_index(o.ptr);
        double *g = log + e * 7;
        g[0] = o.ptr; g[1] = o.last; g[2] = o.step; g[3] = o.freq; g[4] = index; g[5] = flag ? 1.0 : 0.0; g[6] = frac;
    }
}

int probe_osc_launch(int n_lanes, int n_ops, const int32_t *op, const double *arg, double samplerate, double *log, cudaStream_t s)
{
    probe_osc_kernel<<<(n_lanes + 63) / 64, 64, 0, s>>>(n_lanes, n_ops, op, arg, samplerate, log);
    JB_CUDA(cudaGetLastError());
    return 0;
}

} // namespace jb
