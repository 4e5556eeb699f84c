#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "fastfir.cuh"
namespace jb {

struct PreParams {                        // 8400 bps pre-filter front end
    int n_channels, cpad;
    double *osc;                          // [4][cpad]: mixer_fir_pre WTptr, WTstep, freq, mix-up pointer
    double2 *x;                           // [ch][xstride] mixed-down -> filtered -> mixed-up samples of the current call
    size_t xstride;
    const double *sin_t, *cos_t;
};

int pre_down_launch(const PreParams &q, const int16_t *pcm, size_t stride, int n, cudaStream_t s);
int fir_exchange_up_launch(const PreParams &q, const FastFir &f, int i0, int i1, int fill0, cudaStream_t s);
int pre_finish_launch(const PreParams &q, const double *m2_freq_sum, int n, double Fs, cudaStream_t s);
}
