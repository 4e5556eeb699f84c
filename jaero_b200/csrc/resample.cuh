// PCM rate converter — device data layout and launch prototypes (see resample.cu).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace jb {

static const int RS_TILE = 32;              // stage-in transpose tile: 32 channels x 32 samples
static const int RS_WARPS = 16;             // warps of a polyphase CTA: they share its 32 channels and work on neighbouring outputs
static const int RS_WARP_M = 4;             // outputs per warp in one CTA chunk of RS_WARPS * RS_WARP_M consecutive outputs

struct ResampleParams {
    int n_channels, cpad;                   // cpad: channels rounded up to 32, the row pitch of every [row][channel] table
    int L, M, K;                            // output rate = input rate * L / M; K taps of the prototype at L * input rate
    int R;                                  // taps per phase, ceil(K / L)
    int H;                                  // input rows carried between writes, R
    const double *hp;                       // [L][R] phase table, hp[phi][r] = h[phi + r L], zero-padded
    double *hist;                           // [H][cpad] the input rows before the current write
    unsigned long long *clipped;            // [n_channels]
};

// One write of n >= 1 samples per channel, global indices n0 .. n0+n-1 (n0 = samples per channel before this write).
// pcm_in: [n_channels][in_stride] int16 rows (device); xd: work buffer of [H + n][cpad] doubles; out: [n_channels][out_stride]
// rows of the outputs this write completes.
int resample_run(const ResampleParams &p, const int16_t *pcm_in, size_t in_stride, long long n0, long long n, double *xd,
                 int16_t *out, size_t out_stride, cudaStream_t st, long long *launches);

} // namespace jb
