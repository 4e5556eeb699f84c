// Mode identifier — averaged spectrum of each PCM channel's squared analytic signal (see ident.cu, include/jaero_b200.h
// jaero_ident_*).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace jb {

static const int IDENT_TILE = 16;                 // sequences of one shared-memory tile (16 x 16 B = 256 B global segments)
static const int IDENT_THREADS = 256;
static const int IDENT_MAXN = 128;                // longest row / column transform: nfft 2^14 = 128 x 128
static const int IDENT_SMEM = IDENT_TILE * (IDENT_MAXN + 1) * 16;
static const long long IDENT_PASS_ELEMS = 1 << 20; // frame bins of one batched pass: two 16 MB work matrices, both L2-resident

struct IdentPlan {
    int nfft, n1, n2, hop;                        // nfft = n1 * n2 (four-step: n1-point columns, n2-point rows), hop = nfft / 2
    int n_channels;
    const double2 *tw;                            // [nfft] exp(-2 pi i k / nfft)
    const double *win;                            // [nfft] periodic Hann
    double inv_wss2;                              // 1 / (sum w^2)^2
    double *sum;                                  // [n_channels][nfft] running sum of the normalised |Y|^2, fftshift order
};

// xs[c * pitch + j] = PCM sample x0 + j of channel c. Frames f0 .. f0+F-1 of every channel (frame f = samples f*hop .. f*hop+nfft-1,
// all inside xs) are transformed and added to sum in frame order. w0, w1: [G][nfft] double2 work matrices, G the frames of one pass.
int ident_frames(const IdentPlan &p, const int16_t *xs, size_t pitch, long long x0, long long f0, long long F, int G, double2 *w0,
                 double2 *w1, cudaStream_t st, long long *launches);

} // namespace jb
