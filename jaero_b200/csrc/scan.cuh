// Wideband carrier scanner — averaged power spectrum of one IQ stream (see scan.cu, include/jaero_b200.h jaero_scan_*).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace jb {

static const int SCAN_TILE = 16;                 // sequences of one shared-memory tile (16 x 16 B = 256 B global segments)
static const int SCAN_THREADS = 256;
static const int SCAN_MAXN = 256;                // longest row / column transform: nfft 2^16 = 256 x 256
static const int SCAN_SMEM = SCAN_TILE * (SCAN_MAXN + 1) * 16;
static const long long SCAN_PASS_ELEMS = 1 << 21; // frame bins of one batched pass: 32 MB of work matrix + 16 MB of powers

struct ScanPlan {
    int nfft, n1, n2, hop;                       // nfft = n1 * n2 (four-step: n1-point columns, n2-point rows)
    const double2 *tw;                           // [nfft] exp(-2 pi i k / nfft)
    const double *win;                           // [nfft] periodic Hann
    double inv_wss;                              // 1 / sum w^2
    double *sum, *maxh;                          // [nfft] running sum / max of the normalised |X|^2, fftshift order
};

// xd[j] = converted sample x0 + j. Frames f0 .. f0+F-1 (frame f = samples f*hop .. f*hop+nfft-1, all inside xd) are transformed and
// added to sum / maxh in frame order. work: [G][nfft] double2, pw: [G][nfft] double, G = the frames of one pass.
int scan_frames(const ScanPlan &p, const double2 *xd, long long x0, long long f0, long long F, int G, double2 *work, double *pw,
                cudaStream_t st, long long *launches);
// xd[i] = the n raw samples of d_iq converted as the down-converter converts them
int scan_convert(const void *d_iq, int format, long long n, double2 *xd, cudaStream_t st, long long *launches);

} // namespace jb
