// Wideband IQ digital down-converter — device data layout and launch prototypes (see ddc.cu).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "../../include/jaero_b200.h"

namespace jb {

// Raw IQ sample i of a cu8 / cs16 stream as a complex double (the carrier scanner converts its input the same way)
__device__ __forceinline__ double2 iq_sample(const void *raw, long long i, int format)
{
    if (format == JAERO_IQ_CU8) {
        const uchar2 v = reinterpret_cast<const uchar2 *>(raw)[i];
        return make_double2(((double)v.x - 127.5) * (1.0 / 128.0), ((double)v.y - 127.5) * (1.0 / 128.0));
    }
    const short2 v = reinterpret_cast<const short2 *>(raw)[i];
    return make_double2((double)v.x * (1.0 / 32768.0), (double)v.y * (1.0 / 32768.0));
}

static const int DDC_WARP_J = 8;            // stage-1 outputs one thread accumulates (register blocking over j)
static const int DDC_WARPS = 4;             // warps of a stage-1 CTA; all of them share the CTA's 32 channels
static const int DDC_TILE_J = DDC_WARP_J * DDC_WARPS;
static const int DDC_MAX_TILE = 12288;      // input samples of one stage-1 tile, (DDC_TILE_J - 1) * D1 + K1: 192 KB of shared memory

struct DdcParams {
    int n_channels, cpad;                   // cpad: channels rounded up to 32, the row pitch of every [row][channel] table
    int D1, K1, D2, K2;                     // output rate = input rate * L / (D1 * D2); D2 is stage 2's decimation M2
    double scale;                           // gain * 32768
    const double2 *h1c;                     // [K1][cpad] folded stage-1 taps h1[k] * exp(+2 pi i ((k T_c) mod 2^32) / 2^32)
    const double *h2;                       // [L][R] polyphase stage-2 taps, row phi = h2[phi + r L], zero-padded (L = 1: h2 itself)
    const uint32_t *T, *S;                  // [n_channels] tuning words
    double2 *xhist;                         // [K1 - 1] the input samples before the current write (shared by every channel)
    double2 *uhist;                         // [H2][cpad] the stage-1 outputs before the current write
    unsigned long long *clipped;            // [n_channels]
    int L;                                  // stage 2's interpolation (1: a plain decimator)
    int R;                                  // stage-2 taps per phase, ceil(K2 / L)
    int H2;                                 // stage-1 rows carried between writes: K2 - 1 for L = 1, R for L > 1
};

// One write of n >= 1 input samples, global indices n0 .. n0+n-1 (n0 = samples before this write).
// xd: work buffer of K1 - 1 + n samples; ubuf: work buffer of [H2 + J][cpad] stage-1 outputs, J = the stage-1 outputs
// this write completes; pcm: [n_channels][pcm_stride] rows, one per channel, of the outputs this write completes.
int ddc_run(const DdcParams &p, const void *d_iq, int format, long long n0, long long n, double2 *xd, double2 *ubuf,
            int16_t *pcm, size_t pcm_stride, cudaStream_t st, long long *launches);

} // namespace jb
