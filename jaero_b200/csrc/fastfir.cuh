// JFastFir, the reference's streaming overlap-save FFT convolution (un-vendored jontio/JFFT; observable contract pinned by
// JAERO/tests/jfastfir_tests.cpp: out[n] = sum_k h[k] x[n-L-k], zeros for n < 2L), batched over channels. It serves the 8400 bps
// pre-filter (K6: 2049-tap RRC, nfft 4096, L 2048) and the burst demodulators' Hilbert filter (2048 taps, nfft 8192, L 6145).
//
// Every sample of a write is exchanged against the L-sample staging block: the caller's exchange kernel stores the new input in
// inblk and takes the output of the previous block from outblk, fusing its own per-sample work. When the staging block fills,
// fastfir_block_launch runs [K-1 history | L new] -> FFT -> xH -> inverse FFT -> last L outputs, scaled by 1/nfft, into outblk;
// the first block's output is zero. The history is the last K-1 samples of the concatenation.
#pragma once
#include <cuda_runtime.h>

namespace jb {

// channel-major, so that one CTA owns one channel's block
struct FastFir {
    int K, L, nfft;                       // taps, block length L = nfft - K + 1
    double2 *H, *tw;                      // FFT of the zero-padded kernel, W_nfft^k (shared by all channels)
    double2 *hist, *inblk, *outblk;       // [ch][K-1], [ch][L], [ch][L]
    int fill; long long blocks;           // host side: samples in the staging block, blocks transformed so far
};

// the (taps, nfft) pairs the block kernel is built for; both have L >= K-1
inline bool fastfir_size_supported(int K, int nfft) { return (nfft == 4096 && K == 2049) || (nfft == 8192 && K == 2048); }

int fastfir_block_launch(const FastFir &f, int n_channels, int first_block, cudaStream_t s);

} // namespace jb
