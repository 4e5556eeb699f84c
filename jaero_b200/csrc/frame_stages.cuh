// The pieces of AeroL (JAERO/aerol.cpp, aerol.h) that the P-channel, C-channel and R/T frame layers share, written once.
// Each layer keeps its own state struct and frame logic; the stages below take the state by reference.
#pragma once
#include "frame_layers.cuh"
#include "demod.cuh"                         // LOST_CAP

namespace jb {

static const unsigned UWORD = 0xE15AE893u;   // the unique word (aerol.cpp:947)

// AeroLScrambler::pre_state (aerol.h:397-437), the first 5000 bits of the scrambler sequence, in each memory space a kernel reads
// it from: global for the P-channel SU kernel (each lane reads its own entry), constant for the C-channel and R/T kernels.
__device__ uint8_t g_scr[5000];
__constant__ uint8_t c_scr[5000];

int frame_set_scrambler()
{
    uint8_t seq[5000];
    int st[15] = {1, 1, 0, 1, 0, 0, 1, 0, 1, 0, 1, 1, 0, 0, 1};
    for (int a = 0; a < 5000; a++) { const int v = st[0] ^ st[14]; seq[a] = (uint8_t)v; for (int i = 14; i > 0; i--) st[i] = st[i - 1]; st[0] = v; }
    JB_CUDA(cudaMemcpyToSymbol(g_scr, seq, sizeof seq));
    JB_CUDA(cudaMemcpyToSymbol(c_scr, seq, sizeof seq));
    return 0;
}

// AeroL::updateDCD (aerol.cpp:1109-1122)
template <class S> __device__ __forceinline__ void dcd_tick(S &s)
{
    if (s.datacdcountdown > 0) s.datacdcountdown -= 3;
    else if (s.datacdcountdown < 0) s.datacdcountdown = 0;
    if (s.datacd && !s.datacdcountdown) s.datacd = 0;
}

// AeroL::LostSignal (aerol.h:925-931); also the burst time-out (aerol.cpp:2018-2026) resets the same three members
template <class S> __device__ __forceinline__ void lost_signal(S &s)
{
    s.cntr = CNTR_IDLE; s.datacdcountdown = 0; s.datacd = 0;
}

// LostSignal at the soft-bit positions where the demodulator recorded its SignalStatus(false) events (lost_n may be null:
// none). take(s, i) applies the events at or before bit i; finish(s) those after the last bit.
struct LostCursor {
    const int *pos; size_t pitch; int ch, n, k, next;
    __device__ __forceinline__ LostCursor(const int *lost_n, const int *lost_pos, size_t lost_pitch, int ch_, int &overflow)
        : pos(lost_pos), pitch(lost_pitch), ch(ch_), k(0)
    {
        n = lost_n ? min(lost_n[ch], LOST_CAP) : 0;
        if (lost_n && lost_n[ch] > LOST_CAP) overflow = 1;
        next = n ? pos[ch] : 0x7fffffff;
    }
    template <class S> __device__ __forceinline__ void take(S &s, int i)
    {
        while (i >= next) { lost_signal(s); k++; next = k < n ? pos[(size_t)k * pitch + ch] : 0x7fffffff; }
    }
    template <class S> __device__ __forceinline__ void finish(S &s) const { if (k < n) lost_signal(s); }
};

// a phase-inverted arm: the hard bit flips and the soft value mirrors about 128 (aerol.cpp:1203-1231, :1255-1266, :2255-2281)
__device__ __forceinline__ void invert_soft(int &bit, int &soft_bit)
{
    bit = 1 - bit;
    if (soft_bit != 128) soft_bit = 255 - soft_bit;
}

// PreambleDetectorPhaseInvariant::Update (aerol.cpp:781-804) with tollerence TOL, the buffer a 32-bit shift register
template <int TOL> __device__ __forceinline__ int uw_phase_invariant(unsigned &sr, int bit, int &inverted)
{
    sr = (sr << 1) | (unsigned)bit;
    if constexpr (TOL == 0) {                // xorsum 32 or 0: compared directly, which keeps pchan_frame_kernel's SASS as it was
        if (sr == ~UWORD) { inverted = 1; return 1; }
        if (sr == UWORD) { inverted = 0; return 1; }
        return 0;
    }
    const int xorsum = __popc(sr ^ UWORD);
    if (xorsum >= 32 - TOL) { inverted = 1; return 1; }
    if (xorsum <= TOL) { inverted = 0; return 1; }
    return 0;
}

// The OQPSK branch of AeroL::Decode and DecodeC (aerol.cpp:1156-1233, :2205-2281): the bits alternate between two arms, each
// with its own unique-word detector and inversion flag. The arm's detector runs only while `search`; of two hits in a row (one
// per arm) the first is suppressed. detect(arm, bit, inv) runs the detector of arm 1 (realimag after the toggle) or arm 0.
// Returns gotsync; bit and soft_bit come back corrected for the arm's inversion.
template <class Detect>
__device__ __forceinline__ int oqpsk_arm_search(int &realimag, int &gotsync_last, int &inv1, int &inv0, bool search, int &bit,
                                                int &soft_bit, Detect detect)
{
    int gotsync = 0, inv;
    realimag++; realimag %= 2;
    if (realimag) { if (search) gotsync = detect(1, bit, inv1); inv = inv1; }
    else { if (search) gotsync = detect(0, bit, inv0); inv = inv0; }
    if (search) { if (!gotsync_last) { gotsync_last = gotsync; gotsync = 0; } else gotsync_last = 0; }
    else { gotsync = 0; gotsync_last = 0; }
    if (inv) invert_soft(bit, soft_bit);
    return gotsync;
}

// AeroLcrc16 (aerol.h:287-362): one message bit into the CRC-16 register (polynomial 0x8408, LSB first)
__device__ __forceinline__ unsigned crc16_step(unsigned crc, unsigned mb)
{
    const unsigned cb = crc & 1u;
    crc >>= 1;
    if (cb ^ mb) crc ^= 0x8408u;
    return crc;
}
// calcusingbytes (aerol.h:334-362): n bytes, each LSB first
__device__ __forceinline__ unsigned crc16_bytes(const uint8_t *bytes, int n)
{
    unsigned crc = 0xFFFF;
    for (int i = 0; i < n; i++) {
        unsigned byte = bytes[i];
        for (int t = 0; t < 8; t++) { crc = crc16_step(crc, byte & 1u); byte >>= 1; }
    }
    return (~crc) & 0xFFFFu;
}
// calcusingbitsandcheck (aerol.h:287-313): n bits, one per byte, the last 16 of them the received CRC
__device__ __forceinline__ bool crc16_bits_ok(const uint8_t *bits, int n)
{
    unsigned crc_rec = 0;
    for (int i = n - 1; i >= n - 16; i--) { crc_rec <<= 1; crc_rec |= bits[i]; }
    unsigned crc = 0xFFFF;
    for (int i = 0; i < n - 16; i++) crc = crc16_step(crc, bits[i]);
    return crc_rec == ((~crc) & 0xFFFFu);
}

template <class State> __global__ void frame_tick_kernel(State *state, int n_channels, int *demod_dcd)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= n_channels) return;
    State &s = state[ch];
    dcd_tick(s);
    if (demod_dcd) demod_dcd[ch] = s.datacd;
}

template <class State> __global__ void frame_lost_kernel(State *state, int n_channels, int channel, int *demod_dcd)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= n_channels || (channel >= 0 && channel != ch)) return;
    lost_signal(state[ch]);
    if (demod_dcd) demod_dcd[ch] = 0;
}

// The read has copied out the state with its overflow flag, which reported every record lost since the previous read: both
// start again, so one overflow fails one read, not every later one.
template <class State> __global__ void frame_out_reset_kernel(State *state, int n_channels)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch < n_channels) { state[ch].out_count = 0; state[ch].overflow = 0; }
}

// The C API launches the kernels above through these: a template kernel is launched only in the unit that defines it, and
// frame_layers.cu instantiates these for the layers that use them.
template <class State> int frame_tick(State *state, int n_channels, int *demod_dcd, cudaStream_t st)
{
    return per_channel_launch(frame_tick_kernel<State>, n_channels, st, state, n_channels, demod_dcd);
}
template <class State> int frame_lost(State *state, int n_channels, int channel, int *demod_dcd, cudaStream_t st)
{
    return per_channel_launch(frame_lost_kernel<State>, n_channels, st, state, n_channels, channel, demod_dcd);
}
template <class State> int frame_out_reset(State *state, int n_channels, cudaStream_t st)
{
    return per_channel_launch(frame_out_reset_kernel<State>, n_channels, st, state, n_channels);
}

} // namespace jb
