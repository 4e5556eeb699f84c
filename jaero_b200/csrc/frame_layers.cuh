// P-channel, C-channel and R/T frame layers: device data layouts and the kernels the C API launches (frame_layers.cu).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "common.cuh"

namespace jb {

static const int CNTR_IDLE = 1000000000;     // AeroL's frame counter while no frame runs (aerol.cpp:899, LostSignal aerol.h:927)

// ---------------------------------------------------------------- P-channel (pchannel.cu)
static const int PCHAN_QUEUE_MIN = 4;        // completed blocks a channel may queue within one process() call: at least this many;
                                             // PChanParams::queue is sized at create time from the demodulator's soft-bit ring
                                             // (2 s of soft bits) so that a full ring never overflows it

struct PChanState {                          // members of AeroL used by Decode (JAERO/aerol.h:937-1016)
    unsigned sr_plain, sr_imag, sr_real;     // preamble detector buffers as 32-bit shift registers
    int inv_imag, inv_real, realimag, gotsync_last;
    int cntr, blockcnt;
    unsigned short frameinfo, lastframeinfo;
    int datacdcountdown, datacd;
    int scr_pos, dl2_ptr, info_len, first_decode_done;
    int nframes, blocks_ready, carry_slot, queue_overflow;
    int su_count;                            // SUs waiting in the output ring
    long long su_total, su_ok, bits_seen;
    int dcd_rises;
};
struct PChanBlockMeta { int scr_pos, info_off, n_valid, frame_done, frame_index; };

struct PChanParams {
    int n_channels, oqpsk, cols, block_len, number_of_bits, bits_in_header, total_number_of_bits, paddinglength;
    int dl2_len, info_cap, su_cap;
    int queue;              // block slots per channel (>= PCHAN_QUEUE_MIN)
    PChanState *state;
    uint8_t *blocks;        // [ch][queue][block_len] interleaved soft values
    uint8_t *decoded;       // [ch][queue][block_len/2]
    PChanBlockMeta *meta;   // [ch][queue]
    int *ready;             // [ch] blocks queued by the frame stage
    uint8_t *dl2;           // [ch][dl2_len]
    uint8_t *infofield;     // [ch][info_cap]
    uint8_t *su_out;        // [ch][su_cap][16]: 12 SU bytes, crc_ok, index in frame, frame number (lo,hi)
};

__global__ void pchan_init_kernel(PChanParams pp);
__global__ void pchan_su_reset_kernel(PChanParams pp);
int pchan_process(const PChanParams &pp, const int16_t *d_soft, const int *d_soft_count, int soft_cap, int *demod_dcd,
                  uint8_t *vit_overlap, int *vit_overlap_len, int *vit_renorm, int *vit_valid, int max_queue, cudaStream_t st,
                  long long *launches, const int *lost_n = nullptr, const int *lost_pos = nullptr, size_t lost_pitch = 0);

// ---------------------------------------------------------------- C-channel, 8400 bps (cchannel.cu)
static const int CC_FRAME_BITS = 4096;     // AERO_SPEC_NumberOfBits (aerol.cpp:1039)
static const int CC_CODED = 5460;          // de-punctured soft values per frame (4095 + 1365 erasures)
static const int CC_CODED_PITCH = 5472;    // row pitch (16-byte multiple)
static const int CC_DEC = 2730;            // decoded bits per frame before resize(2714)
static const int CC_KEEP = 2714;
static const int CC_QUEUE = 4;             // frames that may complete per channel in one call
static const int CC_SLOTS = CC_QUEUE + 1;  // code-order rows per channel: the queue and the frame still being filled after it
static const int CC_OUT = 8;               // decoded frames held per channel until read
static const int CC_RECORD = 352;          // 3 x (12 SU bytes + crc flag + 3 pad) + 300 voice bytes + 4 (frame number)

struct CChanState {
    unsigned long long b1_real, b2_real, b1_imag, b2_imag;     // OQPSKPreambleDetectorAndAmbiguityCorrection x2 (52-bit registers)
    int inv_real, inv_imag, realimag, gotsync_last;
    int cntr, index, datacd, datacdcountdown;
    int dl2_ptr, frames_ready, carry_slot, nframes, out_count, overflow;
    long long bits_seen, su_total, su_ok;
};
struct CChanParams {
    int n_channels, dl2_len;
    CChanState *state;
    uint8_t *coded;         // [ch][CC_SLOTS][CC_CODED_PITCH] code-order soft values (erasures = 128 pre-filled)
    uint8_t *decoded;       // [ch][CC_QUEUE][CC_DEC]
    int *ready;             // [ch]
    uint8_t *dl2;           // [ch][dl2_len]
    uint8_t *out;           // [ch][CC_OUT][CC_RECORD]
};

__global__ void cchan_init_kernel(CChanParams cp);
int cchan_process(const CChanParams &cp, const int16_t *d_soft, const int *d_soft_count, size_t soft_stride, int *demod_dcd,
                  uint8_t *vit_overlap, int *vit_overlap_len, int *vit_renorm, int *vit_valid, cudaStream_t st, long long *launches,
                  const int *lost_n = nullptr, const int *lost_pos = nullptr, size_t lost_pitch = 0);

// ---------------------------------------------------------------- R/T burst channel (rtchannel.cu)
static const int RT_BLOCK = 64 * 95;       // RTChannelDeleaveFECScram::block (aerol.h:575)
static const int RT_SLOTS = 8;             // packets that may be open per channel between two trial passes
static const int RT_OUT = 8;               // decoded packets held per channel until read
static const int RT_OUT_BYTES = 400;       // 16-byte header + up to 379 payload bytes

struct RtState {                           // AeroL members used by the burst branch of Decode (aerol.h:937-1016)
    unsigned sr_imag, sr_real, sr_msk;
    int inv_imag, inv_real, inv_msk, realimag, gotsync_last;
    int cntr, muw, datacd, datacdcountdown;
    int slot_head, slot_cur, n_open;
    int rc, lastpacketstate, n_bad, n_trials, out_count, overflow;
    long long bits_seen;
};
struct RtSlot { int fill, next_trial, done, closed, targetSUSize, targetBlocks; long long start_bit; };

struct RtParams {
    int n_channels, oqpsk, ifb, number_of_bits, total_number_of_bits;
    RtState *state;
    RtSlot *slots;          // [ch][RT_SLOTS]
    uint8_t *blocks;        // [ch][RT_SLOTS][RT_BLOCK] soft values in arrival order
    uint8_t *out;           // [ch][RT_OUT][RT_OUT_BYTES]
};

__global__ void rt_init_kernel(RtParams rp);
int rt_process(const RtParams &rp, const int16_t *d_soft, const int *d_soft_count, size_t soft_stride, cudaStream_t st, long long *launches, int vmode = 0);

// ---------------------------------------------------------------- shared by the layers (frame_stages.cuh)
int frame_set_scrambler();                 // AeroLScrambler::pre_state into the current device's tables, which the kernels read
// One launch, one thread per channel, on stream st (frame_stages.cuh). State is PChanState, CChanState or RtState; demod_dcd
// (may be null) receives the channel's new DCD.
// AeroL::updateDCD, the reference's 1 s timer
template <class State> int frame_tick(State *state, int n_channels, int *demod_dcd, cudaStream_t st);
// AeroL::LostSignal on one channel (>= 0) or all (-1); P- and C-channel
template <class State> int frame_lost(State *state, int n_channels, int channel, int *demod_dcd, cudaStream_t st);
// the decoded-record queue has been read out: its count and overflow flag start again; C-channel and R/T
template <class State> int frame_out_reset(State *state, int n_channels, cudaStream_t st);

// a kernel with one thread per channel
template <class K, class... A> int per_channel_launch(K kernel, int n_channels, cudaStream_t st, A... args)
{
    kernel<<<(n_channels + 127) / 128, 128, 0, st>>>(args...);
    JB_CUDA(cudaGetLastError());
    return 0;
}

} // namespace jb
