// C-channel (8400 bps) frame layer (SURVEY.md §8(f)3): soft bits -> per frame 3 sub-band signal units + 25 voice frames.
//
// Replaces AeroL::DecodeC (JAERO/aerol.cpp:2187-2500): dual unique-word detector with I/Q ambiguity correction
// (OQPSKPreambleDetectorAndAmbiguityCorrection, :848-896, tollerence 6), 16 x (64 x 4) block de-interleave
// (:2308-2319), PuncturedCode::depunture_soft_block(...,4) (:2505-2518), Decode_Continuous (K5), DelayLine dl2,
// AeroLScrambler, the 24 x 12-bit sub-band field -> three 12-byte signal units with CRC-16 and the DCD countdown
// (:2342-2385), and the 25 x 96-bit voice payload (:2457-2479); minus text output and the vocoder. Three stages per call:
//   1. cchan_frame_kernel   thread per channel: bit-serial detectors; every frame bit is scattered straight to its
//                           de-interleaved, de-punctured code-order position (erasure slots are pre-filled with 128)
//   2. viterbi (K5)         one launch per queue slot, continuous mode (overlap + padding carried per channel)
//   3. cchan_su_kernel      dl2 -> scrambler -> signal units + CRC + DCD -> voice bytes
// Integer/byte work throughout: bit-exact against the oracle (oracle/restated/fec_oracle.cpp CChannelOracle).
#include <cstdint>
#include "viterbi.cuh"
#include "frame_stages.cuh"

namespace jb {

static const unsigned long long CC_PRE1 = 216866263330005ULL, CC_PRE2 = 3012071630031408ULL;   // aerol.cpp:953-954
static const unsigned long long CC_MASK = (1ULL << 52) - 1;

// OQPSKPreambleDetectorAndAmbiguityCorrection::Update: the second buffer only shifts when the first does not match
__device__ __forceinline__ int cc_uw(unsigned long long &b1, unsigned long long &b2, int val, int &inverted)
{
    b1 = ((b1 << 1) | (unsigned long long)val) & CC_MASK;
    int xorsum = __popcll(b1 ^ CC_PRE1);
    if (xorsum >= 52 - 6) { inverted = 1; return 1; }
    if (xorsum <= 6) { inverted = 0; return 1; }
    b2 = ((b2 << 1) | (unsigned long long)val) & CC_MASK;
    xorsum = __popcll(b2 ^ CC_PRE2);
    if (xorsum >= 52 - 6) { inverted = 1; return 1; }
    if (xorsum <= 6) { inverted = 0; return 1; }
    return 0;
}

__global__ void __launch_bounds__(64)
cchan_frame_kernel(CChanParams cp, const int16_t *__restrict__ soft, const int *__restrict__ soft_count, size_t soft_stride,
                   const int *__restrict__ lost_n /* may be null */, const int *__restrict__ lost_pos, size_t lost_pitch)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= cp.n_channels) return;
    CChanState s = cp.state[ch];
    const int n = soft_count[ch];
    const int16_t *bits = soft + (size_t)ch * soft_stride;
    uint8_t *coded = cp.coded + (size_t)ch * CC_SLOTS * CC_CODED_PITCH;
    if (s.carry_slot > 0) {
        // the frame that was being filled when the previous call ended sits in slot `carry_slot`: it continues in slot 0
        const int4 *src = reinterpret_cast<const int4 *>(coded + (size_t)s.carry_slot * CC_CODED_PITCH);
        int4 *dst = reinterpret_cast<int4 *>(coded);
        for (int k = 0; k < CC_CODED_PITCH / 16; k++) dst[k] = src[k];
        s.carry_slot = 0;
    }
    s.frames_ready = 0;
    LostCursor lost(lost_n, lost_pos, lost_pitch, ch, s.overflow);
    for (int i = 0; i < n; i++) {
        lost.take(s, i);
        const int v = bits[i];
        s.bits_seen++;
        int bit = (((unsigned char)v) >= 128) ? 1 : 0;
        int soft_bit = (unsigned short)v;
        const bool search = (s.cntr > CC_FRAME_BITS - 112 || s.cntr <= 0);                   // :2212,2236
        const int gotsync = oqpsk_arm_search(s.realimag, s.gotsync_last, s.inv_real, s.inv_imag, search, bit, soft_bit,
            [&](int arm, int b, int &inv) { return arm ? cc_uw(s.b1_real, s.b2_real, b, inv) : cc_uw(s.b1_imag, s.b2_imag, b, inv); });
        if (gotsync) { s.cntr = -1; s.index = -1; }                                           // :2286-2296
        else {
            if (s.cntr < CNTR_IDLE) s.cntr++;
            if (s.cntr <= CC_FRAME_BITS - 1) {
                // block[index] -> deinterleave_ba(block,4) -> append -> depuncture: the code-order slot of frame bit c
                const int c = s.cntr, b = c >> 8, idx = c & 255, r = idx >> 2, j = idx & 3;
                const int k = j * 64 + ((r * 19) & 63);                                       // 19 = 27^-1 mod 64
                const int p = 256 * b + k;
                // row frames_ready: after a full queue the next frame still has a row, so it can finish in the next call
                if (p < CC_FRAME_BITS - 1) coded[(size_t)s.frames_ready * CC_CODED_PITCH + p + p / 3] = (uint8_t)soft_bit;
            }
            if (s.cntr == CC_FRAME_BITS - 1) {                                                 // frame complete
                if (s.frames_ready < CC_QUEUE) s.frames_ready++; else s.overflow = 1;    // a fifth frame in one call is lost (reported)
            }
        }
    }
    lost.finish(s);
    s.carry_slot = s.frames_ready;
    cp.state[ch] = s;
    cp.ready[ch] = s.frames_ready;
}

__global__ void __launch_bounds__(64)
cchan_su_kernel(CChanParams cp, int *__restrict__ demod_dcd)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= cp.n_channels) return;
    CChanState s = cp.state[ch];
    uint8_t *dl2 = cp.dl2 + (size_t)ch * cp.dl2_len;
    for (int q = 0; q < s.frames_ready; q++) {
        uint8_t *dec = cp.decoded + ((size_t)ch * CC_QUEUE + q) * CC_DEC;
        // deconvol.resize(2714); dl2.update; scrambler.update (reset at the frame's unique word)   :2326-2333
        for (int h = 0; h < CC_KEEP; h++) {
            int b = dec[h];
            dl2[s.dl2_ptr] = (uint8_t)b; s.dl2_ptr++; if (s.dl2_ptr >= cp.dl2_len) s.dl2_ptr = 0; b = dl2[s.dl2_ptr];
            dec[h] = (uint8_t)(b ^ c_scr[h]);
        }
        uint8_t *rec = nullptr;
        if (s.out_count < CC_OUT) rec = cp.out + ((size_t)ch * CC_OUT + s.out_count) * CC_RECORD; else s.overflow = 1;
        uint8_t info[12]; int ninfo = 0, charptr = 0, nsu = 0; unsigned ch8 = 0;
        for (int y = 0; y < 24; y++) {                                           // :2342-2385
            const int offset = y * (1 + 96 + 12);
            for (int h = offset + 97; h < offset + 109; h++) {
                ch8 |= (unsigned)dec[h] * 128u;
                charptr++; charptr %= 8;
                if (charptr == 0) { info[ninfo++] = (uint8_t)ch8; ch8 = 0; } else ch8 >>= 1;
            }
            if (ninfo == 12) {
                const unsigned crc_calc = crc16_bytes(info, 10);
                const unsigned crc_rec = ((unsigned)info[11] << 8) | info[10];
                const int ok = crc_calc == crc_rec;
                if (ok) { if (s.datacdcountdown < 12) s.datacdcountdown += 2; }
                else { if (s.datacdcountdown > 0) s.datacdcountdown -= 5; }
                if (!s.datacd && s.datacdcountdown > 2) s.datacd = 1;
                s.su_total++; s.su_ok += ok;
                if (rec && nsu < 3) { for (int b = 0; b < 12; b++) rec[nsu * 16 + b] = info[b]; rec[nsu * 16 + 12] = (uint8_t)ok; }
                nsu++; ninfo = 0;
            }
        }
        int bitsin = 0, vb = 0;
        for (int h = 1; h < CC_KEEP; h++) {                                      // :2457-2479
            ch8 |= (unsigned)dec[h] * 128u;
            charptr++; charptr %= 8;
            if (charptr == 0) { if (rec && vb < 300) rec[48 + vb] = (uint8_t)ch8; vb++; ch8 = 0; } else ch8 >>= 1;
            bitsin++;
            if (bitsin == 96) { bitsin = 0; h += 13; }
        }
        if (rec) { *reinterpret_cast<int *>(rec + 348) = s.nframes; s.out_count++; }
        s.nframes++;
    }
    s.frames_ready = 0;
    cp.state[ch] = s;
    if (demod_dcd) demod_dcd[ch] = s.datacd;
}

__global__ void cchan_init_kernel(CChanParams cp)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= cp.n_channels) return;
    CChanState s;
    memset(&s, 0, sizeof s);
    s.cntr = CNTR_IDLE;                                        // AeroL ctor (aerol.cpp:907,927); index = 0 (:957)
    cp.state[ch] = s;
    uint8_t *coded = cp.coded + (size_t)ch * CC_SLOTS * CC_CODED_PITCH;
    for (int q = 0; q < CC_SLOTS; q++) for (int k = 0; k < CC_CODED_PITCH; k++) coded[(size_t)q * CC_CODED_PITCH + k] = 128;   // erasure slots
}

int cchan_process(const CChanParams &cp, const int16_t *d_soft, const int *d_soft_count, size_t soft_stride, int *demod_dcd,
                  uint8_t *vit_overlap, int *vit_overlap_len, int *vit_renorm, int *vit_valid, cudaStream_t st, long long *launches,
                  const int *lost_n, const int *lost_pos, size_t lost_pitch)
{
    const int grid = (cp.n_channels + 63) / 64;
    cchan_frame_kernel<<<grid, 64, 0, st>>>(cp, d_soft, d_soft_count, soft_stride, lost_n, lost_pos, lost_pitch);
    JB_CUDA(cudaGetLastError());
    (*launches)++;
    for (int q = 0; q < CC_QUEUE; q++) {
        if (viterbi_launch(cp.coded + (size_t)q * CC_CODED_PITCH, CC_CODED, 0, 0, 24, vit_overlap, vit_overlap_len, vit_renorm,
                           cp.decoded + (size_t)q * CC_DEC, vit_valid, cp.n_channels, st, (size_t)CC_SLOTS * CC_CODED_PITCH, (size_t)CC_QUEUE * CC_DEC,
                           cp.ready, q)) return -1;
        (*launches)++;
    }
    cchan_su_kernel<<<grid, 64, 0, st>>>(cp, demod_dcd);
    JB_CUDA(cudaGetLastError());
    (*launches)++;
    return 0;
}

} // namespace jb
