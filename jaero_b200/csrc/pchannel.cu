// P-channel frame layer on the GPU (SURVEY.md §8f rank 1): soft bits -> CRC-checked 12-byte signal units,
// one thread per channel, plus the data-carrier-detect (DCD) state machine that feeds back into the
// demodulators.
//
// Replaces the continuous (non-burst) branch of AeroL::Decode for 600 / 1200 / 10500 bps
// (JAERO/aerol.cpp:1124-1322 unique-word detection + header, :1540-1610 block fill, de-interleave,
// Decode_Continuous, DelayLine, scrambler, byte packing, CRC-16, :1990-2039 sync handling,
// AeroL::updateDCD :1109-1122) minus all text output. Three stages per call:
//   1. pchan_frame_kernel   bit-serial UW detectors, frame counter, block fill into a per-channel queue
//   2. viterbi (K5)         one launch per queue slot, de-interleave fused (viterbi.cu)
//   3. pchan_su_kernel      DelayLine dl2 (aerol.h:451-481) -> AeroLScrambler (aerol.h:397-437) ->
//                           LSB-first byte packing (:1568-1580) -> per-SU CRC (aerol.h:334-362) -> DCD countdown
// Integer/byte work throughout: bit-exact against the oracle. Known deviation, stated in DESIGN.md §8: CRC-driven
// updates of datacdcountdown (aerol.cpp:1601-1608) are applied after stage 3, i.e. at the end of the call that
// completed the frame, not in the middle of the bit loop. Two effects within one call: a UW sync after the frame's end
// (which sets the countdown to 12) comes before the frame's updates instead of after them, so the countdown and the DCD
// that later ticks leave can differ; and a frame whose CRCs raise DCD does not stop the 10.5 kbps detectors searching the
// rest of the call, so an exact UW copy in the next frame's data region syncs here and not in the reference.
#include <cstdint>
#include "viterbi.cuh"
#include "frame_stages.cuh"

namespace jb {

// PreambleDetector::Update (aerol.cpp:744-750): exact match, buffer zeroed on a hit
__device__ __forceinline__ int uw_exact(unsigned &sr, int bit)
{
    sr = (sr << 1) | (unsigned)bit;
    if (sr == UWORD) { sr = 0; return 1; }
    return 0;
}

// One soft bit through AeroL::Decode's continuous branch. Every lane of the channel's warp runs it with the same state
// (the state is warp-uniform); lane 0 does the stores.
__device__ __forceinline__ void pchan_frame_bit(const PChanParams &pp, PChanState &s, int ch, int v, int idle_idx, int lane)
{
    const int block_len = pp.block_len, QD = pp.queue;
    int bit = (((unsigned char)v) >= 128) ? 1 : 0;                           // aerol.cpp:1136-1139
    int soft_bit = (unsigned short)v;
    if (v < 0) return;                                                       // burst marker: never in continuous modes
    int gotsync;
    if (pp.oqpsk) {                                                          // :1156-1233
        // oqpsk_arm_search written out: through the shared stage (its invert_soft) this kernel's SASS changes
        s.realimag++; s.realimag %= 2;
        const bool search = (s.cntr > pp.number_of_bits - 68 || s.cntr <= 0 || !s.datacd);
        int inv;
        if (s.realimag) {                                                    // explicit arms: the state stays in registers
            if (search) gotsync = uw_phase_invariant<0>(s.sr_imag, bit, s.inv_imag);
            inv = s.inv_imag;
        } else {
            if (search) gotsync = uw_phase_invariant<0>(s.sr_real, bit, s.inv_real);
            inv = s.inv_real;
        }
        if (search) { if (!s.gotsync_last) { s.gotsync_last = gotsync; gotsync = 0; } else s.gotsync_last = 0; }
        else { gotsync = 0; s.gotsync_last = 0; }
        if (inv) { bit = 1 - bit; if (soft_bit != 128) soft_bit = 255 - soft_bit; }
    } else gotsync = uw_exact(s.sr_plain, bit);                              // :1269-1272

    if (s.cntr < CNTR_IDLE) s.cntr++;
    if (s.cntr < 16) {                                                       // :1275-1300
        if (s.cntr == 0) { s.frameinfo = (unsigned short)bit; s.info_len = 0; }
        else s.frameinfo = (unsigned short)((s.frameinfo << 1) | bit);
    }
    if (s.cntr == 15) {                                                      // :1301-1319
        const unsigned short t = s.frameinfo; s.frameinfo = s.lastframeinfo; s.lastframeinfo = t;
    }
    if (s.cntr >= 16) {                                                      // :1540-1552
        int idx;                                                             // (cntr-BitsInHeader)%block_len, negative -> 0
        if (s.cntr >= CNTR_IDLE) idx = idle_idx;
        else { idx = s.cntr - pp.bits_in_header; if (idx < 0) idx = 0; idx %= block_len; }
        // every slot holds a completed block the Viterbi stage has not decoded yet: this bit has nowhere to go. Flag it
        // (read_sus / get_stats report JAERO_E_OVERFLOW) instead of overwriting a queued block.
        if (s.blocks_ready >= QD) s.queue_overflow = 1;
        else if (lane == 0) pp.blocks[((size_t)ch * QD + s.blocks_ready) * block_len + idx] = (uint8_t)soft_bit;
        if (idx == block_len - 1) {
            // block complete: queue it for the Viterbi stage with what the SU stage needs to know
            if (s.blocks_ready < QD) {
                PChanBlockMeta m;
                const int nbits = s.first_decode_done ? block_len / 2 : block_len / 2 - (pp.paddinglength / 2 + 1);
                m.scr_pos = s.scr_pos; m.info_off = s.info_len; m.n_valid = nbits;
                m.frame_done = ((s.cntr - pp.bits_in_header) == (pp.number_of_bits - 1)) ? 1 : 0;   // :1582
                m.frame_index = s.nframes;
                if (lane == 0) pp.meta[(size_t)ch * QD + s.blocks_ready] = m;
                s.scr_pos += nbits;                                          // scrambler.update advances by deconvol.size()
                s.info_len += nbits / 8;                                     // whole bytes appended (:1568-1580)
                s.first_decode_done = 1;
                if (m.frame_done) s.nframes++;
                s.blocks_ready++;
            } else s.queue_overflow = 1;
            // The reference reuses one `block` buffer, so a block that completed without every position rewritten would carry
            // the previous block's values. That cannot happen while the counter runs: the index goes 0, 1, 2 ... (or back to 0
            // at a unique word), so by the time it reaches block_len-1 every position has been written since the last restart.
            // Only the idle index could complete a stale block, and only if it were block_len-1 (it is 2366 / 240 / 48 for the
            // three rates): then, and only then, the previous contents are copied forward.
            if (idle_idx == block_len - 1 && s.blocks_ready < QD) {
                __syncwarp();
                const uint8_t *srcb = pp.blocks + ((size_t)ch * QD + (s.blocks_ready - 1)) * block_len;
                uint8_t *dstb = pp.blocks + ((size_t)ch * QD + s.blocks_ready) * block_len;
                for (int k = lane; k < block_len; k += 32) dstb[k] = srcb[k];
                __syncwarp();
            }
        }
    }
    if (gotsync) {                                                           // :1990-2011
        s.cntr = -1; s.datacd = 1; s.datacdcountdown = 12; s.scr_pos = 0; s.dcd_rises++;
    }
    if (s.cntr + 1 == pp.total_number_of_bits) { s.scr_pos = 0; s.cntr = -1; }   // :2013-2016
}

// bits 0, 2, 4 ... of x packed into the low 16 bits
__device__ __forceinline__ unsigned even_bits(unsigned x)
{
    x &= 0x55555555u;
    x = (x | (x >> 1)) & 0x33333333u;
    x = (x | (x >> 2)) & 0x0f0f0f0fu;
    x = (x | (x >> 4)) & 0x00ff00ffu;
    x = (x | (x >> 8)) & 0x0000ffffu;
    return x;
}

// One warp per channel. The bit loop of AeroL::Decode is a state machine, but between its events it is regular: while the
// frame counter runs inside a block (or idles at 1e9) and no unique word appears, soft bit i + j goes to block position
// idx + j, the real / imaginary arm alternates, and nothing else changes. Those stretches are taken 32 bits at a time, one
// bit per lane (the unique-word shift registers of all 32 positions are formed from a ballot and compared in parallel);
// header bits, block completions, frame wrap, unique-word hits, LostSignal events and the 600 / 1200 bps framing take the
// bit-serial path above. Both paths apply the same updates, so the result does not depend on where the stretches end.
__global__ void __launch_bounds__(128)
pchan_frame_kernel(PChanParams pp, const int16_t *__restrict__ soft, const int *__restrict__ soft_count, int soft_cap,
                   int *__restrict__ demod_dcd /* may be null */, const int *__restrict__ lost_n /* may be null */,
                   const int *__restrict__ lost_pos, size_t lost_pitch)
{
    const int lane = threadIdx.x & 31;
    const int ch = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (ch >= pp.n_channels) return;
    PChanState s = pp.state[ch];
    const int n = soft_count[ch];
    const int16_t *bits = soft + (size_t)ch * soft_cap;
    const int block_len = pp.block_len, QD = pp.queue;
    // while the frame counter sits at its idle value 1e9 the block index is the constant (1e9 - BitsInHeader) % block_len
    const int idle_idx = (CNTR_IDLE - pp.bits_in_header) % block_len;
    s.blocks_ready = 0;
    // AeroL::LostSignal at the soft-bit positions the demodulator recorded its SignalStatus(false) events. LostCursor written
    // out: through it this kernel's SASS changes.
    int nev = lost_n ? min(lost_n[ch], LOST_CAP) : 0, ev = 0;
    if (lost_n && lost_n[ch] > LOST_CAP) s.queue_overflow = 1;
    int next_ev = nev ? lost_pos[ch] : 0x7fffffff;
    int i = 0;
    while (i < n) {
        while (i >= next_ev) { lost_signal(s); ev++; next_ev = ev < nev ? lost_pos[(size_t)ev * lost_pitch + ch] : 0x7fffffff; }
        int r = min(32, min(n, next_ev) - i);                                // bits this round may take (>= 1)
        const int v = (lane < r) ? (int)bits[i + lane] : 0;
        const unsigned negm = __ballot_sync(0xffffffffu, v < 0);
        if (negm) r = min(r, __ffs(negm) - 1);
        const int c = s.cntr;
        const bool idle = (c >= CNTR_IDLE);
        bool fast = pp.oqpsk && r > 0 && s.blocks_ready < QD;
        bool searching = true;
        int idx0 = idle_idx;
        if (fast && !idle) {
            // the counter runs: stay clear of the header (cntr < 16), the end of the block and the frame wrap
            fast = (c >= 16) && (c + 1 >= pp.bits_in_header);
            if (fast) {
                idx0 = (c + 1 - pp.bits_in_header) % block_len;
                r = min(r, block_len - 1 - idx0);
                r = min(r, pp.total_number_of_bits - 2 - c);
                searching = (!s.datacd) || (c > pp.number_of_bits - 68);
                if (!searching) r = min(r, pp.number_of_bits - 68 - c + 1);
                fast = r > 0;
            }
        } else if (fast) fast = (idle_idx != block_len - 1);
        if (fast) {
            const unsigned valid = (r == 32) ? 0xffffffffu : ((1u << r) - 1u);
            // lane j carries bit i + j; its arm: realimag after the increment
            const int a_imag = ((s.realimag + 1) & 1) ? 0 : 1;               // offset of the first imaginary-arm bit in this round
            const bool mine_imag = ((lane & 1) == a_imag);
            if (searching) {
                const int bit = (((unsigned char)v) >= 128) ? 1 : 0;
                const unsigned B = __ballot_sync(0xffffffffu, bit != 0) & valid;
                const unsigned E0 = even_bits(B), E1 = even_bits(B >> 1);    // bits of the even / odd lanes, in order
                const unsigned Em = (lane & 1) ? E1 : E0;
                const unsigned srp = mine_imag ? s.sr_imag : s.sr_real;
                const int k = lane >> 1;
                const unsigned W = (srp << (k + 1)) | (__brev(Em) >> (31 - k));   // the register after this lane's bit
                const bool hit = (lane < r) && (W == UWORD || W == ~UWORD);
                if (__any_sync(0xffffffffu, hit)) fast = false;              // a unique word inside the round: bit-serial
                else {
                    const int n0 = (r + 1) >> 1, n1 = r >> 1;                // bits taken by the even / odd lanes
                    const unsigned sr_e = s.sr_imag, sr_r = s.sr_real;
                    const unsigned imag_E = a_imag ? E1 : E0, real_E = a_imag ? E0 : E1;
                    const int imag_n = a_imag ? n1 : n0, real_n = a_imag ? n0 : n1;
                    if (imag_n) s.sr_imag = (sr_e << imag_n) | (__brev(imag_E) >> (32 - imag_n));
                    if (real_n) s.sr_real = (sr_r << real_n) | (__brev(real_E) >> (32 - real_n));
                }
            }
        }
        if (fast) {
            const bool mine_imag = ((lane & 1) == (((s.realimag + 1) & 1) ? 0 : 1));
            const int inv = mine_imag ? s.inv_imag : s.inv_real;
            int soft_bit = (unsigned short)v;
            if (inv && soft_bit != 128) soft_bit = 255 - soft_bit;
            uint8_t *blk = pp.blocks + ((size_t)ch * QD + s.blocks_ready) * block_len;
            if (idle) { if (lane == r - 1) blk[idle_idx] = (uint8_t)soft_bit; }      // every bit lands on the idle index: the last one stays
            else { if (lane < r) blk[idx0 + lane] = (uint8_t)soft_bit; s.cntr = c + r; }
            s.realimag = (s.realimag + r) & 1;
            s.gotsync_last = 0;
            i += r;
        } else {
            // one bit, serially (lane 0 holds bit i; a burst marker is only skipped)
            pchan_frame_bit(pp, s, ch, __shfl_sync(0xffffffffu, v, 0), idle_idx, lane);
            i++;
        }
    }
    if (ev < nev) lost_signal(s);                                            // events after the last soft bit
    s.bits_seen += n;
    // carry the partially filled block of slot `blocks_ready` back to slot 0 for the next call
    if (s.blocks_ready > 0 && s.blocks_ready < QD) s.carry_slot = s.blocks_ready; else s.carry_slot = 0;
    if (lane == 0) {
        pp.state[ch] = s;
        pp.ready[ch] = s.blocks_ready;
        if (demod_dcd) demod_dcd[ch] = s.datacd;
    }
}

// One warp per channel. The delay line, the scrambler and the byte packing are position-wise, so they run 32 decoded bits
// at a time (the delay line is far longer than 32, so a round's reads never see the round's own writes; the packed bytes are
// the ballot of the descrambled bits); the CRCs of a frame's signal units are computed one unit per lane, and only the
// DCD countdown and the output-ring bookkeeping walk the units in order.
__global__ void __launch_bounds__(128)
pchan_su_kernel(PChanParams pp, int *__restrict__ demod_dcd)
{
    const unsigned FULLM = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const int ch = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (ch >= pp.n_channels) return;
    PChanState s = pp.state[ch];
    const int block_len = pp.block_len, half = block_len / 2, QD = pp.queue, L = pp.dl2_len;
    uint8_t *dl2 = pp.dl2 + (size_t)ch * L;
    uint8_t *info = pp.infofield + (size_t)ch * pp.info_cap;
    for (int q = 0; q < s.blocks_ready; q++) {
        const PChanBlockMeta m = pp.meta[(size_t)ch * QD + q];
        const uint8_t *dec = pp.decoded + ((size_t)ch * QD + q) * half;
        int outb = m.info_off;
        // DelayLine::update (aerol.h:465-473) writes slot ptr and returns slot ptr+1, a value stored dl2_len-1 steps earlier
        for (int h0 = 0; h0 < m.n_valid; h0 += 32) {
            const int cnt = min(32, m.n_valid - h0);
            int rp = s.dl2_ptr + 1 + lane; if (rp >= L) rp -= L;
            int wp = s.dl2_ptr + lane; if (wp >= L) wp -= L;
            int b = 0; uint8_t newv = 0;
            if (lane < cnt) { b = dl2[rp]; newv = dec[h0 + lane]; b ^= g_scr[m.scr_pos + h0 + lane]; }   // aerol.h:421-429
            __syncwarp();
            if (lane < cnt) dl2[wp] = newv;
            __syncwarp();
            s.dl2_ptr += cnt; if (s.dl2_ptr >= L) s.dl2_ptr -= L;
            // LSB-first bytes (aerol.cpp:1568-1580): a trailing partial byte is dropped, as the reference drops ch8 at the next block
            const unsigned word = __ballot_sync(FULLM, b & 1);
            const int nbytes = cnt >> 3;
            if (lane < nbytes && outb + lane < pp.info_cap) info[outb + lane] = (uint8_t)(word >> (8 * lane));
            outb += nbytes;
        }
        if (m.frame_done) {                                                  // :1582-1610
            __syncwarp();
            const int nsu = outb / 12;
            for (int k0 = 0; k0 < nsu; k0 += 32) {
                const int k = k0 + lane;
                int ok = 0;
                if (k < nsu) {
                    const uint8_t *su = info + k * 12;
                    unsigned crc = 0xFFFF;                                   // AeroLcrc16::calcusingbytes (aerol.h:334-362)
                    int tsum = 0;
                    for (int i = 0; i < 10; i++) {
                        unsigned byte = su[i];
                        tsum += (int)byte;
                        for (int t = 0; t < 8; t++) { crc = crc16_step(crc, byte & 1u); byte >>= 1; }
                    }
                    unsigned crc_calc = (~crc) & 0xFFFFu;
                    const unsigned crc_rec = ((unsigned)su[11] << 8) | su[10];
                    if ((!crc_rec) && (crc_calc != crc_rec) && tsum == 0) crc_calc = 0;
                    ok = (crc_calc == crc_rec);
                }
                const int gcnt = min(32, nsu - k0);
                for (int j = 0; j < gcnt; j++) {
                    const int okj = __shfl_sync(FULLM, ok, j);
                    if (okj) { if (s.datacdcountdown < 12) s.datacdcountdown += 2; }
                    else { if (s.datacdcountdown > 0) s.datacdcountdown -= 3; }
                    if (!s.datacd && s.datacdcountdown > 2) { s.datacd = 1; s.dcd_rises++; }
                    if (s.su_count < pp.su_cap) {
                        uint8_t *o = pp.su_out + ((size_t)ch * pp.su_cap + s.su_count) * 16;
                        const uint8_t *su = info + (k0 + j) * 12;
                        if (lane < 12) o[lane] = su[lane];
                        else if (lane == 12) o[12] = (uint8_t)okj;
                        else if (lane == 13) o[13] = (uint8_t)(k0 + j);
                        else if (lane == 14) o[14] = (uint8_t)(m.frame_index & 255);
                        else if (lane == 15) o[15] = (uint8_t)((m.frame_index >> 8) & 255);
                        s.su_count++;
                    } else s.queue_overflow = 1;
                    s.su_total++; s.su_ok += okj;
                }
            }
        }
    }
    // move the partially filled block to slot 0
    if (s.carry_slot > 0) {
        const uint8_t *srcb = pp.blocks + ((size_t)ch * QD + s.carry_slot) * block_len;
        uint8_t *dstb = pp.blocks + ((size_t)ch * QD) * block_len;
        if ((block_len & 15) == 0) {
            const int4 *s4 = reinterpret_cast<const int4 *>(srcb); int4 *d4 = reinterpret_cast<int4 *>(dstb);
            for (int k = lane; k < block_len / 16; k += 32) d4[k] = s4[k];
        } else for (int k = lane; k < block_len; k += 32) dstb[k] = srcb[k];
        s.carry_slot = 0;
    }
    s.blocks_ready = 0;
    if (lane == 0) {
        pp.state[ch] = s;
        if (demod_dcd) demod_dcd[ch] = s.datacd;
    }
}

__global__ void pchan_init_kernel(PChanParams pp)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= pp.n_channels) return;
    PChanState s;
    memset(&s, 0, sizeof s);
    s.cntr = CNTR_IDLE;                      // aerol.cpp:899
    s.blockcnt = -1;
    pp.state[ch] = s;
}

// the signal-unit ring has been read out
__global__ void pchan_su_reset_kernel(PChanParams pp)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch < pp.n_channels) { pp.state[ch].su_count = 0; pp.state[ch].queue_overflow = 0; }
}

int pchan_process(const PChanParams &pp, const int16_t *d_soft, const int *d_soft_count, int soft_cap, int *demod_dcd,
                  uint8_t *vit_overlap, int *vit_overlap_len, int *vit_renorm, int *vit_valid, int max_queue, cudaStream_t st,
                  long long *launches, const int *lost_n, const int *lost_pos, size_t lost_pitch)
{
    pchan_frame_kernel<<<(pp.n_channels + 3) / 4, 128, 0, st>>>(pp, d_soft, d_soft_count, soft_cap, demod_dcd, lost_n, lost_pos, lost_pitch);
    JB_CUDA(cudaGetLastError());
    (*launches)++;
    for (int q = 0; q < max_queue; q++) {
        if (viterbi_launch(pp.blocks + (size_t)q * pp.block_len, pp.block_len, pp.cols, 0, pp.paddinglength, vit_overlap, vit_overlap_len,
                           vit_renorm, pp.decoded + (size_t)q * (pp.block_len / 2), vit_valid, pp.n_channels, st,
                           (size_t)pp.queue * pp.block_len, (size_t)pp.queue * (pp.block_len / 2), pp.ready, q)) return -1;
        (*launches)++;
    }
    pchan_su_kernel<<<(pp.n_channels + 3) / 4, 128, 0, st>>>(pp, demod_dcd);
    JB_CUDA(cudaGetLastError());
    (*launches)++;
    return 0;
}

} // namespace jb
