// R/T burst channel layer (SURVEY.md §8(f)2): soft bits with -1 start-of-burst markers -> R / T packets.
//
// Replaces the burst branch of AeroL::Decode (JAERO/aerol.cpp:1124-1350 unique-word detection with the burst timing
// gates, :1985-2031 sync / time-out handling, AeroL::updateDCD :1109-1122) and RTChannelDeleaveFECScram
// (JAERO/aerol.h:554-895: block fill, trial de-interleave at every candidate length, Decode_soft, AeroLScrambler,
// CRC-16 decisions, LSB-first byte packing), minus all text output / ACARS parsing. Two stages per call:
//   1. rt_frame_kernel   thread per channel: bit-serial detectors (tolerance 4), muw / cntr logic, fills the packet slots.
//                        Nothing the trial decodes decide feeds back into this stage (a successful decode only makes the
//                        reference ignore later bits of the same packet), so the decodes can run afterwards.
//   2. rt_trial_kernel   warp per channel: for every open packet slot, the reference's sequence of trial decodes in order
//                        (K5 Viterbi core, block mode; the renormalisation counter persists across trials exactly as the
//                        reference's single JConvolutionalCodec does), descramble, CRC-16 per lane, decision, packing.
// Integer / byte work: bit-exact against the oracle (oracle/restated/fec_oracle.cpp RTChannelOracle).
// Known deviation (DESIGN.md): the reference returns from Decode() in the middle of a 32-value vector when the burst
// time-out fires (aerol.cpp:2018-2027) and so drops the rest of that vector; here the stream is processed without drops.
#include <cstdint>
#include "viterbi_core.cuh"
#include "frame_stages.cuh"

namespace jb {

enum { RT_OK_R = 3, RT_OK_T = 5, RT_BAD = 0, RT_TEST_FAILED = 32, RT_NOTHING = 8 };

__global__ void __launch_bounds__(64)
rt_frame_kernel(RtParams rp, const int16_t *__restrict__ soft, const int *__restrict__ soft_count, size_t soft_stride, int vmode)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= rp.n_channels) return;
    RtState s = rp.state[ch];
    const int n = soft_count[ch];
    const int16_t *bits = soft + (size_t)ch * soft_stride;
    RtSlot *slots = rp.slots + (size_t)ch * RT_SLOTS;
    uint8_t *blocks = rp.blocks + (size_t)ch * RT_SLOTS * RT_BLOCK;
    int cur = s.slot_cur;
    int fill = slots[cur].fill;
    // vmode != 0: the reference's vector semantics. AeroL::Decode is called once per emitted soft-bit vector and RETURNS when the
    // burst time-out fires (aerol.cpp:2018-2027), dropping the rest of that vector. vmode > 0: the soft ring holds whole vectors of
    // the burst demodulator, vmode values each, one more when a vector opens with the start-of-burst marker (the demodulators clear
    // their buffer, push -1, then add pairs until >= vmode); vmode < 0: the whole call is one vector (host-supplied soft bits).
    int vec_left = 0; bool skipping = false;
    for (int i = 0; i < n; i++) {
        const int v = bits[i];
        if (vmode) {
            if (vec_left == 0) { vec_left = vmode > 0 ? vmode + (v < 0 ? 1 : 0) : n; skipping = false; }
            vec_left--;
            if (skipping) continue;
        }
        s.bits_seen++;
        int bit = (((unsigned char)v) >= 128) ? 1 : 0;                       // aerol.cpp:1136-1139
        int soft_bit = (unsigned short)v;
        if (v < 0) { s.muw = 0; continue; }                                  // :1146-1151
        if (s.muw < 100000) s.muw++;
        int gotsync = 0;
        if (rp.oqpsk) {                                                      // :1156-1233
            const bool search = (s.cntr > rp.number_of_bits - 68 || s.cntr <= 0 || !s.datacd);
            gotsync = oqpsk_arm_search(s.realimag, s.gotsync_last, s.inv_imag, s.inv_real, search, bit, soft_bit,
                                       [&](int arm, int b, int &inv) { return uw_phase_invariant<4>(arm ? s.sr_imag : s.sr_real, b, inv); });
            if (gotsync) { if (rp.ifb == 10500 && (abs(s.muw - 80) > 150)) gotsync = 0; }   // :1193-1200
        } else {                                                             // :1236-1266
            const int inverted = s.inv_msk;
            gotsync = uw_phase_invariant<4>(s.sr_msk, bit, s.inv_msk);
            if (s.muw > 250 && gotsync) { if (inverted != s.inv_msk) s.inv_msk = inverted; gotsync = 0; }
            if (s.inv_msk) invert_soft(bit, soft_bit);
        }
        if (s.cntr < CNTR_IDLE) s.cntr++;
        if (s.cntr < 16) {                                                   // :1275-1300
            if (s.cntr == 0) {
                s.cntr = 16;
                // rtchanneldeleavefecscram.resetblockptr(): a new packet slot
                slots[cur].fill = fill; slots[cur].closed = 1;
                if (s.n_open < RT_SLOTS) { cur++; if (cur >= RT_SLOTS) cur = 0; s.n_open++; }
                else s.overflow = 1;                                         // no slot left: the oldest pending packet of this call is lost (reported)
                RtSlot ns; ns.fill = 0; ns.next_trial = rp.oqpsk ? 64 * 2 : 64 * 5; ns.done = 0; ns.closed = 0; ns.targetSUSize = 0; ns.targetBlocks = 0; ns.start_bit = s.bits_seen;
                slots[cur] = ns;
                fill = 0;
            }
        }
        if (s.cntr >= 16) {                                                  // :1327-1345 block[blockptr++]=soft_bit
            if (fill < RT_BLOCK) { blocks[(size_t)cur * RT_BLOCK + fill] = (uint8_t)soft_bit; fill++; }
        }
        if (gotsync) { s.cntr = -1; s.datacd = 1; s.datacdcountdown = 12; }  // :1990-2011
        if (s.cntr + 1 == rp.total_number_of_bits) { lost_signal(s); if (vmode) skipping = true; }   // burst time-out :2013-2029
    }
    slots[cur].fill = fill;
    s.slot_cur = cur;
    rp.state[ch] = s;
}

__global__ void __launch_bounds__(128)
rt_trial_kernel(RtParams rp, int smem_per_warp, int sbuf_bytes)
{
    extern __shared__ __align__(16) unsigned char rt_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int ch = blockIdx.x * (blockDim.x >> 5) + warp;
    if (ch >= rp.n_channels) return;
    unsigned char *base = rt_smem + (size_t)warp * smem_per_warp;
    uint8_t *sbuf = base;
    uint2 *hist = reinterpret_cast<uint2 *>(base + sbuf_bytes);
    uint8_t *obits = reinterpret_cast<uint8_t *>(hist + V_CAP);
    RtState *sp = rp.state + ch;
    RtSlot *slots = rp.slots + (size_t)ch * RT_SLOTS;
    int rc = sp->rc, lastpacketstate = sp->lastpacketstate, n_bad = sp->n_bad, out_count = sp->out_count, trials = sp->n_trials;
    int head = sp->slot_head, n_open = sp->n_open;
    const int cur = sp->slot_cur;
    for (int q = 0, sidx = head; q < n_open; q++, sidx = (sidx + 1 == RT_SLOTS ? 0 : sidx + 1)) {
        RtSlot sl = slots[sidx];
        const uint8_t *block = rp.blocks + ((size_t)ch * RT_SLOTS + sidx) * RT_BLOCK;
        // the reference evaluates a trial as soon as blockptr reaches a candidate length; after OK the packet is closed
        while (!sl.done && sl.next_trial <= sl.fill && sl.next_trial <= RT_BLOCK) {
            const int bp = sl.next_trial, nblk = bp / 64;
            bool run = true;
            if (!rp.oqpsk) run = (nblk == 5 || nblk == sl.targetBlocks || nblk == 11 || nblk == 50);   // aerol.h:649-652
            if (run) {
                // ---- de-interleave into code order (deinterleave_ba / deinterleaveMSK_ba)
                for (int k = lane; k < bp; k += 32) {
                    const int i = k & 63, j = k >> 6;
                    int entry;
                    if (rp.oqpsk) entry = ((i * 27) & 63) * nblk + j;
                    else if (j < 5) entry = ((i * 27) & 63) * 5 + j;
                    else { const int g = (j - 5) / 3, jj = (j - 5) - 3 * g; entry = 64 * (5 + 3 * g) + (((i * 27) & 63) * 3 + jj); }
                    sbuf[k] = block[entry];
                }
                const int sets = bp >> 1;
                for (int k = lane; k < sets; k += 32) obits[k] = 0;
                __syncwarp();
                viterbi_decode_warp(sbuf, sets, hist, obits, rc, lane);
                __syncwarp();
                for (int k = lane; k < sets; k += 32) obits[k] ^= c_scr[k];            // scrambler.reset(); scrambler.update(deconvol)
                __syncwarp();
                trials++;
                int result = RT_NOTHING, nsus = 0, nbytes = 0;
                if (bp == 64 * 5) {                                                       // R packet test
                    if (!rp.oqpsk) { sl.targetSUSize = 0; sl.targetBlocks = 0; }
                    const bool ok = crc16_bits_ok(obits, 8 * 19);                             // every lane computes the same value
                    if (ok) { result = RT_OK_R; nbytes = 19; }
                    else if (rp.oqpsk) result = RT_TEST_FAILED;
                } else {
                    const bool hdr = crc16_bits_ok(obits, 8 * 6);
                    if (rp.oqpsk) {                                                       // aerol.h:822-877
                        if (!hdr) result = (bp >= RT_BLOCK) ? RT_BAD : RT_TEST_FAILED;
                        else {
                            nsus = 1 + (bp - 64 * 5) / (64 * 3);
                            const bool mine = (lane < nsus) ? crc16_bits_ok(obits + 8 * 6 + 8 * 12 * lane, 8 * 12) : true;
                            const bool all_ok = __all_sync(0xffffffffu, mine);
                            if (!all_ok) result = (bp >= RT_BLOCK) ? RT_BAD : RT_TEST_FAILED;
                            else { result = RT_OK_T; nbytes = sets / 8 - 1; }             // packintobytes(); chop(1)
                        }
                    } else {                                                              // aerol.h:696-770
                        if (!hdr) result = RT_BAD;
                        else if (nblk == 11) {
                            const uint8_t *isu = obits + 8 * 6 + 8 * 12;
                            int bin = 2 + isu[0] + isu[1] * 2 + isu[2] * 4 + isu[3] * 8 + isu[4] * 16 + isu[5] * 32;
                            if (bin >= 16) bin = bin / 2 + 1;
                            sl.targetSUSize = bin; sl.targetBlocks = (bin + 1) * 3 + 2;
                        } else if (nblk == sl.targetBlocks) { result = RT_OK_T; nsus = sl.targetSUSize; nbytes = sets / 8 - 1; }
                    }
                }
                if (result == RT_OK_R || result == RT_OK_T) {
                    if (out_count < RT_OUT) {
                        uint8_t *o = rp.out + ((size_t)ch * RT_OUT + out_count) * RT_OUT_BYTES;
                        for (int b = lane; b < nbytes && b < RT_OUT_BYTES - 16; b += 32) {    // LSB-first packing (aerol.h:602-628)
                            unsigned v = 0;
                            for (int t = 0; t < 8; t++) v |= (unsigned)obits[b * 8 + t] << t;
                            o[16 + b] = (uint8_t)v;
                        }
                        if (lane == 0) {
                            int *hdr32 = reinterpret_cast<int *>(o);
                            hdr32[0] = (result == RT_OK_R) ? 1 : 2; hdr32[1] = nsus; hdr32[2] = nbytes;
                            hdr32[3] = (int)(sl.start_bit & 0x7fffffff);
                        }
                        out_count++;
                    } else sp->overflow = 1;
                    sl.done = 1;
                    lastpacketstate = result;
                } else if (result == RT_TEST_FAILED || result == RT_BAD) lastpacketstate = result;
            }
            sl.next_trial += 64 * 3;
        }
        if (sl.next_trial > RT_BLOCK) sl.done = 1;
        if (sl.closed) {
            // no more bits will arrive: the packet is finished; resetblockptr() of the next packet reports a failed test
            if (lastpacketstate == RT_TEST_FAILED) n_bad++;
            lastpacketstate = RT_NOTHING;
        }
        if (lane == 0) slots[sidx] = sl;
    }
    __syncwarp();
    if (lane == 0) {
        // retire closed slots
        int h = head, no = n_open;
        while (no > 1 && slots[h].closed) { h++; if (h >= RT_SLOTS) h = 0; no--; }
        sp->slot_head = h; sp->n_open = no;
        sp->rc = rc; sp->lastpacketstate = lastpacketstate; sp->n_bad = n_bad; sp->out_count = out_count; sp->n_trials = trials;
    }
    (void)cur;
}

__global__ void rt_init_kernel(RtParams rp)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= rp.n_channels) return;
    RtState s;
    memset(&s, 0, sizeof s);
    s.cntr = CNTR_IDLE;                                        // AeroL ctor (aerol.cpp:907,927)
    s.lastpacketstate = RT_NOTHING;
    s.n_open = 1;                                              // the block the RT object starts with
    rp.state[ch] = s;
    // update() tests ((blockptr-320)%192)==0 with C's truncating %, which also holds at blockptr = 128 (aerol.h:794): the
    // OQPSK trial sequence is 128, 320, 512, ...; updateMSK() additionally requires blockptr/64 in {5, target, 11, 50}
    RtSlot ns; ns.fill = 0; ns.next_trial = rp.oqpsk ? 64 * 2 : 64 * 5; ns.done = 0; ns.closed = 0; ns.targetSUSize = 0; ns.targetBlocks = 0; ns.start_bit = 0;
    rp.slots[(size_t)ch * RT_SLOTS] = ns;
}

int rt_process(const RtParams &rp, const int16_t *d_soft, const int *d_soft_count, size_t soft_stride, cudaStream_t st, long long *launches, int vmode)
{
    rt_frame_kernel<<<(rp.n_channels + 63) / 64, 64, 0, st>>>(rp, d_soft, d_soft_count, soft_stride, vmode);
    JB_CUDA(cudaGetLastError());
    const int sb = (RT_BLOCK + 15) & ~15, ob = ((RT_BLOCK / 2) + 15) & ~15;
    const int per_warp = sb + 2 * V_CAP * (int)sizeof(unsigned) + ob;
    const int warps = 4;
    JB_CUDA(cudaFuncSetAttribute(rt_trial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, per_warp * warps));
    rt_trial_kernel<<<(rp.n_channels + warps - 1) / warps, warps * 32, per_warp * warps, st>>>(rp, per_warp, sb);
    JB_CUDA(cudaGetLastError());
    *launches += 2;
    return 0;
}

} // namespace jb
