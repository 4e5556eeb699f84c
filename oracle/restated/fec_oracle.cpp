// TEST INFRASTRUCTURE ONLY (oracle): CPU restatement, never linked into the product.
#include "fec_oracle.h"
#include <cstring>
#include <cmath>

// JAERO/aerol.cpp:531-535: interleaverowdepermute[i]=(i*27)%64 ; :613-621 out[k++]=block[depermute[i]*cols+j]
void oracle_deinterleave(const int *block, int cols, uint8_t *out)
{
    int k = 0;
    for (int j = 0; j < cols; j++)
        for (int i = 0; i < 64; i++)
            out[k++] = (uint8_t)block[((i * 27) % 64) * cols + j];
}

ContinuousViterbiOracle::ContinuousViterbiOracle(int pad) : paddinglength(pad)
{
    correct_convolutional_polynomial_t poly[2] = {109, 79};    // jconvolutionalcodec.cpp:13-14
    conv = correct_convolutional_create(2, 7, poly);
}
ContinuousViterbiOracle::~ContinuousViterbiOracle() { correct_convolutional_destroy(conv); }

std::vector<int> ContinuousViterbiOracle::decode(const uint8_t *soft, int n)
{
    const int k = 62;                                           // jconvolutionalcodec.cpp:153
    std::vector<uint8_t> buf(overlap);                          // :155 overlap ‖ block
    buf.insert(buf.end(), soft, soft + n);
    buf.insert(buf.end(), paddinglength, (uint8_t)128);         // :158-160 erasure padding
    std::vector<uint8_t> decoded(buf.size() / 2 + 1, 0);        // :167
    correct_convolutional_decode_soft(conv, buf.data(), buf.size(), decoded.data());   // :169
    int dbits = (int)buf.size() / 2;                            // :172
    std::vector<int> bits(dbits, 0);
    for (int i = 0; i < dbits; i++) bits[i] = (decoded[i >> 3] >> (7 - (i & 7))) & 1;  // :177-190 MSB first
    std::vector<int> out;                                       // :194 mid(paddinglength+1, n/2)
    int pos = paddinglength + 1;
    for (int i = 0; i < n / 2 && pos + i < dbits; i++) out.push_back(bits[pos + i]);
    int kk = k < n ? k : n;                                     // :197-198 right(k) of the *new* block, resized to k
    overlap.assign(soft + n - kk, soft + n);
    overlap.resize(k, 0);
    return out;
}

uint16_t oracle_crc16(const uint8_t *bytes, int n)
{
    uint16_t crc = 0xFFFF;
    for (int i = 0; i < n; i++) {
        int b = (int8_t)bytes[i];                               // `message_byte=bytes[i]` with char bytes (sign irrelevant for 8 shifts)
        for (int k = 0; k < 8; k++) {
            int mb = b & 1; b >>= 1;
            int cb = crc & 1; crc >>= 1;
            if (cb ^ mb) crc ^= 0x8408;
        }
    }
    return (uint16_t)~crc;
}

PChannelOracle::PChannelOracle(int fb) : codec(24)
{
    ifb = fb;
    switch (ifb) {                                              // aerol.cpp:1013-1052
    case 600:  cols = 6;  NumberOfBits = 1152; BitsInHeader = 16; TotalNumberOfBits = 16 + 1152 + 32; useingOQPSK = false; break;
    case 10500: cols = 78; NumberOfBits = 4992; BitsInHeader = 16 + 178; TotalNumberOfBits = 16 + 178 + 4992 + 64; useingOQPSK = true; break;
    default:   cols = 9;  NumberOfBits = 1152; BitsInHeader = 16; TotalNumberOfBits = 16 + 1152 + 32; useingOQPSK = false; break;
    }
    block.assign(cols * 64, 0);
    int dl2len = (ifb == 10500) ? 4992 - 6 : 576 - 6;           // aerol.cpp:1018,1026,1047
    dl2.assign(dl2len + 1, 0); dl2_ptr = 0;
    // scrambler (aerol.h:397-419)
    int st[15] = {1, 1, 0, 1, 0, 0, 1, 0, 1, 0, 1, 1, 0, 0, 1};
    scr.resize(5000);
    for (int a = 0; a < 5000; a++) {
        int v = st[0] ^ st[14];
        scr[a] = v;
        for (int i = 14; i > 0; i--) st[i] = st[i - 1];
        st[0] = v;
    }
    scr_pos = 0;
    preamble.clear();                                           // 0xE15AE893 MSB first (aerol.cpp:730-743,947)
    for (int i = 31; i >= 0; i--) preamble.push_back((3780831379ULL >> i) & 1);
    buf_plain.assign(32, 0); buf_imag.assign(32, 0); buf_real.assign(32, 0);
    inv_imag = inv_real = false;
    realimag = 0; gotsync_last = 0;
    cntr = 1000000000; blockcnt = -1;
    frameinfo = lastframeinfo = 0; formatid = supfrmaker = framecounter1 = framecounter2 = 0;
    datacdcountdown = 0; datacd = false;
    nframes = 0; bits_seen = 0; n_syncs = 0;
}

// PreambleDetectorPhaseInvariant::Update with tollerence 0 (aerol.cpp:781-804, non-burst :1003-1005)
static int uw_update_invariant(std::vector<int> &buf, const std::vector<int> &pre, int val, bool &inverted)
{
    int n = (int)buf.size(), xorsum = 0;
    for (int i = 0; i < n - 1; i++) { buf[i] = buf[i + 1]; xorsum += buf[i] ^ pre[i]; }
    xorsum += val ^ pre[n - 1];
    buf[n - 1] = val;
    if (xorsum >= n) { inverted = true; return 1; }
    if (xorsum <= 0) { inverted = false; return 1; }
    return 0;
}
// PreambleDetector::Update (aerol.cpp:744-750): exact match, buffer cleared on hit
static int uw_update_exact(std::vector<int> &buf, const std::vector<int> &pre, int val)
{
    int n = (int)buf.size();
    for (int i = 0; i < n - 1; i++) buf[i] = buf[i + 1];
    buf[n - 1] = val;
    if (buf == pre) { std::fill(buf.begin(), buf.end(), 0); return 1; }
    return 0;
}

void PChannelOracle::updateDCD()
{
    if (datacdcountdown > 0) datacdcountdown -= 3;
    else if (datacdcountdown < 0) datacdcountdown = 0;
    if (datacd && !datacdcountdown) { datacd = false; dcd_events.push_back((bits_seen << 1) | 0); }
}
void PChannelOracle::lostSignal()
{
    cntr = 1000000000; datacdcountdown = 0; datacd = false; dcd_events.push_back((bits_seen << 1) | 0);
}

void PChannelOracle::process(const short *bits, int n)
{
    for (int i = 0; i < n; i++) {
        bits_seen++;
        int bit = (((uint8_t)bits[i]) >= 128) ? 1 : 0;          // aerol.cpp:1136-1139
        int soft_bit = (uint16_t)bits[i];
        if (bits[i] < 0) continue;                              // burst marker (never in continuous modes)
        int gotsync;
        if (useingOQPSK) {                                      // aerol.cpp:1156-1233
            realimag++; realimag %= 2;
            std::vector<int> &buf = realimag ? buf_imag : buf_real;
            bool &inv = realimag ? inv_imag : inv_real;
            if (cntr > NumberOfBits - 68 || cntr <= 0 || !datacd) {
                gotsync = uw_update_invariant(buf, preamble, bit, inv);
                if (!gotsync_last) { gotsync_last = gotsync; gotsync = 0; } else gotsync_last = 0;
            } else { gotsync = 0; gotsync_last = 0; }
            if (inv) { bit = 1 - bit; if (soft_bit != 128) soft_bit = 255 - soft_bit; }
        } else gotsync = uw_update_exact(buf_plain, preamble, bit);   // aerol.cpp:1269-1272

        if (cntr < 1000000000) cntr++;
        if (cntr < 16) {                                        // :1275-1300 header
            if (cntr == 0) { frameinfo = (uint16_t)bit; infofield.clear(); }
            else { frameinfo = (uint16_t)((frameinfo << 1) | bit); }
        }
        if (cntr == 15) {                                       // :1301-1319 (delayed by one frame)
            uint16_t t = frameinfo; frameinfo = lastframeinfo; lastframeinfo = t;
            formatid = (frameinfo >> 12) & 15; supfrmaker = (frameinfo >> 8) & 15;
            framecounter1 = (frameinfo >> 4) & 15; framecounter2 = frameinfo & 15;
        }
        if (cntr >= 16) {                                       // :1540-1610
            if (cntr == 16) blockcnt = -1;
            int idx = (int)((cntr - BitsInHeader) % (long)block.size());
            if (idx < 0) idx = 0;
            block[idx] = soft_bit;
            if (idx == (int)block.size() - 1) {
                blockcnt++;
                std::vector<uint8_t> dl(block.size());
                oracle_deinterleave(block.data(), cols, dl.data());
                std::vector<int> dec = codec.decode(dl.data(), (int)dl.size());
                for (size_t h = 0; h < dec.size(); h++) {       // dl2.update (aerol.h:465-473)
                    dl2[dl2_ptr] = dec[h]; dl2_ptr++; dl2_ptr %= (int)dl2.size(); dec[h] = dl2[dl2_ptr];
                }
                for (size_t h = 0; h < dec.size(); h++) { dec[h] ^= scr[scr_pos]; scr_pos++; }   // scrambler.update
                int charptr = 0; uint8_t ch = 0;                // :1568-1580 LSB-first packing
                for (size_t h = 0; h < dec.size(); h++) {
                    ch |= (uint8_t)(dec[h] * 128);
                    charptr++; charptr %= 8;
                    if (charptr == 0) { infofield.push_back(ch); ch = 0; } else ch >>= 1;
                }
                if ((cntr - BitsInHeader) == (NumberOfBits - 1)) {   // :1582 frame done
                    for (int k = 0; k < (int)infofield.size() / 12; k++) {
                        uint16_t crc_calc = oracle_crc16(&infofield[k * 12], 10);
                        uint16_t crc_rec = (uint16_t)((infofield[k * 12 + 11] << 8) | infofield[k * 12 + 10]);
                        if ((!crc_rec) && (crc_calc != crc_rec)) {
                            int tsum = 0; for (int ii = 0; ii < 10; ii++) tsum += infofield[k * 12 + ii];
                            if (tsum == 0) crc_calc = 0;
                        }
                        if (crc_calc == crc_rec) { if (datacdcountdown < 12) datacdcountdown += 2; }
                        else { if (datacdcountdown > 0) datacdcountdown -= 3; }
                        if (!datacd && datacdcountdown > 2) { datacd = true; dcd_events.push_back((bits_seen << 1) | 1); }
                        SignalUnit su; memcpy(su.bytes, &infofield[k * 12], 12);
                        su.crc_ok = (crc_calc == crc_rec); su.frame = nframes;
                        sus.push_back(su);
                    }
                    nframes++;
                }
            }
        }
        if (gotsync) {                                          // :1990-2011
            cntr = -1; datacd = true; datacdcountdown = 12; dcd_events.push_back((bits_seen << 1) | 1);
            scr_pos = 0; n_syncs++;
        }
        if (cntr + 1 == TotalNumberOfBits) { scr_pos = 0; cntr = -1; }   // :2013-2016
    }
}


// ====================================================================================== R/T burst channel
namespace {
enum { RT_OK_R = 3, RT_OK_T = 5, RT_BAD = 0, RT_TEST_FAILED = 32, RT_NOTHING = 8, RT_FULL = 16 };
const uint32_t RT_UW = 0xE15AE893u;                            // aerol.cpp:947,959-963
// AeroLcrc16::calcusingbitsandcheck (aerol.h:287-313)
bool crc_bits_check(const int *bits, int numberofbits)
{
    uint16_t crc_rec = 0;
    for (int i = numberofbits - 1; i >= numberofbits - 16; i--) { crc_rec <<= 1; crc_rec |= (uint16_t)bits[i]; }
    numberofbits -= 16;
    uint16_t crc = 0xFFFF;
    for (int i = 0; i < numberofbits; i++) {
        const int crc_bit = crc & 1;
        crc >>= 1;
        if (crc_bit ^ bits[i]) crc = crc ^ 0x8408;
    }
    crc = (uint16_t)~crc;
    return crc_rec == crc;
}
// PreambleDetectorPhaseInvariant::Update (aerol.cpp:781-804) on a 32-bit shift register
int uw_invariant_tol(uint32_t &sr, int bit, bool &inverted, int tol)
{
    sr = (sr << 1) | (uint32_t)bit;
    const int xorsum = __builtin_popcount(sr ^ RT_UW);
    if (xorsum >= (32 - tol)) { inverted = true; return 1; }
    if (xorsum <= tol) { inverted = false; return 1; }
    return 0;
}
}

RTChannelOracle::RTChannelOracle(int fb)
{
    ifb = fb;
    useingOQPSK = (fb == 10500 || fb == 8400);
    NumberOfBits = (fb == 10500) ? 4992 : (fb == 8400 ? 4096 : 1152);                 // aerol.cpp:1012-1050
    TotalNumberOfBits = useingOQPSK ? ifb : ifb * 3;                                    // :1062-1070
    sr_imag = sr_real = sr_msk = 0; inv_imag = inv_real = inv_msk = false;
    realimag = 0; gotsync_last = 0;
    cntr = 1000000000; muw = 0; datacd = false; datacdcountdown = 0;
    block.assign(64 * 95, 0); blockptr = 0; lastpacketstate = RT_NOTHING; targetSUSize = targetBlocks = numberofsus = 0;
    correct_convolutional_polynomial_t poly[2] = {109, 79};
    conv = correct_convolutional_create(2, 7, poly);
    {   // AeroLScrambler (aerol.h:397-437)
        int st[15] = {1, 1, 0, 1, 0, 0, 1, 0, 1, 0, 1, 1, 0, 0, 1};
        scr.resize(5000);
        for (int a = 0; a < 5000; a++) {
            const int v = st[0] ^ st[14];
            scr[a] = v;
            for (int i = 14; i > 0; i--) st[i] = st[i - 1];
            st[0] = v;
        }
    }
    n_bad = n_trials = bits_seen = 0;
}
RTChannelOracle::~RTChannelOracle() { correct_convolutional_destroy(conv); }

int RTChannelOracle::resetblockptr()                           // aerol.h:590-601
{
    blockptr = 0;
    if (lastpacketstate == RT_TEST_FAILED) { lastpacketstate = RT_NOTHING; return RT_BAD; }
    lastpacketstate = RT_NOTHING;
    return RT_NOTHING;
}

static void rt_decode(RTChannelOracle &o, const std::vector<uint8_t> &del, int nsoft)
{
    // JConvolutionalCodec::Decode_soft (jconvolutionalcodec.cpp:98-125) + scrambler.reset/update
    std::vector<uint8_t> dec(nsoft / 2 / 8 + 8, 0);
    correct_convolutional_decode_soft(o.conv, del.data(), (size_t)nsoft, dec.data());
    const int dbits = nsoft / 2;
    o.deconvol.assign(dbits, 0);
    for (int i = 0; i < dbits; i++) o.deconvol[i] = (dec[i >> 3] >> (7 - (i & 7))) & 1;
    for (int i = 0; i < dbits; i++) o.deconvol[i] ^= o.scr[i];
    o.n_trials++;
}
static void rt_pack(RTChannelOracle &o)                        // packintobytes (aerol.h:602-628)
{
    o.infofield.clear();
    int charptr = 0; uint8_t ch = 0;
    for (size_t h = 0; h < o.deconvol.size(); h++) {
        ch |= (uint8_t)(o.deconvol[h] * 128);
        charptr++; charptr %= 8;
        if (charptr == 0) { o.infofield.push_back(ch); ch = 0; } else ch >>= 1;
    }
}

int RTChannelOracle::rt_update(int bit)                        // aerol.h:786-877
{
    if (blockptr >= (int)block.size()) return RT_FULL;
    block[blockptr] = bit; blockptr++;
    if (((blockptr - (64 * 5)) % (64 * 3)) == 0) {
        const int cols = blockptr / 64;
        std::vector<uint8_t> del((size_t)blockptr);
        { int k = 0; for (int j = 0; j < cols; j++) for (int i = 0; i < 64; i++) del[k++] = (uint8_t)block[((i * 27) % 64) * cols + j]; }   // deinterleave_ba
        rt_decode(*this, del, blockptr);
        if (blockptr == (64 * 5)) {
            if (!crc_bits_check(deconvol.data(), 8 * 19)) { lastpacketstate = RT_TEST_FAILED; return RT_TEST_FAILED; }
            rt_pack(*this);
            blockptr = (int)block.size();
            lastpacketstate = RT_OK_R;
            return RT_OK_R;
        }
        if (!crc_bits_check(deconvol.data(), 8 * 6)) {
            if (blockptr >= (int)block.size()) { lastpacketstate = RT_BAD; return RT_BAD; }
            lastpacketstate = RT_TEST_FAILED; return RT_TEST_FAILED;
        }
        numberofsus = 1 + (blockptr - (64 * 5)) / (64 * 3);
        for (int i = 0; i < numberofsus; i++) {
            if (!crc_bits_check(deconvol.data() + (8 * 6) + (8 * 12) * i, 8 * 12)) {
                if (blockptr >= (int)block.size()) { lastpacketstate = RT_BAD; return RT_BAD; }
                lastpacketstate = RT_TEST_FAILED; return RT_TEST_FAILED;
            }
        }
        rt_pack(*this);
        if (!infofield.empty()) infofield.pop_back();          // chop(1)
        blockptr = (int)block.size();
        lastpacketstate = RT_OK_T;
        return RT_OK_T;
    }
    return RT_NOTHING;
}

int RTChannelOracle::rt_updateMSK(int bit)                     // aerol.h:631-783
{
    if (blockptr >= (int)block.size()) return RT_FULL;
    block[blockptr] = bit; blockptr++;
    int ok = 0;
    bool cont = false;
    if ((((blockptr - (64 * 5)) % (64 * 3)) == 0) && (blockptr / 64 == 5 || blockptr / 64 == targetBlocks || blockptr / 64 == 11 || blockptr / 64 == 50)) cont = true;
    if (cont) {
        const int blocks = blockptr / 64;
        std::vector<uint8_t> del((size_t)blockptr);
        {   // deinterleaveMSK_ba (aerol.cpp:673-714): 5 columns first, then groups of 3
            int k = 0;
            for (int j = 0; j < 5; j++) for (int i = 0; i < 64; i++) del[k++] = (uint8_t)block[((i * 27) % 64) * 5 + j];
            int procblocks = 5;
            while (k < blocks * 64) {
                for (int j = 0; j < 3; j++) for (int i = 0; i < 64; i++) del[k++] = (uint8_t)block[(64 * procblocks) + (((i * 27) % 64) * 3 + j)];
                procblocks += 3;
            }
        }
        rt_decode(*this, del, blockptr);
        if (blockptr == (64 * 5)) {
            targetSUSize = 0; targetBlocks = 0;
            if (crc_bits_check(deconvol.data(), 8 * 19)) {
                rt_pack(*this);
                blockptr = (int)block.size();
                lastpacketstate = RT_OK_R;
                return RT_OK_R;
            }
            return RT_NOTHING;
        }
        if (!crc_bits_check(deconvol.data(), 8 * 6)) { lastpacketstate = RT_BAD; return RT_BAD; }
        if (blockptr / 64 == 11) {
            const int *isu = deconvol.data() + (8 * 6) + (8 * 12) * 1;
            int bin = 2;
            bin += ((isu[0] * 1) + (isu[1] * 2) + (isu[2] * 4) + (isu[3] * 8) + (isu[4] * 16) + (isu[5] * 32));
            targetSUSize = bin;
            if (targetSUSize >= 16) targetSUSize = (int)floor(targetSUSize / 2) + 1;
            targetBlocks = ((targetSUSize + 1) * 3) + 2;
            return RT_NOTHING;
        }
        if (blockptr / 64 == targetBlocks) {
            for (int i = 0; i < targetSUSize - 3; i++) if (crc_bits_check(deconvol.data() + (8 * 6) + (8 * 12) * i, 8 * 12)) ok++;
            if (ok <= targetSUSize) {
                rt_pack(*this);
                if (!infofield.empty()) infofield.pop_back();
                numberofsus = targetSUSize;
                blockptr = (int)block.size();
                lastpacketstate = RT_OK_T;
                return RT_OK_T;
            }
        }
        return RT_NOTHING;
    }
    return RT_NOTHING;
}

void RTChannelOracle::process(const short *bits, int n, bool vector_semantics)
{
    for (int i = 0; i < n; i++) {
        bits_seen++;
        int bit = (((uint8_t)bits[i]) >= 128) ? 1 : 0;          // aerol.cpp:1136-1139
        int soft_bit = (uint16_t)bits[i];
        if (bits[i] < 0) { muw = 0; continue; }                 // :1146-1151 start-of-burst marker
        if (muw < 100000) muw++;
        int gotsync = 0;
        if (useingOQPSK) {                                      // :1156-1233
            realimag++; realimag %= 2;
            uint32_t &sr = realimag ? sr_imag : sr_real;
            bool &inv = realimag ? inv_imag : inv_real;
            if (cntr > NumberOfBits - 68 || cntr <= 0 || !datacd) {
                gotsync = uw_invariant_tol(sr, bit, inv, 4);
                if (!gotsync_last) { gotsync_last = gotsync; gotsync = 0; } else gotsync_last = 0;
            } else { gotsync = 0; gotsync_last = 0; }
            if (gotsync) { if (ifb == 10500 && (labs(muw - 80) > 150)) gotsync = 0; }   // :1193-1200
            if (inv) { bit = 1 - bit; if (soft_bit != 128) soft_bit = 255 - soft_bit; }
        } else {                                                // :1236-1266
            const bool inverted = inv_msk;
            gotsync = uw_invariant_tol(sr_msk, bit, inv_msk, 4);
            if (muw > 250 && gotsync) { if (inverted != inv_msk) inv_msk = inverted; gotsync = 0; }
            if (inv_msk) { bit = 1 - bit; if (soft_bit != 128) soft_bit = 255 - soft_bit; }
        }
        if (cntr < 1000000000) cntr++;
        if (cntr < 16) {                                        // :1275-1300: no header on R/T channels
            if (cntr == 0) { cntr = 16; if (resetblockptr() == RT_BAD) n_bad++; }
        }
        if (cntr >= 16) {                                       // :1327-1345
            const int result = useingOQPSK ? rt_update(soft_bit) : rt_updateMSK(soft_bit);
            if (result == RT_OK_R) { RTPacket pk; pk.type = 1; pk.nsus = 0; pk.bit_index = bits_seen; pk.bytes.assign(infofield.begin(), infofield.begin() + 19); packets.push_back(pk); }
            else if (result == RT_OK_T) { RTPacket pk; pk.type = 2; pk.nsus = numberofsus; pk.bit_index = bits_seen; pk.bytes = infofield; packets.push_back(pk); }
        }
        if (gotsync) { cntr = -1; datacd = true; datacdcountdown = 12; }   // :1990-2011
        if (cntr + 1 == TotalNumberOfBits) {                    // :2013-2029
            cntr = 1000000000; datacd = false; datacdcountdown = 0;
            if (vector_semantics) return;
        }
    }
}

void RTChannelOracle::updateDCD()                              // aerol.cpp:1109-1122
{
    if (datacdcountdown > 0) datacdcountdown -= 3;
    else { if (datacdcountdown < 0) datacdcountdown = 0; }
    if (datacd && !datacdcountdown) datacd = false;
}


// ====================================================================================== C channel (8400 bps)
namespace {
const uint64_t C_PRE1 = 216866263330005ULL, C_PRE2 = 3012071630031408ULL;   // aerol.cpp:953-954 (Q word, I word), 52 bits
const uint64_t C_MASK = (1ULL << 52) - 1;
// OQPSKPreambleDetectorAndAmbiguityCorrection::Update (aerol.cpp:848-896), tollerence 6: the second buffer is only
// shifted when the first one does not match
int c_uw_update(uint64_t &b1, uint64_t &b2, int val, bool &inverted)
{
    b1 = ((b1 << 1) | (uint64_t)val) & C_MASK;
    int xorsum = __builtin_popcountll(b1 ^ C_PRE1);
    if (xorsum >= 52 - 6) { inverted = true; return 1; }
    if (xorsum <= 6) { inverted = false; return 1; }
    b2 = ((b2 << 1) | (uint64_t)val) & C_MASK;
    xorsum = __builtin_popcountll(b2 ^ C_PRE2);
    if (xorsum >= 52 - 6) { inverted = true; return 1; }
    if (xorsum <= 6) { inverted = false; return 1; }
    return 0;
}
}

CChannelOracle::CChannelOracle() : codec(24)
{
    b1_real = b2_real = b1_imag = b2_imag = 0; inv_real = inv_imag = false;
    realimag = 0; gotsync_last = 0; cntr = 1000000000; index = 0;                  // AeroL ctor: index = 0 (aerol.cpp:957)
    block.assign(4 * 64, 0);
    dl2.assign(2714 - 6 + 1, 0); dl2_ptr = 0;                                       // dl2.setLength(2714-6) (aerol.cpp:1037)
    {
        int st[15] = {1, 1, 0, 1, 0, 0, 1, 0, 1, 0, 1, 1, 0, 0, 1};
        scr.resize(5000);
        for (int a = 0; a < 5000; a++) { const int v = st[0] ^ st[14]; scr[a] = v; for (int i = 14; i > 0; i--) st[i] = st[i - 1]; st[0] = v; }
    }
    datacdcountdown = 0; datacd = false; bits_seen = 0; nframes = 0;
}

void CChannelOracle::process(const short *bits, int n)
{
    const int NumberOfBits = 4096;
    for (int i = 0; i < n; i++) {
        bits_seen++;
        int bit = (((uint8_t)bits[i]) >= 128) ? 1 : 0;
        int soft_bit = (uint16_t)bits[i];
        int gotsync = 0;
        realimag++; realimag %= 2;
        const bool search = (cntr > NumberOfBits - 112 || cntr <= 0);
        if (realimag) {
            if (search) { gotsync = c_uw_update(b1_real, b2_real, bit, inv_real); if (!gotsync_last) { gotsync_last = gotsync; gotsync = 0; } else gotsync_last = 0; }
            else { gotsync = 0; gotsync_last = 0; }
            if (inv_real) { bit = 1 - bit; if (soft_bit != 128) soft_bit = 255 - soft_bit; }
        } else {
            if (search) { gotsync = c_uw_update(b1_imag, b2_imag, bit, inv_imag); if (!gotsync_last) { gotsync_last = gotsync; gotsync = 0; } else gotsync_last = 0; }
            else { gotsync = 0; gotsync_last = 0; }
            if (inv_imag) { bit = 1 - bit; if (soft_bit != 128) soft_bit = 255 - soft_bit; }
        }
        if (gotsync) { cntr = -1; index = -1; deleavered.clear(); }            // :2286-2296 (scrambler.reset: position 0 per frame)
        else {
            if (cntr < 1000000000) cntr++;
            if (cntr <= NumberOfBits - 1) { index++; if (index >= 0 && index < 256) block[index] = soft_bit; }
            if (index == 255) {                                                // :2308-2319 deinterleave_ba(block, 4)
                for (int j = 0; j < 4; j++) for (int r = 0; r < 64; r++) deleavered.push_back((uint8_t)block[((r * 27) % 64) * 4 + j]);
                index = -1;
            }
            if (cntr == NumberOfBits - 1) {                                    // :2320-2498 frame complete
                std::vector<uint8_t> dep;                                      // depunture_soft_block(..., 4, true) (:2505-2518)
                { int ptr = 0; for (int k = 0; k + 1 < (int)deleavered.size(); k++) { ptr++; dep.push_back(deleavered[k]); if (ptr >= 3) dep.push_back(128); ptr %= 3; } }
                std::vector<int> dec = codec.decode(dep.data(), (int)dep.size());
                dec.resize(2714, 0);
                for (size_t h = 0; h < dec.size(); h++) { dl2[dl2_ptr] = dec[h]; dl2_ptr++; dl2_ptr %= (int)dl2.size(); dec[h] = dl2[dl2_ptr]; }
                for (size_t h = 0; h < dec.size(); h++) dec[h] ^= scr[h];
                CFrame fr; memset(&fr, 0, sizeof fr); fr.bit_index = bits_seen;
                std::vector<uint8_t> info; int charptr = 0; uint8_t ch = 0; int nsu = 0;
                for (int y = 0; y < 24; y++) {
                    const int offset = y * (1 + 96 + 12);
                    for (int h = offset + 97; h < offset + 109; h++) {
                        ch |= (uint8_t)(dec[h] * 128);
                        charptr++; charptr %= 8;
                        if (charptr == 0) { info.push_back(ch); ch = 0; } else ch >>= 1;
                    }
                    if (info.size() == 12) {
                        const uint16_t crc_calc = oracle_crc16(info.data(), 10);
                        const uint16_t crc_rec = (uint16_t)((info[11] << 8) | info[10]);
                        const bool ok = crc_calc == crc_rec;
                        if (ok) { if (datacdcountdown < 12) datacdcountdown += 2; }
                        else { if (datacdcountdown > 0) datacdcountdown -= 5; }
                        if (!datacd && datacdcountdown > 2) datacd = true;
                        if (nsu < 3) { memcpy(fr.su[nsu].bytes, info.data(), 12); fr.su[nsu].crc_ok = ok ? 1 : 0; fr.su[nsu].frame = nframes; nsu++; }
                        info.clear();
                    }
                }
                int bitsin = 0, vb = 0;
                for (int h = 1; h < 2714; h++) {                               // voice payload: 25 x 96 bits (:2457-2479)
                    ch |= (uint8_t)(dec[h] * 128);
                    charptr++; charptr %= 8;
                    if (charptr == 0) { if (vb < 300) fr.voice[vb++] = ch; ch = 0; } else ch >>= 1;
                    bitsin++;
                    if (bitsin == 96) { bitsin = 0; h += 13; }
                }
                frames.push_back(fr); nframes++;
                index = -1;
            }
        }
    }
}

void CChannelOracle::updateDCD()
{
    if (datacdcountdown > 0) datacdcountdown -= 3;
    else { if (datacdcountdown < 0) datacdcountdown = 0; }
    if (datacd && !datacdcountdown) datacd = false;
}
void CChannelOracle::lostSignal() { cntr = 1000000000; datacdcountdown = 0; datacd = false; }

// ====================================================================================== pinning hooks
// The pieces of this restatement one by one, for tests/test_fec_pinning.py, which holds them against the reference's own
// classes compiled verbatim (oracle/ref_fec_driver.cpp -> oracle/_ref/libjaero_ref_fec.so).
extern "C" {
// kind 0: PreambleDetector (exact, cleared on a hit); 1: PreambleDetectorPhaseInvariant, tollerence 0, on a bit vector;
// 2: OQPSKPreambleDetectorAndAmbiguityCorrection (two 52-bit words, tollerence 6); 3: phase-invariant on a shift register with `tol`
void jor_pin_detect(int kind, int tol, const int *bits, int n, int *out, int *inv)
{
    std::vector<int> pre; for (int i = 31; i >= 0; i--) pre.push_back((3780831379ULL >> i) & 1);
    std::vector<int> buf(32, 0); bool inverted = false; uint32_t sr = 0; uint64_t b1 = 0, b2 = 0;
    for (int i = 0; i < n; i++) {
        if (kind == 0) out[i] = uw_update_exact(buf, pre, bits[i]);
        else if (kind == 1) out[i] = uw_update_invariant(buf, pre, bits[i], inverted);
        else if (kind == 2) out[i] = c_uw_update(b1, b2, bits[i], inverted);
        else out[i] = uw_invariant_tol(sr, bits[i], inverted, tol);
        inv[i] = inverted ? 1 : 0;
    }
}
int jor_pin_crc_bits_check(const int *bits, int n) { return crc_bits_check(bits, n) ? 1 : 0; }
void jor_pin_scrambler(int *out, int n) { PChannelOracle p(600); for (int i = 0; i < n; i++) out[i] = p.scr[i]; }
// C-channel frame: 16 blocks of 4 x 64 soft values -> de-interleaved, de-punctured code-order stream (as CChannelOracle::process builds it)
int jor_pin_c_code_order(const int *frame4096, unsigned char *out)
{
    std::vector<uint8_t> deleavered;
    for (int b = 0; b < 16; b++) {
        const int *block = frame4096 + 256 * b;
        for (int j = 0; j < 4; j++) for (int r = 0; r < 64; r++) deleavered.push_back((uint8_t)block[((r * 27) % 64) * 4 + j]);
    }
    int ptr = 0, n = 0;
    for (int k = 0; k + 1 < (int)deleavered.size(); k++) { ptr++; out[n++] = deleavered[k]; if (ptr >= 3) out[n++] = 128; ptr %= 3; }
    return n;
}
void *jor_pin_rt_new(int fb) { return new RTChannelOracle(fb); }
void jor_pin_rt_free(void *h) { delete (RTChannelOracle *)h; }
int jor_pin_rt_reset(void *h) { return ((RTChannelOracle *)h)->resetblockptr(); }
int jor_pin_rt_update(void *h, int msk, int soft) { RTChannelOracle *r = (RTChannelOracle *)h; return msk ? r->rt_updateMSK(soft) : r->rt_update(soft); }
int jor_pin_rt_info(void *h, unsigned char *out, int cap, int *numberofsus)
{
    RTChannelOracle *r = (RTChannelOracle *)h;
    int n = (int)r->infofield.size() < cap ? (int)r->infofield.size() : cap;
    for (int i = 0; i < n; i++) out[i] = r->infofield[i];
    *numberofsus = r->numberofsus;
    return (int)r->infofield.size();
}
}
