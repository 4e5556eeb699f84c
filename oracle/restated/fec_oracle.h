// TEST INFRASTRUCTURE ONLY (oracle): CPU restatement, never linked into the product.
// De-interleaver + continuous K=7 r=1/2 soft Viterbi wrapper + P-channel framing of the reference.
#ifndef JAERO_FEC_ORACLE_H
#define JAERO_FEC_ORACLE_H
#include <cstdint>
#include <vector>
extern "C" {
#include "correct.h"
}

// AeroLInterleaver::deinterleave_ba  (JAERO/aerol.cpp:523-538 row permutation, :603-625 gather)
void oracle_deinterleave(const int *block, int cols, uint8_t *out);

// JConvolutionalCodec::Decode_Continuous  (JAERO/jconvolutionalcodec.cpp:151-201)
struct ContinuousViterbiOracle
{
    correct_convolutional *conv;
    int paddinglength;                 // AeroL passes 24 (JAERO/aerol.cpp:940)
    std::vector<uint8_t> overlap;      // last 62 soft values of the previous block
    ContinuousViterbiOracle(int paddinglength = 24);
    ~ContinuousViterbiOracle();
    // soft: n values 0..255 ; returns n/2 bits (0/1)
    std::vector<int> decode(const uint8_t *soft, int n);
};

struct SignalUnit { uint8_t bytes[12]; int crc_ok; long frame; };

// AeroL::Decode, continuous (non-burst) P-channel branch for 600 / 1200 / 10500 bps
// (JAERO/aerol.cpp:1124-1322 UW + header, :1540-1610 block/FEC/CRC, :1990-2039 sync), minus all text output.
struct PChannelOracle
{
    int ifb; bool useingOQPSK;
    int NumberOfBits, BitsInHeader, TotalNumberOfBits, cols;
    std::vector<int> block;
    ContinuousViterbiOracle codec;
    std::vector<int> dl2; int dl2_ptr;             // DelayLine (aerol.h:451-481)
    std::vector<int> scr; int scr_pos;             // AeroLScrambler (aerol.h:397-437)
    // preamble detectors
    std::vector<int> preamble, buf_plain, buf_imag, buf_real;
    bool inv_imag, inv_real;
    int realimag, gotsync_last;
    long cntr; int blockcnt;
    uint16_t frameinfo, lastframeinfo; int formatid, supfrmaker, framecounter1, framecounter2;
    std::vector<uint8_t> infofield;
    int datacdcountdown; bool datacd;
    long nframes;
    // outputs
    std::vector<SignalUnit> sus;
    std::vector<long> dcd_events;                  // (bit index<<1)|dcd at every DataCarrierDetect emit
    long bits_seen, n_syncs;                       // n_syncs: unique-word syncs so far
    explicit PChannelOracle(int fb);
    void process(const short *soft, int n);        // AeroL::processDemodulatedSoftBits -> Decode(bits,true)
    void updateDCD();                              // AeroL::updateDCD (aerol.cpp:1109-1122), 1 s tick
    void lostSignal();                             // AeroL::LostSignal (aerol.h:925-931)
};
uint16_t oracle_crc16(const uint8_t *bytes, int n);

// ---- AeroL::DecodeC, 8400 bps C-channel (JAERO/aerol.cpp:2187-2500; dual-UW detector :848-896; PuncturedCode :2505-2518)
struct CFrame { SignalUnit su[3]; uint8_t voice[300]; long bit_index; };
struct CChannelOracle
{
    uint64_t b1_real, b2_real, b1_imag, b2_imag; bool inv_real, inv_imag;     // OQPSKPreambleDetectorAndAmbiguityCorrection x2
    int realimag, gotsync_last; long cntr; int index;
    std::vector<int> block; std::vector<uint8_t> deleavered;
    ContinuousViterbiOracle codec;
    std::vector<int> dl2; int dl2_ptr;
    std::vector<int> scr;
    int datacdcountdown; bool datacd;
    std::vector<CFrame> frames; long bits_seen, nframes;
    CChannelOracle();
    void process(const short *soft, int n);
    void updateDCD();
    void lostSignal();                             // AeroL::LostSignal (aerol.h:925-931): the members DecodeC uses
};

// ---- burst (R/T channel) branch of AeroL::Decode (JAERO/aerol.cpp:1124-1350, :1985-2031) with
// RTChannelDeleaveFECScram (JAERO/aerol.h:554-895), minus all text output / ACARS parsing.
struct RTPacket { int type; int nsus; long bit_index; std::vector<uint8_t> bytes; };   // type 1 = R packet (19 bytes), 2 = T packet (6+12n)
struct RTChannelOracle
{
    int ifb; bool useingOQPSK; int NumberOfBits, TotalNumberOfBits;
    uint32_t sr_imag, sr_real, sr_msk; bool inv_imag, inv_real, inv_msk;   // PreambleDetectorPhaseInvariant x3, tollerence 4
    int realimag, gotsync_last;
    long cntr, muw; bool datacd; int datacdcountdown;
    // RTChannelDeleaveFECScram
    std::vector<int> block; int blockptr; int lastpacketstate; int targetSUSize, targetBlocks, numberofsus;
    correct_convolutional *conv;
    std::vector<int> scr;
    std::vector<int> deconvol;
    std::vector<uint8_t> infofield;
    // outputs
    std::vector<RTPacket> packets; long n_bad, n_trials, bits_seen;
    explicit RTChannelOracle(int fb);
    ~RTChannelOracle();
    // one call per processDemodulatedSoftBits emit when vector_semantics (the reference returns from Decode() in the middle
    // of a vector when the burst time-out fires, aerol.cpp:2018-2027); otherwise the stream is processed without drops
    void process(const short *soft, int n, bool vector_semantics);
    void updateDCD();
    int rt_update(int soft_bit);        // RTChannelDeleaveFECScram::update (OQPSK)
    int rt_updateMSK(int soft_bit);     // RTChannelDeleaveFECScram::updateMSK
    int resetblockptr();
};   // AeroLcrc16::calcusingbytes (aerol.h:334-362)
#endif
