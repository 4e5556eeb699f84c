"""Soft-bit streams for the P-, C- and R/T-channel frame layers, built to reach the edges of their detectors, fast paths and
queues. Pure numpy plus jaero_b200.synth (and, for the C-channel, the restated demodulator over the committed 8400 bps
recording); no device.

Every builder returns a list of family members. A member is a dict:
    soft    int16 soft bits, 0..255, with -1 only where a burst demodulator emits its start-of-burst marker
    cuts    lengths of the successive process calls (they sum to len(soft))
    lost    indices of the calls after which LostSignal is raised on this channel (P- and C-channel)
    tag     what the member exercises
plus family-specific facts the CPU tests check on the oracle. The same member is fed to the device and to one oracle object
per channel under the same schedule; a global tick (AeroL::updateDCD) after every `tick_every`-th call is the runner's choice.
"""
import functools

import numpy as np

from jaero_b200 import synth

HI, LO = 230, 25
UW_BITS = np.array([(synth.UW >> (31 - i)) & 1 for i in range(32)], dtype=np.uint8)


def to_soft(bits, hi=HI, lo=LO):
    return np.where(np.asarray(bits) == 1, hi, lo).astype(np.int16)


def invert(soft):
    """the soft values as the opposite phase gives them: v -> 255 - v, erasures (128) and markers (-1) kept"""
    s = np.asarray(soft, dtype=np.int16).copy()
    m = (s >= 0) & (s != 128)
    s[m] = 255 - s[m]
    return s


def cut_sequence(n, rng, sizes):
    """call lengths summing to n, drawn from `sizes` (0 allowed: a call with nothing for this channel)"""
    cuts, a = [], 0
    while a < n:
        k = min(int(rng.choice(sizes)), n - a)
        cuts.append(k); a += k
    return cuts


def member(soft, cuts=None, lost=(), tag="", **facts):
    soft = np.asarray(soft, dtype=np.int16)
    if cuts is None:
        cuts = [len(soft)]
    assert sum(cuts) == len(soft)
    return dict(soft=soft, cuts=list(cuts), lost=set(lost), tag=tag, **facts)


# ---------------------------------------------------------------------------------------------------------------- P-channel
def p_geometry(fb):
    fp = synth.frame_params(fb)
    uw_len = 64 if fp["uw_interleaved"] else 32
    number_of_bits = 4992 if int(fb) == 10500 else 1152
    bits_in_header = 16 + fp["header_extra"]
    return dict(frame=fp["frame_bits"], uw_len=uw_len, number_of_bits=number_of_bits, bits_in_header=bits_in_header,
                oqpsk=fp["uw_interleaved"], sus_per_frame=fp["sus"])


def p_frames(fb, n_frames, seed):
    bits, sus = synth.pchannel_bits(fb, n_frames, seed=seed, return_sus=True)
    return bits, sus.reshape(-1, 12)


def noise_bits(rng, n):
    """random bits that carry no exact unique word on either arm or in the serial stream"""
    while True:
        b = rng.integers(0, 2, size=n).astype(np.uint8)
        if not _has_uw(b):
            return b


def _has_uw(b):
    b = np.asarray(b, dtype=np.int64)
    if len(b) < 32:
        return False
    w = np.lib.stride_tricks.sliding_window_view(b, 32) @ (1 << np.arange(31, -1, -1, dtype=np.int64))
    if np.any((w == synth.UW) | (w == (~synth.UW & 0xFFFFFFFF))):
        return True
    for arm in (0, 1):
        a = b[arm::2]
        if len(a) >= 32:
            w = np.lib.stride_tricks.sliding_window_view(a, 32) @ (1 << np.arange(31, -1, -1, dtype=np.int64))
            if np.any((w == synth.UW) | (w == (~synth.UW & 0xFFFFFFFF))):
                return True
    return False


def p_offset_family(fb, seed=1):
    """A unique word whose last bit falls at every offset 0..31 from the start of a call, on both arms (10.5 kbps), on a
    channel that has never synced (idle counter, noise before the first frame) and on one whose counter runs (the UW of the
    second of back-to-back frames). The call that holds the UW's last bit starts `offset` bits before it."""
    g = p_geometry(fb)
    rng = np.random.default_rng(seed)
    out = []
    arms = (0, 1) if g["oqpsk"] else (0,)
    n_frames = 5 if g["oqpsk"] else 4                            # the delay line holds two 10.5 kbps frames, one at 600 / 1200
    for state in ("idle", "running"):
        for arm in arms:
            for off in range(32):
                frames, sus = p_frames(fb, n_frames, seed=seed * 1000 + off * 2 + arm)
                pre = noise_bits(rng, 80 + arm)
                bits = np.concatenate([pre, frames])
                uw_last = len(pre) + g["uw_len"] - 1 + (g["frame"] if state == "running" else 0)
                a = uw_last - off
                rest = len(bits) - a
                cuts = [a] + cut_sequence(rest, rng, [off + 1, 97, 1000, 4093])
                out.append(member(to_soft(bits), cuts, tag="p-offset-%s-arm%d-%d" % (state, arm, off), sus=sus, n_frames=n_frames,
                                  offset=off, arm=arm, state=state))
    return out


def _set_uw(bits, start, g, flip=()):
    """write the unique word (both arms at 10.5 kbps) at bits[start:], with the listed UW bit indices flipped (on both arms)"""
    uw = UW_BITS.copy()
    for k in flip:
        uw[k] ^= 1
    w = np.repeat(uw, 2) if g["oqpsk"] else uw
    bits[start:start + len(w)] = w


def p_mutation_family(fb, seed=2):
    """Arm-wise inversion, a one-bit-wrong UW next to its exact twin, exact UW copies planted around the search gate
    `cntr > number_of_bits - 68` of a synced frame, one-bit slips, erasure and saturated runs, -1 values in the continuous
    stream, long noise on the idle counter, and LostSignal between calls."""
    g = p_geometry(fb)
    rng = np.random.default_rng(seed)
    F = g["frame"]
    out = []
    sizes = [1, 31, 32, 33, 500, 2049]

    def add(soft, tag, lost=(), **facts):
        out.append(member(soft, cut_sequence(len(soft), rng, sizes), lost=lost, tag=tag, **facts))

    base, sus = p_frames(fb, 5, seed=seed)
    pre = noise_bits(rng, 50)
    bits = np.concatenate([pre, base])
    soft = to_soft(bits)
    add(soft, "p-clean", sus=sus, n_frames=5)
    if g["oqpsk"]:
        for arm in (0, 1):
            s = soft.copy(); s[arm::2] = invert(s[arm::2])
            add(s, "p-invert-arm%d" % arm)
        add(invert(soft), "p-invert-both", sus=sus, n_frames=5)
    else:
        add(invert(soft), "p-invert-both")
    # one UW bit wrong on the first frame: no sync there (tolerance 0); the exact twin syncs
    for k in (0, 13, 31):
        b = bits.copy(); _set_uw(b, len(pre), g, flip=(k,))
        add(to_soft(b), "p-uw-wrong-%d" % k, uw_wrong=True, first_frame_start=len(pre))
    # planted exact UW copies in the data region of the second frame. A detector's register only shifts while it searches, so
    # with DCD up a copy syncs only if its first bit is framed at a counter value above number_of_bits - 68
    start2 = len(pre) + F                                        # UW of frame 2
    for d in range(-72, -63):
        b = bits.copy()
        first = start2 + g["uw_len"] - 1 + (g["number_of_bits"] + d) + 2     # framed with the counter at number_of_bits + d
        _set_uw(b, first, g)
        add(to_soft(b), "p-plant-%+d" % d, plant_first=first, plant_d=d)
    # one-bit slips in the middle of frame 2: insert or delete a bit
    mid = start2 + F // 2
    add(to_soft(np.concatenate([bits[:mid], [1], bits[mid:]])), "p-slip-insert")
    add(to_soft(np.concatenate([bits[:mid], bits[mid + 1:]])), "p-slip-delete")
    # erasures (128, left alone by an inverted arm) and saturated runs, inside the data and over the UW of frame 3
    for v in (128, 0, 255):
        s = soft.copy(); s[mid:mid + 300] = v; s[len(pre) + 2 * F - 10:len(pre) + 2 * F + 40] = v
        add(s, "p-run-%d" % v)
        if g["oqpsk"]:
            s2 = s.copy(); s2[1::2] = invert(s2[1::2])
            add(s2, "p-run-%d-inverted-arm" % v)
    # -1 values scattered in the continuous stream
    s = soft.copy(); s[rng.choice(len(s), 40, replace=False)] = -1
    add(s, "p-minus-one")
    # long noise on the idle counter before the first UW
    nz = noise_bits(rng, 3 * F + 17)
    add(to_soft(np.concatenate([nz, base])), "p-long-noise", sus=sus, n_frames=5)
    # LostSignal between calls in the middle of frame 2: the layer idles until frame 3's UW
    cuts = [start2 + 700, len(soft) - start2 - 700]
    out.append(member(soft, cuts, lost={0}, tag="p-lost-mid-frame"))
    return out


def p_dcd_deviation_stream(seed=3, copy=True):
    """10.5 kbps, the case the frame layer's one known deviation (DESIGN.md section 8) is about. Six back-to-back frames;
    the UWs of frames 1..4 are corrupted (three bits each), so after frame 0's sync the counter wraps on its own and stays
    aligned. The delay line makes the signal units completed at the ends of frames 0..2 fail their CRCs (the decoder's
    start-up); those completed at the end of frame 3 are good. Calls: up to just past frame 0, then a tick, which takes DCD
    down (frame 0's failures left the countdown at 0); up to just past frame 2; up to just past an exact UW copy inside
    frame 4's data region; the rest. In the reference frame 3's CRCs raise DCD at its last bit, so the detectors stop
    searching and the copy is ignored; the device applies them at the end of the call and so syncs on the copy.
    -> dict(soft, cuts, ticks (call indices followed by a tick), copy_first, call (index of the call holding the copy))"""
    fb = 10500
    g = p_geometry(fb)
    F = g["frame"]
    rng = np.random.default_rng(seed)
    base, _ = p_frames(fb, 6, seed=seed)
    pre = noise_bits(rng, 40)
    bits = np.concatenate([pre, base])
    s0 = len(pre)
    for f in (1, 2, 3, 4):
        _set_uw(bits, s0 + f * F, g, flip=(5, 17, 29))
    copy_first = s0 + 4 * F + g["uw_len"] + g["bits_in_header"] + 1000
    if copy:
        _set_uw(bits, copy_first, g)
    stops = [s0 + F + 10, s0 + 3 * F + 10, copy_first + g["uw_len"] + 100, len(bits)]
    cuts = list(np.diff([0] + stops))
    return dict(soft=to_soft(bits), cuts=cuts, ticks={0}, copy_first=copy_first, call=2)


# ---------------------------------------------------------------------------------------------------------------- C-channel
C_PRE1, C_PRE2 = 216866263330005, 3012071630031408
C_MASK = (1 << 52) - 1


@functools.lru_cache(maxsize=1)
def c_source():
    """soft bits of the committed 8400 bps recording from the restated demodulator, with the restated C-channel's DCD fed back
    as test_c_channel_frames_on_reference_recording computes them"""
    import os
    from oracle import restated
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    import json
    with open(os.path.join(root, "tests", "golden", "expected_outputs.json")) as fh:
        kw = dict(json.load(fh)["oqpsk_8400"]["kw"])
    pcm = np.load(os.path.join(root, "tests", "golden", "oqpsk_8400_excerpt.npz"))["pcm"]
    o = restated.OracleDemod("oqpsk", **kw); oc = restated.OracleCChannel()
    acc = []
    for k, a in enumerate(range(0, len(pcm), 4800)):
        o.write(pcm[a:a + 4800])
        s = o.take_soft(); acc.append(s); oc.process(s)
        o.set_dcd(int(oc.dcd))
        if k % 10 == 9:
            oc.update_dcd(); o.set_dcd(int(oc.dcd))
    o.close(); oc.close()
    return np.concatenate(acc)


def c_arm_words(soft, t):
    """the 52-bit registers of both arms after stream bit t (arm of bit t, arm of bit t - 1), hard-decided"""
    b = (np.asarray(soft[:t + 1]).astype(np.int64) & 255) >= 128
    words = []
    for end in (t, t - 1):
        v = 0
        for k in range(end - 2 * 51, end + 1, 2):
            v = (v << 1) | int(b[k])
        words.append(v & C_MASK)
    return words


def c_detect(word):
    """(hit, inverted, which) of one 52-bit register against the two preamble words, as cc_uw tests them"""
    for which, pre in ((1, C_PRE1), (2, C_PRE2)):
        x = bin(word ^ pre).count("1")
        if x >= 46:
            return True, True, which
        if x <= 6:
            return True, False, which
    return False, False, 0


def c_arm_hits(arm_bits):
    """(word, index) of every hit of one arm's detector (cc_uw) over a bit sequence that begins with word 2's register
    empty of it, indices counted from the start of word 2 (its last 52 bits)"""
    r1 = r2 = 0
    hits, off = [], len(arm_bits) - 52
    for k, v in enumerate(arm_bits):
        r1 = ((r1 << 1) | v) & C_MASK
        x = bin(r1 ^ C_PRE1).count("1")
        if x <= 6 or x >= 46:
            hits.append((1, k - off)); continue
        r2 = ((r2 << 1) | v) & C_MASK
        x = bin(r2 ^ C_PRE2).count("1")
        if x <= 6 or x >= 46:
            hits.append((2, k - off))
    return hits


def c_sync_points(soft):
    """stream indices t where both arms hold a preamble word at t - 1 and t (the bit a sync fires on)"""
    b = ((np.asarray(soft).astype(np.int64) & 255) >= 128).astype(np.int64)
    out = []
    for t in range(104, len(b)):
        if all(c_detect(w)[0] for w in c_arm_words(soft, t)) and not (out and t - out[-1] < 100):
            out.append(t)
    return out


def _c_set_word(soft, end, word, nbits=52):
    """write a 52-bit word MSB first on the arm whose last bit is stream index `end`"""
    for i in range(nbits):
        soft[end - 2 * (nbits - 1 - i)] = HI if (word >> (nbits - 1 - i)) & 1 else LO


def c_family(seed=4):
    """Frames of the recording spliced after 0..63 filler bits; both preamble words at 6 and 7 errors, inverted at 46 and 45
    matching bits, on one arm only; frames split across calls and LostSignal in the middle of a frame."""
    rng = np.random.default_rng(seed)
    src = c_source()
    syncs = c_sync_points(src)
    t0 = syncs[0]
    body = src[t0 - 120:].copy()                                 # from just before the first preamble's last bits
    sync_in_body = [t - (t0 - 120) for t in syncs]
    out = []
    sizes = [1, 63, 64, 840, 4096, 9000]
    for pre in range(0, 64, 3):
        s = np.concatenate([to_soft(noise_bits(rng, pre)), body])
        out.append(member(s, cut_sequence(len(s), rng, sizes), tag="c-shift-%d" % pre, syncs=[t + pre for t in sync_in_body]))
    # the second frame's preamble rewritten exactly, then k bits wrong on both arms (inverted: complemented first)
    t = sync_in_body[1]
    w_t, w_t1 = c_arm_words(body, t)
    for inverted in (False, True):
        for k in (6, 7):
            s = body.copy()
            for end, w in ((t, w_t), (t - 1, w_t1)):
                hit, inv, which = c_detect(w)
                word = C_PRE1 if which == 1 else C_PRE2
                if inverted:
                    word ^= C_MASK
                for p in rng.choice(52, k, replace=False):
                    word ^= 1 << int(p)
                _c_set_word(s, end, word)
            out.append(member(s, cut_sequence(len(s), rng, sizes), tag="c-pre-%s-%d" % ("inv" if inverted else "norm", k),
                              errors=k, inverted=inverted, target_sync=t))
    # one arm only: the other arm's word wrecked
    s = body.copy()
    _c_set_word(s, t - 1, (c_arm_words(body, t)[1] ^ 0x5A5A5A5A5A5) & C_MASK)
    out.append(member(s, cut_sequence(len(s), rng, sizes), tag="c-one-arm", target_sync=t, errors=99, inverted=False))
    # word 1 matching while word 2 is mid-shift: on the arm that carries word 2, the 51 - j bits before it are made word 1's
    # first 51 - j bits. Where word 1's register then matches (within 6) at word 2's bit j, the second register skips that
    # bit; for some j word 2 is still found at its end (the skip costs few bits), for others it is not (word2_lost, from
    # c_arm_hits on the planted bits).
    ends = {c_detect(w)[2]: (end, c_detect(w)[1]) for end, w in ((t, w_t), (t - 1, w_t1))}
    e2, inv2 = ends[2]
    p1 = [(C_PRE1 >> (51 - i)) & 1 for i in range(52)]
    for j in (3, 6, 7, 9, 13, 14, 20):
        s = body.copy()
        first2 = e2 - 2 * 51                                     # stream index of word 2's first bit
        for i in range(51 - j):
            s[first2 - 2 * (51 - j - i)] = HI if p1[i] ^ inv2 else LO
        arm = (((s[first2 - 2 * (51 - j):e2 + 1:2].astype(np.int64) & 255) >= 128) ^ inv2).astype(int).tolist()
        hits = c_arm_hits(arm)                                   # the planted word 1 and the recorded word 2, as received
        out.append(member(s, cut_sequence(len(s), rng, sizes), tag="c-word1-midshift-%d" % j, midshift=j,
                          word1_hit=(1, j) in hits, word2_lost=(2, 51) not in hits, target_sync=t))
    # LostSignal in the middle of frames 2 and 4, between calls
    s = body.copy()
    cuts = [sync_in_body[1] + 2000, sync_in_body[3] + 1000 - sync_in_body[1] - 2000]
    cuts += cut_sequence(len(s) - sum(cuts), rng, sizes)
    out.append(member(s, cuts, lost={0, 1}, tag="c-lost-mid-frame"))
    return out


# ---------------------------------------------------------------------------------------------------------------- R/T channel
FILL = np.tile(np.array([0, 0, 1, 1], dtype=np.uint8), 200)


def rt_info_bits(info_bytes, n_dec):
    """LSB-first bits of the packet, scrambled, zero-padded to the n_dec decoded bits of the trial that carries it"""
    info = np.unpackbits(np.asarray(info_bytes, dtype=np.uint8), bitorder="little")
    u = np.zeros(n_dec, dtype=np.uint8)
    u[:len(info)] = info ^ synth.scrambler_sequence(len(info))
    return u


def crc_unit(body):
    c = synth.crc16(body)
    return np.concatenate([np.asarray(body, dtype=np.uint8), np.array([c & 0xFF, c >> 8], dtype=np.uint8)])


def rt_t_packet_bits(rng, n_sus):
    """OQPSK T packet: 6-byte header (4 + CRC) and n_sus 12-byte signal units (10 + CRC) in one interleaver block of
    5 + 3 (n_sus - 1) columns (decoded at the trial of that length). -> (coded block bits, info bytes)"""
    info = np.concatenate([crc_unit(rng.integers(0, 256, 4, dtype=np.uint8))] +
                          [crc_unit(rng.integers(0, 256, 10, dtype=np.uint8)) for _ in range(n_sus)])
    cols = 5 + 3 * (n_sus - 1)
    coded, _ = synth.conv_encode_stream(rt_info_bits(info, 32 * cols), 0)
    return synth.interleave(coded, cols), info


def rt_msk_t_packet_bits(rng, target):
    """MSK T packet whose initial signal unit (the 6 bits after the header and one unit) announces `target` signal units,
    i.e. a block of (target + 1) * 3 + 2 columns, interleaved as 5 columns then groups of 3 (deinterleaveMSK_ba)"""
    nblk = (target + 1) * 3 + 2
    v = target - 2 if target < 16 else 2 * target - 4
    info = rng.integers(0, 256, 4 * nblk - 1, dtype=np.uint8)
    info[:6] = crc_unit(info[:4])
    u = np.unpackbits(info, bitorder="little")
    u[48 + 96:48 + 96 + 6] = [(v >> i) & 1 for i in range(6)]
    info = np.packbits(u, bitorder="little")
    dec = np.zeros(32 * nblk, dtype=np.uint8)
    n = len(u) - 8                                               # the last byte's bits stay scrambled zeros (chop(1))
    dec[:n] = u[:n] ^ synth.scrambler_sequence(n)
    coded, _ = synth.conv_encode_stream(dec, 0)
    blocks = [synth.interleave(coded[:320], 5)]
    for g in range(5, nblk, 3):
        blocks.append(synth.interleave(coded[64 * g:64 * (g + 3)], 3))
    return np.concatenate(blocks), info[:len(info)], nblk


def rt_burst(fb, block_bits, fill=80, uw_flip=(), inverted=False, marker=True, tail=None):
    """marker, `fill` filler bits, the unique word (both arms at 10.5 kbps) with bits flipped, the block, a tail. At 10.5 kbps
    the detectors stop searching for number_of_bits - 68 bits after a sync while DCD is up, so the default tail keeps the
    next burst's UW clear of that stretch."""
    if tail is None:
        tail = 5000 if int(fb) == 10500 else 240
    uw = UW_BITS.copy()
    for k in uw_flip:
        uw[k] ^= 1
    if int(fb) == 10500:
        uw = np.repeat(uw, 2)
    bits = np.concatenate([FILL[:fill], uw, block_bits, np.tile(np.array([0, 1, 1, 0], dtype=np.uint8), tail // 4)])
    if inverted:
        bits = 1 - bits
    soft = to_soft(bits)
    return np.concatenate([np.array([-1], dtype=np.int16), soft]) if marker else soft


def rt_r_block(payload17):
    c = synth.crc16(payload17)
    info = np.concatenate([np.asarray(payload17, dtype=np.uint8), np.array([c & 0xFF, c >> 8], dtype=np.uint8)])
    coded, _ = synth.conv_encode_stream(rt_info_bits(info, 160), 0)
    return synth.interleave(coded, 5), info


def rt_family(fb, seed=5):
    """Members of several bursts each: R packets; T packets of 2..31 signal units (10.5 kbps: 31 fills the whole block) or
    MSK T packets announcing their length; the UW at 0..400 bits from the marker across the 10.5 kbps window
    |muw - 80| <= 150 and the MSK gate muw > 250; UWs at 4 and 5 errors, normal and inverted; bursts with no marker; garbage
    bursts (failed trials); MSK T packets longer than the burst time-out."""
    rng = np.random.default_rng(seed)
    oq = int(fb) == 10500
    uwl = 64 if oq else 32
    out = []
    sizes = [1, 97, 320, 1000, 4096]

    def add(bursts, tag, **facts):
        s = np.concatenate(bursts)
        out.append(member(s, cut_sequence(len(s), rng, sizes), tag=tag, **facts))

    r_blocks = [rt_r_block(rng.integers(0, 256, 17, dtype=np.uint8)) for _ in range(4)]
    add([rt_burst(fb, b) for b, _ in r_blocks], "rt-r", planted=[(1, 0, i) for _, i in r_blocks])
    add([rt_burst(fb, b, inverted=bool(k & 1)) for k, (b, _) in enumerate(r_blocks)], "rt-r-inverted",
        planted=[(1, 0, i) for _, i in r_blocks])
    if oq:
        for group in ([2, 5, 16], [30, 31], [3, 9, 23]):
            tp = [rt_t_packet_bits(rng, n) for n in group]
            add([rt_burst(fb, b) for b, _ in tp], "rt-t-%s" % "-".join(map(str, group)),
                planted=[(2, n, i) for n, (_, i) in zip(group, tp)])
    else:
        for group in ([3, 4, 9], [12, 15, 20]):
            tp = [rt_msk_t_packet_bits(rng, n) for n in group]
            add([rt_burst(fb, b) for b, _, _ in tp], "rt-t-%s" % "-".join(map(str, group)),
                planted=[(2, n, i) for n, (_, i, _) in zip(group, tp)])
        # longer than the burst time-out (TotalNumberOfBits = 3 fb after the UW): the time-out idles the counter, which
        # keeps filling the block, so the packet still completes
        tp = [rt_msk_t_packet_bits(rng, n) for n in (28, 5)]
        add([rt_burst(fb, b) for b, _, _ in tp], "rt-t-timeout", planted=[(2, 28, tp[0][1]), (2, 5, tp[1][1])])
    # the UW at distances 0..400 from the marker: the 10.5 kbps window ends at muw 230 (UW end = fill + 64), the MSK gate at 250
    edge = 230 - uwl if oq else 250 - uwl
    fills = sorted(set(list(range(0, 401, 40)) + [edge - 1, edge, edge + 1, edge + 2]))
    for k in range(0, len(fills), 4):
        chunk = fills[k:k + 4]
        add([rt_burst(fb, r_blocks[j % 4][0], fill=f) for j, f in enumerate(chunk)], "rt-muw-%d" % chunk[0],
            fills=chunk, accepted=[f + uwl <= (230 if oq else 250) for f in chunk])
    # 4 and 5 UW errors, normal and inverted
    for nerr in (4, 5):
        for inv in (False, True):
            flips = tuple(rng.choice(32, nerr, replace=False))
            add([rt_burst(fb, r_blocks[j][0], uw_flip=flips, inverted=inv) for j in range(2)], "rt-uw%d-%s" % (nerr, "inv" if inv else "norm"),
                uw_errors=nerr)
    # no marker (muw keeps counting from the previous burst), garbage bursts, then a good one
    g = rng.integers(0, 2, 64 * 20).astype(np.uint8)
    add([rt_burst(fb, r_blocks[0][0]), rt_burst(fb, r_blocks[1][0], marker=False, fill=8), rt_burst(fb, g), rt_burst(fb, r_blocks[2][0])],
        "rt-nomarker-garbage")
    return out


def rt_many_packets(fb, n, seed=6):
    """n R packets back to back, each in its own burst; -> (soft, payloads, index of each packet's UW last bit)"""
    rng = np.random.default_rng(seed)
    bl = [rt_r_block(rng.integers(0, 256, 17, dtype=np.uint8)) for _ in range(n)]
    bursts = [rt_burst(fb, b) for b, _ in bl]
    uwl = 64 if int(fb) == 10500 else 32
    starts = np.cumsum([0] + [len(b) for b in bursts[:-1]])
    return np.concatenate(bursts), [i for _, i in bl], [int(s) + 1 + 80 + uwl - 1 for s in starts]
