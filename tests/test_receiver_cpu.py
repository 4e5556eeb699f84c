"""The receiver's transmitter and argument checks, without a device: synth.pchannel_bits_from_sus framed signal units come back
from the restated P-channel frame layer exactly, ACARS messages framed that way come back from the Reassembler, and Receiver
and tools/receive.py refuse bad arguments before they touch a device."""
import os
import subprocess
import sys

import numpy as np
import pytest

import frame_streams as fs
import reasm_synth
from jaero_b200 import synth
from oracle import restated

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sus_per_frame(fb):
    fp = synth.frame_params(fb)
    return fp["blocks"] * 64 * fp["cols"] // 2 // 96


def _messages(seed, n):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        aes = 0x400000 + int(rng.integers(1, 1 << 20))
        reg = "G-%s" % "".join("ABCDEFGHJK"[k] for k in rng.integers(0, 10, 4))
        label = "".join("HQ15AB_"[k] for k in rng.integers(0, 7, 2))
        text = "MSG %d SEED %d" % (i, seed) + "X" * int(rng.integers(0, 60))
        ud = reasm_synth.acars_userdata(reg, label, ord("A") + i % 26, text)
        out.append((aes, reg, label, text, reasm_synth.isu_to_sus(aes, 0x90, i & 15, (i * 3) & 15, ud)))
    return out


def _decode(fb, sus, loop):
    """the SUs framed with two frames of fill before and after (the decoder's start-up and its delay line), through the restated
    frame layer -> (12-byte units, crc_ok)"""
    k = _sus_per_frame(fb)
    seq = [synth.FILL_SU] * (2 * k) + list(sus) + [synth.FILL_SU] * (2 * k)
    bits = synth.pchannel_bits_from_sus(fb, seq, loop=loop, even_parity=loop)
    assert len(bits) % synth.frame_params(fb)["frame_bits"] == 0
    o = restated.OraclePChannel(fb)
    o.process(fs.to_soft(bits))
    b, ok, _ = o.take_sus()
    o.close()
    return b, ok


@pytest.mark.parametrize("loop", [False, True])
@pytest.mark.parametrize("fb", [600, 1200, 10500])
def test_framed_signal_units_come_back_exactly(fb, loop):
    rng = np.random.default_rng(fb + loop)
    given = [synth.make_su(rng, 0x71 if k % 4 == 0 else None) for k in range(3 * _sus_per_frame(fb) + 5)]
    b, ok = _decode(fb, given, loop)
    fill = synth.FILL_SU
    got = [x for x, o in zip(b, ok) if o]
    planted = [x for x in got if bytes(x[:10]) != fill]
    assert len(planted) == len(given)
    assert all(np.array_equal(x, g) for x, g in zip(planted, given))
    assert all(synth.crc16(x[:10]) == (int(x[10]) | int(x[11]) << 8) for x in planted)


@pytest.mark.parametrize("fb", [600, 1200, 10500])
def test_ten_byte_payloads_get_their_crc(fb):
    msgs = _messages(fb, 2)
    sus = [s for m in msgs for s in m[4]]
    b, ok = _decode(fb, sus, True)
    got = [bytes(x[:10]) for x, o in zip(b, ok) if o and bytes(x[:10]) != synth.FILL_SU]
    assert got == sus


def test_bad_signal_units_are_refused():
    with pytest.raises(ValueError):
        synth.pchannel_bits_from_sus(1200, [bytes(11)])
    bits = synth.pchannel_bits_from_sus(1200, [])
    assert len(bits) == synth.frame_params(1200)["frame_bits"]             # one frame of fill


@pytest.mark.parametrize("fb", [600, 1200, 10500])
def test_acars_messages_survive_framing_and_reassembly(fb):
    import jaero_b200
    msgs = _messages(100 + fb, 3)
    sus = [s for m in msgs for s in m[4]]
    b, ok = _decode(fb, sus, fb != 10500)
    rs = jaero_b200.Reassembler()
    for x, o in zip(b, ok):
        if o:
            rs.push_su(x)
    recs = rs.pop_all()
    rs.close()
    got = [(r["aesid"], r["reg"].decode("latin-1").strip("."), r["label"].decode(), r["text"].decode("latin-1")) for r in recs]
    assert got == [(aes, reg, label, text) for aes, reg, label, text, _ in msgs]


@pytest.mark.parametrize("kw, err", [
    (dict(input_rate=2.4e6 + 0.5, fmt="cu8"), ValueError),
    (dict(input_rate=-48000, fmt="cu8"), ValueError),
    (dict(input_rate=2.4e6, fmt="cs8"), ValueError),
    (dict(input_rate=2.4e6, fmt="cu8", acquire_seconds=0), ValueError),
    (dict(input_rate=2.4e6, fmt="cu8", acquire_seconds=-1.0), ValueError),
    (dict(input_rate=2.4e6, fmt="cu8", block_seconds=1e-5), ValueError),
    (dict(input_rate=2.4e6, fmt="cu8", block_seconds=0), ValueError),
    (dict(input_rate=2.4e6, fmt="cu8", block_seconds=2.0), ValueError),
    (dict(input_rate=2.4e6, fmt="cu8", threshold=3.0), TypeError),
])
def test_receiver_refuses_bad_arguments_before_the_device(kw, err):
    import jaero_b200
    with pytest.raises(err):
        jaero_b200.Receiver(**kw)


def test_receiver_block_must_hold_one_output_sample():
    """at 2.5 MS/s the down-converter makes one 48 kHz sample per 52.08 input samples: a 20 us block (50 samples) is refused"""
    import jaero_b200
    with pytest.raises(ValueError, match="shorter than one"):
        jaero_b200.Receiver(2.5e6, "cu8", block_seconds=20e-6)


@pytest.mark.parametrize("args, text", [
    (["--rate", "2.4e6x", "--format", "cu8", "-"], "--rate"),
    (["--rate", "2400000.5", "--format", "cu8", "-"], "--rate"),
    (["--rate", "2400000", "--format", "cs8", "-"], "--format"),
    (["--rate", "2400000", "--format", "cu8", "--acquire", "0", "-"], "--acquire"),
    (["--rate", "2400000", "--format", "cu8", "--block", "0.00001", "-"], "--block"),
    (["--rate", "7", "--format", "cu8", "-"], "interpolation"),
])
def test_cli_refuses_bad_arguments(args, text):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "receive.py")] + args, capture_output=True, text=True,
                       stdin=subprocess.DEVNULL, timeout=120)
    assert r.returncode != 0
    assert text in r.stderr and "Traceback" not in r.stderr, r.stderr
    assert r.stdout == ""
