"""Generate tests/golden/expected_outputs.json by running the VERBATIM reference (oracle/_ref, built from
/root/reference by oracle/Makefile) over the committed PCM excerpts. Build container only.

For each excerpt: SHA-256 of the emitted soft-bit stream, its length, the final loop state, the coarse
estimator log digest, and the signal units + CRC flags that the restated AeroL P-channel framing decodes
from those soft bits (the Viterbi arithmetic inside is the restated libcorrect: parity unpinned upstream,
pinned here by CRC-16-valid SUs)."""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref, restated  # noqa: E402
import control_schedules  # noqa: E402

CASES = {
    "oqpsk_10500": dict(kind="oqpsk", kw=dict(fb=10500, freq_center=5760, lockingbw=10500, fft_power=14, signalthreshold=0.65, afc=True)),
    "oqpsk_10500_noafc_dcd": dict(kind="oqpsk", excerpt="oqpsk_10500", dcd_at=96000,
                                  kw=dict(fb=10500, freq_center=5757, lockingbw=10500, fft_power=14, signalthreshold=0.65, afc=False)),
    "oqpsk_8400": dict(kind="oqpsk", nosu=True, kw=dict(fb=8400, freq_center=8000, lockingbw=10500, fft_power=14, signalthreshold=0.65, afc=True)),
    "burst_msk_1200_a": dict(kind="burst_msk", nosu=True, kw=dict(fb=1200.0, freq_center=1000.0, lockingbw=1800.0, signalthreshold=0.6)),
    "burst_msk_1200_b": dict(kind="burst_msk", nosu=True, kw=dict(fb=1200.0, freq_center=1000.0, lockingbw=1800.0, signalthreshold=0.6)),
    "burst_oqpsk_10500": dict(kind="burst_oqpsk", nosu=True, kw=dict(fb=10500.0, freq_center=8000.0, lockingbw=10500.0, signalthreshold=0.6)),
    "msk_600": dict(kind="msk", kw=dict(fb=600, freq_center=1000, lockingbw=900, fft_power=13, signalthreshold=0.5, afc=True)),
    # BASELINE cfg 2 (continuous 1200 bps MSK, mskdemodulator.cpp:189-250 branch): synthetic fixture (tools/make_synth_fixtures.py)
    "msk_1200": dict(kind="msk", kw=dict(fb=1200, freq_center=2000, lockingbw=1800, fft_power=13, signalthreshold=0.5, afc=True)),
    "msk_1200_noafc_dcd": dict(kind="msk", excerpt="msk_1200", dcd_at=144000,
                               kw=dict(fb=1200, freq_center=2030, lockingbw=1800, fft_power=13, signalthreshold=0.5, afc=False)),
}
# the run-time controls (tests/control_schedules.py): the centre-change slot, AFC, squelch, CPU-reduce and DCD called between writes
for _name, (_kind, _kw, _) in control_schedules.RECORDINGS.items():
    CASES[_name + "_controls"] = dict(kind=_kind, excerpt=_name, kw=_kw, nosu=_kw["fb"] == 8400, controls=True)


def run_case(name, case, chunk=4800):
    import multiprocessing as mp
    pcm = np.load(os.path.join(ROOT, "tests", "golden", case.get("excerpt", name) + "_excerpt.npz"))["pcm"]
    sched = [(case["dcd_at"], 1)] if "dcd_at" in case else None
    controls = control_schedules.events(control_schedules.recording_schedule(case["excerpt"], len(pcm))) if case.get("controls") else []
    ctx = mp.get_context("spawn")            # fresh process: the reference keeps function-local statics
    with ctx.Pool(1, maxtasksperchild=1) as pool:
        soft, state, cfe = pool.apply(ref.run_demod_job, ((case["kind"], case["kw"], pcm, chunk, sched, controls),))
    if case.get("nosu"):
        su = np.zeros((0, 12), dtype=np.uint8); ok = np.zeros(0, dtype=np.int32); fr = np.zeros(0, dtype=np.int64)
    else:
        p = restated.OraclePChannel(case["kw"]["fb"])
        p.process(soft)
        su, ok, fr = p.take_sus()
    rt_packets = []
    if case["kind"].startswith("burst"):
        # R/T packet layer (restated AeroL burst branch; pinned by the CRC-16s it verifies) on the reference's soft bits
        rt = restated.OracleRTChannel(case["kw"]["fb"])
        rt.process(soft)
        rt_packets = [dict(type=q["type"], nsus=q["nsus"], n_bytes=int(len(q["bytes"])), sha256=hashlib.sha256(q["bytes"].tobytes()).hexdigest())
                      for q in rt.packets()]
    c_frames = {}
    if case["kw"]["fb"] == 8400:
        # C-channel frame layer (restated AeroL::DecodeC; pinned by the sub-band signal units' CRC-16s) on the reference's soft bits
        cc = restated.OracleCChannel()
        cc.process(soft)
        su, cok, voice = cc.take_frames()
        c_frames = dict(n_frames=int(len(su)), n_su_crc_ok=int(cok.sum()),
                        sha256=hashlib.sha256(su.tobytes() + cok.astype("<i4").tobytes() + voice.tobytes()).hexdigest())
    return {
        "c_frames": c_frames,
        "rt_packets": rt_packets,
        "kind": case["kind"], "kw": case["kw"], "excerpt": case.get("excerpt", name), "chunk": chunk,
        "dcd_schedule": sched or [],
        **({"controls": [[int(a), [list(c) for c in calls]] for a, calls in controls]} if controls else {}),
        "n_soft": int(len(soft)), "soft_sha256": hashlib.sha256(soft.astype("<i2").tobytes()).hexdigest(),
        "soft_head": [int(x) for x in soft[:64]],
        "state": {k: float(v) for k, v in state.items()},
        "cfe_log_sha256": hashlib.sha256(np.asarray(cfe, dtype="<f8").tobytes()).hexdigest(), "n_cfe": int(len(cfe)),
        "n_su": int(len(ok)), "n_su_crc_ok": int(ok.sum()),
        "su_sha256": hashlib.sha256(su.tobytes() + ok.astype("<i4").tobytes()).hexdigest(),
        "su_first_ok": [int(x) for x in su[np.argmax(ok)]] if ok.any() else [],
    }


if __name__ == "__main__":
    out = {name: run_case(name, case) for name, case in CASES.items()}
    for k, v in out.items():
        print(k, v["n_soft"], v["n_su"], v["n_su_crc_ok"], v["state"]["mse"])
    with open(os.path.join(ROOT, "tests", "golden", "expected_outputs.json"), "w") as fh:
        json.dump(out, fh, indent=1, sort_keys=True)
