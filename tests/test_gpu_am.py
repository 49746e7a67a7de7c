"""GPU parity of the AM (hybrid MA1, all-digital MA3) path through the C ABI: cs16 in, P1 / P3 / PIDS PDUs and events out, against
the oracle (oracle/nrsc5_oracle_am.c, itself pinned to the unmodified reference) and the golden vectors.

First GPU run: round 1, all green (they ran as `gpu_new` until then; their CPU twins on the emulated kernels
are in tests/test_emu_engine.py)."""
import numpy as np
import pytest

import common
import port
import reftap
import nrsc5_b200
from nrsc5_b200 import engine as eng
from nrsc5_b200 import synth_am

pytestmark = pytest.mark.gpu


def run_am(captures, chunk=None, cu8=False):
    """captures: int16 cs16 arrays, or (cu8=True) uint8 arrays at 1 488 375 S/s that the engine decimates by 32."""
    cap = max(2 * c.size for c in captures) // (16 if cu8 else 1) + 4096
    with nrsc5_b200.Engine(nstreams=len(captures), input_capacity=cap, log_capacity=4 << 20, mode="am", input_cs16=not cu8) as e:
        if cu8:
            n = max(c.size for c in captures)
            step = chunk or (1 << 22)
            for off in range(0, n, step):
                for s, c in enumerate(captures):
                    piece = c[off: off + step]
                    if piece.size:
                        e.push_cu8(s, piece[: piece.size & ~3])
                e.process()
        elif chunk is None:
            for s, c in enumerate(captures):
                e.push_cs16(s, c[: c.size & ~1])
            e.process()
        else:
            n = max(c.size for c in captures)
            for off in range(0, n, chunk):
                for s, c in enumerate(captures):
                    piece = c[off: off + chunk]
                    if piece.size:
                        e.push_cs16(s, piece[: piece.size & ~1])
                e.process()
        return [e.drain(s) for s in range(len(captures))]


def digest(recs):
    out = []
    for t, r in recs:
        if t == eng.REC_FRAME:
            out.append(("F", r["lc"], r["nbits"], r["bits"]))
        elif t == eng.REC_PIDS:
            out.append(("P", r["bits"], r["crc_ok"]))
        elif t == eng.REC_SYNC:
            out.append(("S", r["psmi"], tuple(r["flags"])))
        elif t == eng.REC_LOST_SYNC:
            out.append(("L",))
        elif t == eng.REC_BER:
            out.append(("B", round(r["cber"], 6)))
    return out


def oracle_digest(log):
    out = []
    for t, p in log.records:
        if t == reftap.REC_FRAME:
            out.append(("F", p["lc"], p["nbits"], p["bits"]))
        elif t == reftap.REC_PIDS:
            out.append(("P", p["bits"], p["crc_ok"]))
        elif t == reftap.REC_SYNC:
            out.append(("S", p["psmi"], tuple(p["flags"])))
        elif t == reftap.REC_LOST_SYNC:
            out.append(("L",))
        elif t == reftap.REC_BER:
            out.append(("B", round(p["cber"], 6)))
    return out


@pytest.mark.parametrize("name", list(common.AM_CASES))
def test_am_pdus_bit_exact(name):
    cap = synth_am.make_am_ma1(**common.AM_CASES[name])
    got = digest(run_am([cap.cs16])[0])
    want = oracle_digest(port.decode_am(cap.cs16))
    assert got == want
    assert sum(1 for e in got if e[0] == "F" and e[1] == 0) >= 32 and sum(1 for e in got if e[0] == "F" and e[1] == 1) >= 4
    g = common.golden("synth_am.json")[name]
    if common.fnv1a32(cap.cs16[:1 << 18].tobytes()) == g["input_fnv"]:
        assert [common.fnv1a32(e[3]) for e in got if e[0] == "F"] == [e[3] for e in g["events"] if e[0] == "F"]


def test_am_streams_independent_and_chunked():
    caps = [synth_am.make_am_ma1(nframes=8, seed=40 + i, lead_in=100 + 333 * i, cfo_hz=0.4 * i, psmi=2 if i == 2 else 1)
            for i in range(3)]
    whole = run_am([c.cs16 for c in caps])
    parts = run_am([c.cs16 for c in caps], chunk=1 << 15)
    for c, a, b in zip(caps, whole, parts):
        want = oracle_digest(port.decode_am(c.cs16))
        assert digest(a) == want
        assert digest(b) == want


@pytest.mark.parametrize("psmi", [1, 2])
def test_am_cu8_input_bit_exact(psmi):
    """cu8 at 1 488 375 S/s (input_push_cu8 in AM mode): five halfband stages on the device, then the same chain.
    Pushed in odd-sized pieces so that groups of 32 raw samples straddle pushes and the raw ring wraps."""
    cap = synth_am.make_am_ma1(nframes=8, seed=50 + psmi, lead_in=555, carrier=8000.0, unit=40.0, cfo_hz=-0.6, psmi=psmi)
    cu8 = synth_am.am_to_cu8(cap.cs16)
    want = oracle_digest(port.decode_am(cu8))
    assert sum(1 for e in want if e[0] == "F" and e[1] == 0) >= 16
    assert digest(run_am([cu8], cu8=True)[0]) == want
    assert digest(run_am([cu8], chunk=300004, cu8=True)[0]) == want
