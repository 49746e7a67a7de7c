"""CPU tests: the C-ABI library loads, exports every symbol include/nrsc5_b200.h declares, and fails
loudly (no CPU fallback) when there is no CUDA device."""
import ctypes
import os
import re

import pytest

import nrsc5_b200
from nrsc5_b200 import engine as eng

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "nrsc5_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(nrsc5b_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    L = nrsc5_b200.load_library()
    names = declared_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/nrsc5_b200.h but not exported"
    assert b"sm_90a" in L.nrsc5b_version()


def test_sass_is_sm90a_only():
    import subprocess
    out = subprocess.run(["cuobjdump", "-lelf", nrsc5_b200.lib_path()], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(nrsc5_b200.EngineError):
        nrsc5_b200.Engine(nstreams=1, input_capacity=1 << 16)
    import numpy as np
    with pytest.raises(nrsc5_b200.EngineError):
        eng.halfband_fm(np.zeros(64, dtype=np.uint8))
    with pytest.raises(nrsc5_b200.EngineError):
        eng.l2_frames([(1, 4608, bytes(576))])              # L2 alone: no host path either
    with pytest.raises(nrsc5_b200.EngineError):
        eng.viterbi_k9(np.ones((1, 3 * 80), dtype=np.int8))  # the AM decoder alone: device only
    from nrsc5_b200 import channelizer
    with pytest.raises(nrsc5_b200.EngineError):
        channelizer.Channelizer([0, 9])                     # the channeliser needs a device; its tables do not:
    taps, ph = channelizer.make_tables([0, 9])
    assert taps.shape == (2, 256, 2) and ph.shape == (11907, 2)


def test_record_parser_roundtrip():
    import struct
    raw = b""
    raw += struct.pack("<II", eng.REC_SYNC, 8) + struct.pack("<fi", 12.5, 1)
    raw += struct.pack("<II", eng.REC_PIDS, 10) + bytes(range(10)) + b"\0\0"
    raw += struct.pack("<II", eng.REC_FRAME, 8 + 3) + struct.pack("<II", 0, 24) + b"\x01\x02\x03" + b"\0"
    raw += struct.pack("<II", eng.REC_LOST_SYNC, 0)
    recs = eng.parse_records(raw)
    assert [t for t, _ in recs] == [eng.REC_SYNC, eng.REC_PIDS, eng.REC_FRAME, eng.REC_LOST_SYNC]
    assert recs[0][1]["psmi"] == 1 and recs[2][1]["bits"] == b"\x01\x02\x03"


def test_l2_record_parser():
    """REC_L2 (include/nrsc5_b200.h): header, events in call order, PDU bytes; packet data is cut out of the PDU."""
    import struct
    pdu = bytes(range(40))
    ev = b""
    ev += struct.pack("<II", eng.EV_ALIGN, 12) + struct.pack("<3I", 1, 0, 24)
    ev += struct.pack("<II", eng.EV_AAS, 5) + b"hello" + b"\0\0\0"
    ev += struct.pack("<II", eng.EV_PACKET, 28) + struct.pack("<7I", 1, 0, 9, 1, 0, 6, 30)
    body = struct.pack("<8I", 4096, 1, 4608, 0x38D8D3, 0, len(pdu), len(ev), 7) + ev + pdu
    raw = struct.pack("<II", eng.REC_L2, len(body)) + body
    (ty, r), = eng.parse_records(raw)
    assert ty == eng.REC_L2 and (r["lc"], r["nbits"], r["pci"], r["ordinal"], r["frame_rec_off"]) == (1, 4608, 0x38D8D3, 7, 4080)
    assert [t for t, _ in r["events"]] == [eng.EV_ALIGN, eng.EV_AAS, eng.EV_PACKET]
    assert r["events"][1][1]["data"] == b"hello" and r["events"][2][1]["data"] == pdu[30:36] and r["pdu"] == pdu
