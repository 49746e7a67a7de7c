"""CPU: REC_PAD, the slot the FM engine keeps for a possible sync loss after the P1 frame of a block that also ends a
P3 / P4 frame (include/nrsc5_b200.h), stands for no call: every reader of the record stream skips it."""
import os
import re
import struct

from nrsc5_b200 import engine as eng

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_parser_skips_pad_records():
    raw = b""
    raw += struct.pack("<II", eng.REC_SYNC, 8) + struct.pack("<fi", 12.5, 3)
    raw += struct.pack("<II", eng.REC_BER, 4) + struct.pack("<f", 0.01)
    raw += struct.pack("<II", eng.REC_FRAME, 8 + 3) + struct.pack("<II", 0, 24) + b"\x01\x02\x03" + b"\0"
    raw += struct.pack("<II", eng.REC_PAD, 0)                 # the slot, not needed: no call
    raw += struct.pack("<II", eng.REC_FRAME, 8 + 2) + struct.pack("<II", 1, 16) + b"\x04\x05" + b"\0\0"
    raw += struct.pack("<II", eng.REC_PAD, 0)
    offs = []
    recs = eng.parse_records(raw, offs)
    assert [t for t, _ in recs] == [eng.REC_SYNC, eng.REC_BER, eng.REC_FRAME, eng.REC_FRAME]
    assert [r["lc"] for t, r in recs if t == eng.REC_FRAME] == [0, 1]
    assert offs == [0, 16, 28, 56]                            # byte offsets of the records that are kept


def test_pad_record_is_declared_and_skipped_by_the_dropin():
    src = open(os.path.join(ROOT, "include", "nrsc5_b200.h")).read()
    assert re.search(r"NRSC5B_REC_PAD\s*=\s*%d\b" % eng.REC_PAD, src)
    seam = open(os.path.join(ROOT, "nrsc5_b200", "dropin", "input_seam.c")).read()
    assert re.search(r"case NRSC5B_REC_PAD:\s*/\*[^*]*\*/\s*break;", seam)
