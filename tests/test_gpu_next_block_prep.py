"""GPU: with one CTA per stream (k_stream<false>), the set-up of a block in FINE sync - window offset, NCO angle and
phase - is computed during the previous block's sync, and committed at the block's start only if the block runs; its
NCO table and per-symbol phases are filled from it while the run is being decided.

The same MP1 captures go through the engine one-shot and in irregular pushes.  With the pushes, passes end where the
input runs out in the middle of a frame, so the set-up made during a pass's last block is discarded and the next
pass sets its first block up from the stream's state.  Both feeds must give byte-identical records (soft bits of
every block included), whose L1 PDUs and events are the oracle's.  A sync state forced between two pushes must take
effect at the next block, not be overridden by a set-up made before it."""
import numpy as np
import pytest

import port
import reftap
import nrsc5_b200
from nrsc5_b200 import engine as eng
from nrsc5_b200 import synth
from test_gpu_chain import kinds, oracle_kinds, pdus

pytestmark = pytest.mark.gpu

# push sizes in bytes, used in turn: none is a multiple of a block's input, so passes end mid-block and mid-frame
PUSHES = (3 * (1 << 16) + 4096, 5 * (1 << 16) + 12288, (1 << 17) + 3 * 4096)


@pytest.fixture(autouse=True)
def one_cta(monkeypatch):
    monkeypatch.setenv("NRSC5_B200_CLUSTER", "1")


def captures():
    caps = [synth.make_fm_mp1(nframes=2, seed=610 + i, lead_in=211 + 97 * i, cfo_hz=35.0 * i, noise_lsb=3.0)
            for i in range(2)]
    return [c.cu8[: c.cu8.size & ~3] for c in caps]


def run_raw(cu8s, pushes=None, force=None):
    """Every stream's raw record log.  pushes=None: all input, then one process; else pushes of the sizes in turn,
    a process after each.  force=(push index, state): set every stream's sync state before that push's process."""
    with nrsc5_b200.Engine(nstreams=len(cu8s), input_capacity=max(c.size for c in cu8s) + 4096,
                           log_capacity=8 << 20, emit_soft=True) as e:
        raw = [b"" for _ in cu8s]
        if pushes is None:
            for s, c in enumerate(cu8s):
                e.push_cu8(s, c)
            e.process()
            return [e.drain_raw(s) for s in range(len(cu8s))]
        off, k = 0, 0
        while off < max(c.size for c in cu8s):
            n = pushes[k % len(pushes)]
            for s, c in enumerate(cu8s):
                if c[off: off + n].size:
                    e.push_cu8(s, c[off: off + n])
            if force is not None and k == force[0]:
                for s in range(len(cu8s)):
                    e.set_sync_state(s, force[1])
            e.process()
            for s in range(len(cu8s)):
                raw[s] += e.drain_raw(s)
            off += n
            k += 1
        return raw


def test_pushed_equals_one_shot_and_oracle():
    cu8s = captures()
    one = run_raw(cu8s)
    pushed = run_raw(cu8s, PUSHES)
    for cu8, a, b in zip(cu8s, one, pushed):
        assert a == b
        recs = eng.parse_records(a)
        ref = port.decode(cu8)
        frames = [(r["lc"], r["nbits"], r["bits"]) for t, r in recs if t == eng.REC_FRAME]
        want = [(p["lc"], p["nbits"], p["bits"]) for t, p in ref.records if t == reftap.REC_FRAME]
        assert frames == want and len(frames) >= 2
        assert pdus(recs)[1] == ref.pids_frames
        assert kinds(recs) == oracle_kinds(ref)


def test_forced_state_between_pushes():
    """Sync forced back to NONE in the middle of the first frame: the stream re-acquires at its next block (a second
    SYNC record), and every P1 PDU it decodes is one the oracle decodes from the same capture.  The run is repeated
    with the same pushes: the records are byte-identical."""
    cu8s = captures()
    a = run_raw(cu8s, PUSHES, force=(12, 0))
    assert a == run_raw(cu8s, PUSHES, force=(12, 0))
    for cu8, raw in zip(cu8s, a):
        recs = eng.parse_records(raw)
        assert kinds(recs).count("S") >= 2
        p1 = pdus(recs)[0]
        ref = port.decode(cu8)
        assert p1 and all(f in ref.p1_frames for f in p1)
