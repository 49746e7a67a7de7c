"""GPU parity of the FINE sync phase of k_stream (front_sync): the reference carriers the demodulating teams store in
shared memory beside the kept bins, the data carriers staged while the Costas loops run, the MER tree, and the
record bookkeeping that runs beside the soft demap.

Every block's soft bits (REC_SOFT_PM), every MER record and every PDU must equal the oracle's.  Each case runs with
one CTA per stream (NRSC5_B200_CLUSTER=1: k_stream<false>, whose sync reads the reference carriers from shared
memory) and with the engine's default cluster (k_stream<true>: the helpers' symbols are gathered through L2).
The CPU twins run on the emulated kernels (tests/test_emu_fine_sync.py)."""
import numpy as np
import pytest

import common
import port
import reftap
from nrsc5_b200 import engine as eng
from nrsc5_b200 import synth
from test_gpu_chain import kinds, oracle_kinds, pdus, run_engine

pytestmark = pytest.mark.gpu

CLUSTERS = pytest.mark.parametrize("cluster", ["1", None], ids=["one_cta", "default_cluster"])


def set_cluster(monkeypatch, cluster):
    if cluster is None:
        monkeypatch.delenv("NRSC5_B200_CLUSTER", raising=False)
    else:
        monkeypatch.setenv("NRSC5_B200_CLUSTER", cluster)


def same_as_oracle(cu8, recs, soft=True):
    """PDUs, record order, MER and (with `soft`) every block's soft bits after the first two against the oracle."""
    ref = port.decode(cu8, want_soft=soft)
    frames = [(r["lc"], r["nbits"], r["bits"]) for t, r in recs if t == eng.REC_FRAME]
    want = [(p["lc"], p["nbits"], p["bits"]) for t, p in ref.records if t == reftap.REC_FRAME]
    assert frames == want
    assert pdus(recs)[1] == ref.pids_frames
    assert kinds(recs) == oracle_kinds(ref)
    mer = [r for t, r in recs if t == eng.REC_MER]
    want_mer = ref.of(reftap.REC_MER)
    assert len(mer) == len(want_mer)
    for a, b in zip(mer, want_mer):
        assert abs(a["lower"] - b["lower"]) < 0.05 and abs(a["upper"] - b["upper"]) < 0.05
    if soft:
        sa = [r for t, r in recs if t == eng.REC_SOFT_PM]
        sb = ref.of(reftap.REC_SOFT_PM)
        assert len(sa) == len(sb)
        for a, b in zip(sa[2:], sb[2:]):                  # (the blocks right after acquisition are skipped)
            x, y = a["soft"].astype(np.int16), b["soft"].astype(np.int16)
            assert np.abs(x - y).max() <= 1
    return frames


@CLUSTERS
def test_multi_stream_mp1_soft_bits_mer_and_pdus(cluster, monkeypatch):
    set_cluster(monkeypatch, cluster)
    caps = [synth.make_fm_mp1(nframes=2, seed=400 + i, lead_in=57 + 131 * i, cfo_hz=20.0 * i, noise_lsb=3.0)
            for i in range(3)]
    cu8s = [c.cu8[: c.cu8.size & ~3] for c in caps]
    outs = run_engine(cu8s, emit_soft=True)
    for cu8, recs in zip(cu8s, outs):
        frames = same_as_oracle(cu8, recs)
        assert len(frames) >= 2


@CLUSTERS
@pytest.mark.parametrize("name", ["mp3", "mp11"])
def test_extended_partitions(name, cluster, monkeypatch):
    """MP3 (12 partitions, P3 on PX1) and MP11 (14 partitions: 12 and 13 equalised in global memory, which PX2 reads)."""
    set_cluster(monkeypatch, cluster)
    cap = synth.make_fm_mp3(**common.MP3_CASE) if name == "mp3" else synth.make_fm(**common.FM_MODE_CASES["mp11"])
    cu8 = cap.cu8[: cap.cu8.size & ~3]
    frames = same_as_oracle(cu8, run_engine([cu8], emit_soft=True)[0])
    assert any(f[0] == 1 for f in frames)                 # P3 frames came out
    if name == "mp11":
        assert any(f[0] == 2 for f in frames)             # and P4


@CLUSTERS
def test_cfo_search_then_fine_sync(cluster, monkeypatch):
    """The acquisition runs the integer-CFO search: COARSE blocks vote on the reference carriers, the search writes
    them back into the bins, and the stream then reaches FINE sync."""
    set_cluster(monkeypatch, cluster)
    cap = synth.make_fm_mp1(**common.SYNTH_CASES["mp1_cfo2000_awgn20"])
    cu8 = cap.cu8[: cap.cu8.size & ~3]
    recs = run_engine([cu8], emit_soft=True)[0]
    same_as_oracle(cu8, recs, soft=False)
    assert any(r["cfo"] != 0 for t, r in recs if t == eng.REC_BLOCK)
